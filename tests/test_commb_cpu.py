"""Decoder option "commb" without a GPU: encoder -> checker round trips for random values of every field, the agreement
test of the product's arithmetic (amb_decode_core.h compiled on the host) at its boundaries, option validation in Python
and through the C ABI of the emulated library (tests/simt/library_emul.cc), the header's macros and offsets against
FIELDS_DTYPE (compiled on the host), commb_values, the report line and the CLI's --commb."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import commb_cases as cc  # noqa: E402
import commb_oracle as co  # noqa: E402
import track_cases as tc  # noqa: E402

CORE_SHIM = r"""
#include "amb_decode_core.h"
extern "C" int shim_agree(int gs, int trk, double speed, double track) { return amb_commb_agree(gs, trk, speed, track); }
extern "C" unsigned shim_candidates(uint64_t mb) { return amb_commb_candidates(mb); }
extern "C" void shim_layout(size_t* out)
{
    amb_fields r;
    const char* b = (const char*)&r;
    out[0] = (size_t)((const char*)&AMB_FIELDS_COMMB(&r) - b);
    out[1] = (size_t)((const char*)&AMB_FIELDS_COMMB_REG(&r) - b);
    out[2] = (size_t)((const char*)&AMB_FIELDS_COMMB_MASK(&r) - b);
    out[3] = (size_t)((const char*)&AMB_FIELDS_COMMB_CAND(&r) - b);
    for (int i = 0; i < 8; i++) out[4 + i] = (size_t)((const char*)&AMB_FIELDS_COMMB_RAW(&r, i) - b);
    out[12] = sizeof(AMB_FIELDS_COMMB_RAW(&r, 0));
}
extern "C" void shim_write(amb_fields* r, uint64_t mb, unsigned cand, int outcome, int g)
{
    amb_commb_write(r, mb, cand, outcome, g);
}
"""


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    d = tmp_path_factory.mktemp("commb_core")
    src = d / "shim.cc"
    src.write_text(CORE_SHIM)
    lib = str(d / "libshim.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-shared", "-fPIC",
                    "-I" + os.path.join(ROOT, "gr_air_modes_b200", "csrc"), "-o", lib, str(src)], check=True)
    s = C.CDLL(lib)
    s.shim_agree.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double]
    s.shim_candidates.argtypes = [C.c_uint64]
    s.shim_candidates.restype = C.c_uint
    s.shim_write.argtypes = [C.c_void_p, C.c_uint64, C.c_uint, C.c_int, C.c_int]
    return s


def test_round_trips_of_every_field():
    rng = np.random.default_rng(1)
    for reg in co.REGS:
        for _ in range(400):
            vals = {i: 0 for i in range(5) if rng.random() < 0.6}
            for i in list(vals):
                lo, hi = co.raw_range(reg, i)
                vals[i] = int(rng.integers(lo, hi + 1))
            mb = co.encode(reg, vals)
            _, raws, mask = co.read(mb, reg)
            assert mask == sum(1 << i for i in vals)
            assert raws == [vals.get(i, 0) for i in range(5)]
            assert mb < 1 << 56


def test_candidates_agree_with_the_product(core):
    """The checker's structural test and the product's (amb_commb_candidates) on random and constructed words."""
    rng = np.random.default_rng(2)
    words = [int(x) for x in rng.integers(0, 1 << 56, 3000, dtype=np.uint64)]
    words += [cc.unique_word(co.REGS[k % 3], rng) for k in range(300)]
    words += [cc.ambiguous_word(rng) for _ in range(100)]
    words += [int.from_bytes(bytes.fromhex(h)[4:11], "big") for h, _, _, _ in cc.limits_scene()]
    for mb in words:
        want = sum(1 << co.REGS.index(g) for g in co.candidates(mb))
        assert core.shim_candidates(mb) == want, hex(mb)


def test_agreement_at_its_boundaries(core):
    for gs, trk, speed, track, want in ((200, 0, 380.0, 10.0, 1), (200, 0, 380.0, 10.000001, 0), (200, 0, 420.0, 0.0, 1),
                                        (200, 0, 420.5, 0.0, 0), (200, 0, 379.5, 0.0, 0), (200, -1024, 400.0, 180.0, 1),
                                        (200, -1024, 400.0, 170.0, 1), (200, -1024, 400.0, 169.99, 0),
                                        (200, -6, 400.0, 359.0, 1), (200, 1023, 400.0, 185.0, 1), (200, 0, 400.0, 350.0, 1), (200, 0, 400.0, 349.9, 0),
                                        (200, 512, 400.0, 100.0, 1), (200, 512, 400.0, 79.9, 0)):
        assert core.shim_agree(gs, trk, speed, track) == want == co.agree(gs, trk, speed, track), (gs, trk, speed, track)


def test_header_macros_against_fields_dtype(core):
    from gr_air_modes_b200 import decode
    out = (C.c_size_t * 13)()
    core.shim_layout(out)
    pad = decode.FIELDS_DTYPE.fields["pad_"][1]
    aux = decode.FIELDS_DTYPE.fields["aux"][1]
    assert list(out[:4]) == [pad + 1, pad + 2, pad + 3, pad + 4]
    assert list(out[4:12]) == [aux + 2 * i for i in range(8)] and out[12] == 2
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    for name, v in (("NOT_TRIED", 0), ("DECODED", 1), ("RESOLVED", 2), ("AMBIGUOUS", 3), ("NONE", 4), ("MAX", 600)):
        assert int(re.search(r"#define AMB_COMMB_%s (\d+)" % name, hdr).group(1)) == v
        assert getattr(decode, "COMMB_" + name) == v
    # the product's record writer and the checker's, byte for byte
    rng = np.random.default_rng(3)
    for _ in range(200):
        reg = co.REGS[int(rng.integers(0, 3))]
        mb = cc.unique_word(reg, rng)
        a = np.zeros(1, dtype=decode.FIELDS_DTYPE)
        a["pad_"] = 0xAB00000000000011
        b = a.copy()
        core.shim_write(C.c_void_p(a.ctypes.data), mb, 1 << co.REGS.index(reg), co.DECODED, co.REGS.index(reg))
        co.set_record(b, mb, co.DECODED, reg, [reg])
        assert a.tobytes() == b.tobytes()


def test_commb_values_and_outcome():
    from gr_air_modes_b200 import decode
    r = np.zeros(2, dtype=decode.FIELDS_DTYPE)
    r["status"], r["df"] = 1, 20
    mb = co.encode(0x50, {0: -57, 1: -512, 2: 225, 4: 240})
    co.set_record(r[0:1], mb, co.RESOLVED, 0x50, [0x50, 0x60])
    assert list(decode.commb_outcome(r)) == [co.RESOLVED, co.NOT_TRIED]
    v = decode.commb_values(r[0])
    assert v == {"bds": 0x50, "roll": -57 * 45 / 256, "track": -90.0, "gs": 450.0, "track_rate": None, "tas": 480.0}
    assert decode.commb_values(r[1]) is None
    assert decode.commb_values(decode.record_to_dict(r[0])) == v
    co.set_record(r[1:2], co.encode(0x40, {0: 2000, 2: 2132, 3: 5}), co.DECODED, 0x40, [0x40])
    v = decode.commb_values(r[1])
    assert v["mcp_alt"] == 32000.0 and v["fms_alt"] is None and abs(v["baro"] - 1013.2) < 1e-9 and v["modes"] == 5
    co.set_record(r[1:2], co.encode(0x60, {0: 100, 1: 250, 2: 200, 3: -10, 4: 10}), co.DECODED, 0x60, [0x60])
    v = decode.commb_values(r[1])
    assert v["heading"] == 100 * 90 / 512 and v["ias"] == 250 and abs(v["mach"] - 0.8) < 1e-12 and v["baro_rate"] == -320
    assert v["inertial_rate"] == 320


def test_report_line():
    from gr_air_modes_b200 import decode, report
    r = np.zeros(3, dtype=decode.FIELDS_DTYPE)
    r["status"], r["df"], r["ecc"] = 1, 20, 0x4840D6
    co.set_record(r[0:1], co.encode(0x50, {0: -57, 1: -512, 2: 225, 4: 240}), co.RESOLVED, 0x50, [0x50, 0x60])
    co.set_record(r[1:2], co.encode(0x50, {1: -1000, 2: 200}), co.AMBIGUOUS, None, [0x50, 0x60])
    msg = "a0000000000000000000000000 4840d6 0.5 12 0.25"
    line = report.format_report(msg, r[0])
    assert line == ("(-3 12.25000000) Type 20 BDS5,0 track and turn report from 4840d6: roll -10.0 track -90.0 GS 450kt "
                    "TAS 480kt")
    assert report.format_report(msg, r[1]) is None and report.format_report(msg, r[2]) is None
    co.set_record(r[2:3], co.encode(0x60, {0: 100, 1: 250}), co.DECODED, 0x60, [0x60])
    r[2]["df"] = 21
    assert report.format_report(msg, r[2]).endswith("Type 21 BDS6,0 heading and speed report from 4840d6: heading 17.6 "
                                                    "IAS 250kt")


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    from gr_air_modes_b200 import _lib
    out = str(tmp_path_factory.mktemp("libsimt_commb") / "libairmodes_b200_emulated.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas",
                    "-Wno-psabi", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "simt", "library_emul.cc")],
                   check=True)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def test_option_validation_in_python():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, 600, 30.0):
        assert decode.check_commb(ok) == int(ok)
    for bad in (-1, 601, 1.5, True, None, "x"):
        with pytest.raises(ValueError):
            decode.check_commb(bad)
    assert _lib.COMMB_MAX == decode.COMMB_MAX == 600


def test_option_validation_and_a_stream_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    for name, v in ((b"commb", 601), (b"commb", -1), (b"comm_b", 5)):
        assert d._lib.amb_decoder_set_option(d._h, name, v) == -1
    assert d.get_commb() == 0
    for bad in (-1, 601):
        with pytest.raises(ValueError):
            d.set_commb(bad)
    frames = tc.frames_of(cc.reference_scene(S=30))
    off = d.decode(frames)
    assert d.stats()[0] == 7
    d.close()
    d = decode.batch_decoder(None, commb=30)
    on = np.concatenate([d.decode(frames[:33]), d.decode(frames[33:])])
    assert d.stats()[0] == 2 * 13
    co.assert_records_equal(on, co.replay(frames, off, 30), "emulated C ABI")
    d.reset()
    assert d.get_commb() == 30
    d.close()


def _cli():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200
    return modes_rx_b200


def test_cli_parsing():
    cli = _cli()
    assert cli.parse_args(["-s", "x.cfile", "--reports", "--commb", "30"]).commb == 30
    assert cli.parse_args(["-s", "x.cfile", "-l", "1.0,2.0", "--commb", "600"]).commb == 600
    assert cli.parse_args(["-s", "x.cfile"]).commb == 0
    for bad in (["--commb", "30"], ["--reports", "--commb", "601"], ["--reports", "--commb", "-1"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["-s", "x.cfile"] + bad)
