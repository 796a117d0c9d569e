"""Decoder option "opstatus" without a GPU: encoder round trips, the product's NIC table and record writer
(amb_decode_core.h compiled on the host) against the checker's, the header's macros against FIELDS_DTYPE, option
validation in Python and through the C ABI of the emulated library (tests/simt/library_emul.cc), opstatus_values, the
report lines and the CLI's --opstatus."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import emul_build  # noqa: E402
import opstatus_cases as oc  # noqa: E402
import opstatus_oracle as oo  # noqa: E402
import track_cases as tc  # noqa: E402

CORE_SHIM = r"""
#include "%s"
extern "C" int shim_nic(int tc, int sa, int sb, float* rc) { return amb_nic_table(tc, sa, sb, rc); }
extern "C" int shim_nucp(int tc) { return amb_nucp(tc); }
// the stage's per-record work on one frame and its option-off record: classify (TC 29 / 31 written at once), then, for
// a position, the lookup result given as a slot
extern "C" unsigned shim_classify(const amb_frame* f, amb_fields* r, uint32_t* info, uint32_t* extra)
{
    return amb_es_classify(*f, r, info, extra);
}
extern "C" int shim_position(amb_fields* r, int tc, int nicb, double t, double t_any, double t_surf, uint32_t any,
                             uint32_t surf, int S)
{
    AmbOpsSlot s = {t_any, t_surf, any, surf};
    return amb_es_position(r, tc, nicb, t, &s, S);
}
extern "C" void shim_layout(size_t* out)
{
    amb_fields rec;
    amb_fields* r = &rec;
    const char* b = (const char*)r;
#define OFF(x) (size_t)((const char*)&(x) - b)
    size_t v[] = {OFF(AMB_FIELDS_ES(r)), OFF(AMB_FIELDS_ES_VERSION(r)), OFF(AMB_FIELDS_ES_NIC(r)),
                  OFF(AMB_FIELDS_OPS_CC(r)), OFF(AMB_FIELDS_OPS_OM(r)), OFF(AMB_FIELDS_OPS_SUBTYPE(r)),
                  OFF(AMB_FIELDS_OPS_NIC_A(r)), OFF(AMB_FIELDS_OPS_NACP(r)), OFF(AMB_FIELDS_OPS_GVA(r)),
                  OFF(AMB_FIELDS_OPS_SIL(r)), OFF(AMB_FIELDS_OPS_NIC_BARO(r)), OFF(AMB_FIELDS_OPS_HRD(r)),
                  OFF(AMB_FIELDS_OPS_SIL_SUPP(r)), OFF(AMB_FIELDS_OPS_NIC_C(r)), OFF(AMB_FIELDS_OPS_LW(r)),
                  OFF(AMB_FIELDS_TS_ALT(r)), OFF(AMB_FIELDS_TS_BARO(r)), OFF(AMB_FIELDS_TS_HDG(r)),
                  OFF(AMB_FIELDS_TS_SIL_SUPP(r)), OFF(AMB_FIELDS_TS_ALT_TYPE(r)), OFF(AMB_FIELDS_TS_HDG_STATUS(r)),
                  OFF(AMB_FIELDS_TS_NACP(r)), OFF(AMB_FIELDS_TS_NIC_BARO(r)), OFF(AMB_FIELDS_TS_SIL(r)),
                  OFF(AMB_FIELDS_TS_MODES(r)), OFF(AMB_FIELDS_POS_NIC_A(r)), OFF(AMB_FIELDS_POS_NIC_B(r)),
                  OFF(AMB_FIELDS_POS_NIC_C(r)), OFF(AMB_FIELDS_POS_RC(r)),
                  sizeof(AMB_FIELDS_OPS_CC(r)), sizeof(AMB_FIELDS_TS_HDG(r)), sizeof(AMB_FIELDS_POS_RC(r)),
                  AMB_TS_MODE_STATUS, AMB_TS_AUTOPILOT, AMB_TS_VNAV, AMB_TS_ALT_HOLD, AMB_TS_APPROACH, AMB_TS_TCAS,
                  AMB_TS_LNAV, AMB_ES_NO_VERSION};
#undef OFF
    for (size_t i = 0; i < sizeof v / sizeof v[0]; i++) out[i] = v[i];
}
"""

# the header's slots: (offset in aux, or in pad_ for the first three)
SLOTS = [5, 6, 7, 0, 2, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 0, 2, 4, 6, 7, 8, 9, 10, 11, 12, 0, 1, 2, 4]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    src = tmp_path_factory.mktemp("opstatus_core") / "shim.cc"
    src.write_text(CORE_SHIM % os.path.join(ROOT, "gr_air_modes_b200", "csrc", "amb_decode_core.h"))
    s = C.CDLL(emul_build.build(tmp_path_factory, src))
    s.shim_nic.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float)]
    s.shim_classify.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    s.shim_classify.restype = C.c_uint
    s.shim_position.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_uint32,
                                C.c_uint32, C.c_int]
    return s


def test_round_trips_of_the_encoders():
    rng = np.random.default_rng(1)
    for _ in range(500):
        sub, ver = int(rng.integers(0, 8)), int(rng.integers(0, 8))
        v = dict(cc=int(rng.integers(0, 1 << 16)), om=int(rng.integers(0, 1 << 16)), nica=int(rng.integers(0, 2)),
                 nacp=int(rng.integers(0, 16)), gva=int(rng.integers(0, 4)), sil=int(rng.integers(0, 4)),
                 baro=int(rng.integers(0, 2)), hrd=int(rng.integers(0, 2)), silsupp=int(rng.integers(0, 2)))
        me = oc.opstatus_me(sub, ver, **v)
        b = oo.me_bits
        assert me < 1 << 56 and b(me, 1, 5) == 31 and b(me, 6, 3) == sub and b(me, 41, 3) == ver
        assert (b(me, 9, 16), b(me, 25, 16), b(me, 44, 1), b(me, 45, 4), b(me, 49, 2), b(me, 51, 2), b(me, 53, 1),
                b(me, 54, 1), b(me, 55, 1)) == tuple(v.values())
        nicc, lw = int(rng.integers(0, 2)), int(rng.integers(0, 16))
        me = oc.opstatus_me(1, ver, cc=v["cc"], nicc=nicc, lw=lw)
        assert b(me, 20, 1) == nicc and b(me, 21, 4) == lw and b(me, 9, 11) == v["cc"] >> 5
        t = dict(sub=int(rng.integers(0, 4)), silsupp=int(rng.integers(0, 2)), alt_type=int(rng.integers(0, 2)),
                 alt=int(rng.integers(0, 2048)), baro=int(rng.integers(0, 512)), hdg_status=int(rng.integers(0, 2)),
                 hdg=int(rng.integers(0, 512)), nacp=int(rng.integers(0, 16)), nicbaro=int(rng.integers(0, 2)),
                 sil=int(rng.integers(0, 4)), modes=int(rng.integers(0, 256)))
        me = oc.target_state_me(**t)
        assert b(me, 1, 5) == 29
        assert (b(me, 6, 2), b(me, 8, 1), b(me, 9, 1), b(me, 10, 11), b(me, 21, 9), b(me, 30, 1), b(me, 31, 9),
                b(me, 40, 4), b(me, 44, 1), b(me, 45, 2), b(me, 47, 8)) == tuple(t.values())
    for tcode in oc.AIRBORNE_TC + oc.SURFACE_TC:
        for nicb in (0, 1):
            fr, _ = oc.position(0x123, tcode, nicb)
            me = int.from_bytes(fr[4:11], "big")
            assert oo.me_bits(me, 1, 5) == tcode
            if tcode > 8:
                assert oo.me_bits(me, 8, 1) == nicb


def test_nic_table_against_the_checker(core):
    """Every type code and every supplement combination: the product's one table and the checker's literal copy."""
    rc = C.c_float()
    for tcode in oc.AIRBORNE_TC + oc.SURFACE_TC:
        assert core.shim_nucp(tcode) == oo.NUCP[tcode]
        for sa in (0, 1):
            for sb in (0, 1):
                nic = core.shim_nic(tcode, sa, sb, C.byref(rc))
                want_nic, want_rc = oo.lookup(tcode, sa, sb)
                assert nic == want_nic, (tcode, sa, sb)
                assert (math.isnan(rc.value) and want_rc is None) or rc.value == np.float32(want_rc), (tcode, sa, sb)


def _host_stage(core, frames, off, S):
    """The product's per-record functions run sequentially on the host, with the references found the checker's way:
    classify every record, then each position with its A / C slot."""
    from gr_air_modes_b200 import decode
    out = off.copy()
    slots = {}
    ts = oo.t_of(frames)
    info, extra = C.c_uint32(), C.c_uint32()
    for k in range(len(out)):
        f = np.ascontiguousarray(frames[k:k + 1])
        r = out[k:k + 1]
        kind = core.shim_classify(C.c_void_p(f.ctypes.data), C.c_void_p(r.ctypes.data), C.byref(info), C.byref(extra))
        a = int(out[k]["icao"])
        s = slots.setdefault(a, [math.nan, math.nan, 0xFFFFFFFF, 0xFFFFFFFF])
        if kind in (1, 2):
            s[0], s[2] = float(ts[k]), info.value
            if kind == 2:
                s[1], s[3] = float(ts[k]), extra.value
        elif kind == 3:
            core.shim_position(C.c_void_p(r.ctypes.data), int(info.value), int(extra.value), float(ts[k]), s[0], s[1],
                               s[2], s[3], S)
    assert out.dtype == decode.FIELDS_DTYPE
    return out


@pytest.mark.parametrize("name", ["table", "fields", "age", "burst", "case14"])
def test_core_functions_on_the_host_against_the_checker(core, emulated, name):
    """The record writer and the NIC arithmetic of amb_decode_core.h, fed the option-off records of the emulated
    decoder, give the checker's records byte for byte."""
    from gr_air_modes_b200 import decode
    msgs, S = next((m, s) for nm, m, s in oc.scenes() if nm == name)
    frames = tc.frames_of(msgs)
    d = decode.batch_decoder(None)
    off = d.decode(frames)
    d.close()
    want = oo.replay(frames, off, S)
    oo.assert_records_equal(_host_stage(core, frames, off, S), want, name)
    o = oo.outcome_of(want)
    assert np.any(o != oo.NOT_TRIED)


def test_header_macros_against_fields_dtype(core):
    from gr_air_modes_b200 import decode
    out = (C.c_size_t * 40)()
    core.shim_layout(out)
    pad = decode.FIELDS_DTYPE.fields["pad_"][1]
    aux = decode.FIELDS_DTYPE.fields["aux"][1]
    want = [pad + s for s in SLOTS[:3]] + [aux + s for s in SLOTS[3:]]
    assert list(out[:29]) == want
    assert list(out[29:32]) == [2, 2, 4]
    assert list(out[32:40]) == [0x80, 0x40, 0x20, 0x10, 0x04, 0x02, 0x01, 0xFF]
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    for name, v in (("NOT_TRIED", 0), ("OPSTATUS", 1), ("TARGET_STATE", 2), ("NIC", 3), ("NUC", 4), ("UNSUPPORTED", 5)):
        assert int(re.search(r"#define AMB_ES_%s (\d+)" % name, hdr).group(1)) == v == getattr(oo, name)
        assert getattr(decode, "ES_" + name) == v
    assert int(re.search(r"#define AMB_OPSTATUS_MAX (\d+)", hdr).group(1)) == decode.OPSTATUS_MAX == 600


def test_opstatus_values_and_outcome():
    from gr_air_modes_b200 import decode
    r = np.zeros(4, dtype=decode.FIELDS_DTYPE)
    aux = bytearray(16)
    aux[0:2], aux[2:4] = (0x1234).to_bytes(2, "little"), (0xABCD).to_bytes(2, "little")
    aux[4:14] = bytes([1, 1, 9, 2, 3, 1, 0, 1, 1, 7])
    oo.set_record(r[0:1], aux, oo.OPSTATUS, 2, 0)
    assert list(decode.opstatus_outcome(r)) == [oo.OPSTATUS, 0, 0, 0]
    v = decode.opstatus_values(r[0])
    assert v == {"kind": "opstatus", "version": 2, "subtype": 1, "capability": 0x1234, "op_mode": 0xABCD, "nic_a": 1,
                 "nacp": 9, "gva": 2, "sil": 3, "hrd": 0, "sil_supplement": 1, "trk_hdg": 1, "nic_c": 1,
                 "length_width": 7}
    assert decode.opstatus_values(decode.record_to_dict(r[0])) == v
    aux = bytearray(16)
    aux[0:2], aux[2:4], aux[4:6] = (1001).to_bytes(2, "little"), (267).to_bytes(2, "little"), (256).to_bytes(2, "little")
    aux[6:13] = bytes([1, 1, 1, 10, 1, 3, 0x80 | 0x40 | 0x04 | 0x02])
    oo.set_record(r[1:2], aux, oo.TARGET_STATE, 2, 0)
    v = decode.opstatus_values(r[1])
    assert v["selected_alt"] == 32000 and v["alt_source"] == "FMS" and abs(v["baro"] - 1012.8) < 1e-9
    assert v["heading"] == 180.0 and v["nacp"] == 10 and v["sil"] == 3 and v["sil_supplement"] == 1
    assert (v["autopilot"], v["vnav"], v["alt_hold"], v["approach"], v["lnav"], v["tcas"]) == (True, False, False, True,
                                                                                              False, True)
    aux[0:2] = aux[2:4] = bytes(2)
    aux[8] = 0
    aux[12] = 0x02
    oo.set_record(r[1:2], aux, oo.TARGET_STATE, 2, 0)
    v = decode.opstatus_values(r[1])
    assert v["selected_alt"] is None and v["baro"] is None and v["heading"] is None and v["autopilot"] is None
    assert v["tcas"] is True
    oo.set_record(r[2:3], bytes([1, 0, 1, 0]) + np.float32(370.4).tobytes() + bytes(8), oo.NIC, 2, 7)
    assert decode.opstatus_values(r[2]) == {"kind": "nic", "version": 2, "nic": 7, "nic_a": 1, "nic_b": 0, "nic_c": 1,
                                            "rc": float(np.float32(370.4))}
    oo.set_record(r[3:4], bytes(4) + np.float32(np.nan).tobytes() + bytes(8), oo.NUC, oo.NO_VERSION, 7)
    assert decode.opstatus_values(r[3]) == {"kind": "nuc", "version": None, "nucp": 7, "nic_a": 0, "nic_b": 0,
                                            "nic_c": 0, "rc": None}


def test_report_lines():
    from gr_air_modes_b200 import decode, report
    msgs = [m for m in oc.fields_scene() if bytes.fromhex(m[0])[0] >> 3 == 17 and bytes.fromhex(m[0])[4] >> 3 in (29, 31)]
    frames = tc.frames_of(msgs, unqueued_every=0)
    off = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    off["df"], off["status"], off["icao"] = 17, 1, [int.from_bytes(bytes(f["data"][1:4]), "big") for f in frames]
    on = oo.replay(frames, off, 30)
    strings = ["%s %06x 0.5 12 0.25" % (h, ecc) for h, ecc, _, _ in msgs]
    lines = [report.format_report(m, r) for m, r in zip(strings, on)]
    assert report.format_report(strings[0], off[0]) is None
    got = dict(zip([int(x) for x in oo.outcome_of(on)], lines))
    assert got[oo.OPSTATUS] is not None and got[oo.TARGET_STATE] is not None
    want_v0 = "(-3 12.25000000) Type 17 BDS6,5 (operational status) from 200 version 0 airborne capability 0000 mode 0000"
    assert lines[0] == want_v0
    full = [ln for ln in lines if ln and "version 2 surface capability ffff" in ln]
    assert full[0].endswith("surface capability ffff mode ffff NIC-A 1 NACp 15 SIL 3 NIC-C 1 TRK/HDG 1 L/W 15 HRD 1 "
                            "SIL supp 1")
    ts = [ln for ln, o in zip(lines, oo.outcome_of(on)) if o == oo.TARGET_STATE]
    assert any(ln.endswith("BDS6,2 (target state) from %x NACp 0 NICbaro 0 SIL 0" % a) for ln in ts for a in range(0x200, 0x205))
    assert any(ln.endswith("selected alt 65472ft (FMS) baro 1208.0mb heading 359.3 modes AP VNAV ALT APP LNAV TCAS "
                           "NACp 15 NICbaro 1 SIL 3") for ln in ts)
    for o, ln in zip(oo.outcome_of(on), lines):
        assert (ln is not None) == (o in (oo.OPSTATUS, oo.TARGET_STATE))


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    from gr_air_modes_b200 import _lib
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def test_option_validation_in_python():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, 600, 30.0):
        assert decode.check_opstatus(ok) == int(ok)
    for bad in (-1, 601, 1.5, True, None, "x"):
        with pytest.raises(ValueError):
            decode.check_opstatus(bad)
    assert _lib.OPSTATUS_MAX == decode.OPSTATUS_MAX == decode.OPTION_MAX["opstatus"] == 600


def test_option_validation_and_a_stream_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    for name, v in ((b"opstatus", 601), (b"opstatus", -1), (b"op_status", 5)):
        assert d._lib.amb_decoder_set_option(d._h, name, v) == -1
    assert d.get_opstatus() == 0
    for bad in (-1, 601):
        with pytest.raises(ValueError):
            d.set_opstatus(bad)
    frames = tc.frames_of(oc.age_scene(S=30))
    off = d.decode(frames)
    assert d.stats()[0] == 7
    d.close()
    d = decode.batch_decoder(None, opstatus=30)
    on = np.concatenate([d.decode(frames[:33]), d.decode(frames[33:])])
    assert d.stats()[0] == 2 * 13
    oo.assert_records_equal(on, oo.replay(frames, off, 30), "emulated C ABI")
    d.reset()
    assert d.get_opstatus() == 30
    again = d.decode(frames)
    oo.assert_records_equal(again, oo.replay(frames, off, 30), "after reset")
    d.close()


def _cli():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200
    return modes_rx_b200


def test_cli_parsing():
    cli = _cli()
    assert cli.parse_args(["-s", "x.cfile", "--reports", "--opstatus", "30"]).opstatus == 30
    assert cli.parse_args(["-s", "x.cfile", "-l", "1.0,2.0", "--opstatus", "600"]).opstatus == 600
    assert cli.parse_args(["-s", "x.cfile"]).opstatus == 0
    for bad in (["--opstatus", "30"], ["--reports", "--opstatus", "601"], ["--reports", "--opstatus", "-1"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["-s", "x.cfile"] + bad)
    assert "--opstatus" in cli.__doc__

