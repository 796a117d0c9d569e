"""Decoder option "local_cpr" without a GPU: the brute-force checker (tests/local_cpr_oracle.py) and the product's
__host__ __device__ arithmetic (amb_cpr_local in amb_decode_core.h, through the test-only host shim) against the
reference's cpr_resolve_local as recorded in tests/golden/local_cpr_golden.json.gz, every float bit for bit; the live
reference function on fresh seeds where the reference tree is present; option validation; the record layout."""
import ctypes as C
import gzip
import json
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "local_cpr_golden.json.gz")
REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")

import emul_build  # noqa: E402
import local_cpr_oracle as lo  # noqa: E402


def _golden():
    with gzip.open(GOLDEN, "rb") as f:
        return json.loads(f.read())["cases"]


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "local_cpr_host_shim.cc")))
    s.shim_cpr_local.argtypes = [C.c_double, C.c_double, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_double)]
    s.shim_sizeof_fields.restype = C.c_int
    return s


def test_golden_covers_the_regions():
    g = _golden()
    assert len(g) >= 3000
    assert any(r[0] < 0 for r in g) and any(r[0] > 0 for r in g)
    assert any(abs(r[0]) > 86.5 for r in g) and any(abs(abs(r[1]) - 180.0) < 0.3 for r in g)
    assert {r[4] for r in g} == {0, 1} and {r[5] for r in g} == {0, 1}


def test_checker_reproduces_the_reference_golden():
    bad = [r for r in _golden() if lo.resolve_local(*r[:6]) != (r[6], r[7])]
    assert not bad, bad[:5]


def test_product_arithmetic_reproduces_the_reference_golden(shim):
    out = (C.c_double * 2)()
    bad = []
    for r in _golden():
        shim.shim_cpr_local(r[0], r[1], r[2], r[3], r[4], r[5], out)
        if (out[0], out[1]) != (r[6], r[7]):
            bad.append((r, out[0], out[1]))
    assert not bad, bad[:5]


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "cpr.py")), reason="the reference's Python sources are not present")
def test_checker_against_the_live_reference_on_fresh_seeds():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_local_cpr_golden as mk
    mods = mk.load_reference()
    try:
        for seed in (7, 8):
            cases = mk.make_cases(seed, 1500)
            want = mk.run_reference(cases, mods)
            assert [list(lo.resolve_local(*c)) for c in cases] == want
    finally:
        mk.unload_reference()


def test_checker_semantics_on_a_small_stream():
    """No reference, a global fix, a local fix chained on it, a reference older than S, and the decoded position within
    a few metres of the one sent."""
    import decode_cases as dc
    aa = 0x4840D6
    msgs = []
    for t, lat, odd, surface in ((0.0, 52.0, 0, 1), (1.0, 52.0, 0, 0), (1.5, 52.0, 1, 0), (2.0, 52.001, 1, 1),
                                 (2.5, 52.002, 0, 1), (40.0, 52.003, 0, 1)):
        la, lo_ = dc.cpr_encode(lat, 4.0, odd, bool(surface))
        me = dc.me_surface(7, 10, 1, 5, odd, la, lo_) if surface else dc.me_airborne(11, dc.enc_alt12(1000), odd, la, lo_)
        fr, ecc = dc.df17(aa, me)
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
    recs = lo.decode_local(msgs, None, 10)
    assert [r["local"] for r in recs] == [lo.LOCAL_NO_REF, lo.LOCAL_NO_REF, lo.LOCAL_NOT_TRIED, lo.LOCAL_DECODED,
                                         lo.LOCAL_DECODED, lo.LOCAL_STALE]
    assert abs(recs[4]["lat"] - 52.002) < 1e-4 and abs(recs[4]["lon"] - 4.0) < 1e-4
    assert recs[3]["status"] & lo.do.FS_CPR_NO_POS and recs[3]["status"] & lo.do.FS_HAS_POS
    assert lo.decode_local(msgs, None, 0) == [dict(r, local=0) for r in lo.do.decode_batch(msgs, None)]


def test_option_validation_without_a_device():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, 600, 60.0):
        assert decode.check_local_cpr(ok) == int(ok)
    for bad in (-1, 601, 1.5, True, None, "x"):
        with pytest.raises(ValueError):
            decode.check_local_cpr(bad)
    assert (decode.LOCAL_NOT_TRIED, decode.LOCAL_DECODED, decode.LOCAL_NO_REF, decode.LOCAL_STALE, decode.LOCAL_REJECTED) \
        == (0, 1, 2, 3, 4) == (lo.LOCAL_NOT_TRIED, lo.LOCAL_DECODED, lo.LOCAL_NO_REF, lo.LOCAL_STALE, lo.LOCAL_REJECTED)
    assert _lib.LOCAL_CPR_MAX == decode.LOCAL_CPR_MAX == 600
    assert ("amb_decoder_set_option", C.c_int, [C.c_void_p, C.c_char_p, C.c_int]) in _lib.SYMBOLS
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    for name, v in (("NOT_TRIED", 0), ("DECODED", 1), ("NO_REF", 2), ("STALE", 3), ("REJECTED", 4), ("CPR_MAX", 600)):
        assert re.search(r"#define AMB_LOCAL_%s %d\b" % (name, v), hdr), name


def test_record_layout_is_unchanged(shim):
    import numpy as np
    from gr_air_modes_b200 import _lib, decode
    assert shim.shim_sizeof_fields() == 144 == C.sizeof(_lib.Fields)
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    assert re.search(r"uint64_t pad_;[^\n]*\n\} amb_fields;", hdr)
    assert decode.FIELDS_DTYPE.names[-1] == "pad_" and decode.FIELDS_DTYPE["pad_"] == np.dtype("<u8")
    assert decode.FIELDS_DTYPE.names == (
        "icao", "ecc", "df", "status", "bds", "subtype", "ca", "fs", "vs", "ri", "sl", "cc", "dr", "um", "ftc", "cat",
        "cpr_format", "surface", "eps", "ast", "bds2", "tti", "altitude", "squawk", "threat_alt", "cpr_lat", "cpr_lon",
        "aux", "ident", "lat", "lon", "range", "bearing", "val", "pad_")
    assert decode.FIELDS_DTYPE.itemsize == 144 and decode.FIELDS_DTYPE.fields["pad_"][1] == 136
    f = _lib.Fields()
    f.pad_ = 0x0304
    assert f.local == 4
    rec = np.zeros(2, dtype=decode.FIELDS_DTYPE)
    rec["pad_"] = [1, 0x0203]
    assert decode.local_outcome(rec).tolist() == [1, 3]
    assert decode.record_to_dict(rec[0])["pad_"] == 1


def test_report_prints_a_local_fix_as_the_reference_printer_prints_a_position():
    """report.format_report keys on FS_HAS_POS: a locally decoded BDS0,5 / BDS0,6 record gets msprint.py's position line
    (the same text as for a global fix), where the option-off record prints nothing (CPRNoPositionError)."""
    import decode_cases as dc
    from gr_air_modes_b200 import report
    loc = [52.3, 4.8]
    msgs = []
    for k, (t, odd, surface) in enumerate(((0.0, 0, 0), (0.5, 1, 0), (20.0, 0, 0), (21.0, 1, 1))):
        lat, lon = 52.0 + 0.001 * k, 4.0 + 0.002 * k
        la, lo_ = dc.cpr_encode(lat, lon, odd, bool(surface))
        me = dc.me_surface(7, 10, 1, 40, odd, la, lo_) if surface else dc.me_airborne(11, dc.enc_alt12(5000), odd, la, lo_)
        fr, ecc = dc.df17(0xABCDEF, me)
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
    text = dc.message_strings(msgs)
    off = lo.do.decode_batch(msgs, loc)
    on = lo.decode_local(msgs, loc, 60)
    assert [r["local"] for r in on] == [lo.LOCAL_NO_REF, lo.LOCAL_NOT_TRIED, lo.LOCAL_DECODED, lo.LOCAL_DECODED]
    assert report.format_report(text[2], off[2]) is None and report.format_report(text[3], off[3]) is None
    for k, kind in ((2, "BDS0,5 (position report)"), (3, "BDS0,6 (surface report)")):
        r = on[k]
        line = report.format_report(text[k], r)
        head = report.prefix(text[k].split()[2], msgs[k][2], msgs[k][3]) + "Type 17 %s from abcdef at (%.6f, %.6f)" % (kind, r["lat"], r["lon"])
        assert line.startswith(head), line
        assert ("(%.2f @ %.0f)" % (r["range"], r["bearing"])) in line
        # the same text as a global fix of that position would print
        g = dict(r, status=lo.do.FS_HAS_POS | lo.do.FS_HAS_RANGE)
        assert report.format_report(text[k], g) == line
