"""Decoder option "coverage" without a GPU: the sequential checker (tests/coverage_oracle.py) against the unmodified
reference az_map.py as recorded in tests/golden/coverage_golden.json.gz - (a) addRecord on boundary triples, every
changed cell bit for bit, and (b) az_map_output.output over whole scenes, fed here with the CPU oracle's records; option
validation in Python and through the C ABI of the emulated library (tests/simt/library_emul.cc); the header constants;
coverage_to_dict; the CLI's --coverage rules and the JSON it writes."""
import ctypes as C
import gzip
import json
import math
import os
import re
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
GOLDEN = os.path.join(ROOT, "tests", "golden", "coverage_golden.json.gz")

import coverage_oracle as co  # noqa: E402
import emul_build  # noqa: E402
import make_coverage_golden as mcg  # noqa: E402
import track_cases as tc  # noqa: E402
from oracle import decode_oracle  # noqa: E402

ERR_INVALID, ERR_STATE = -1, -8


def _bits(x: float) -> bytes:
    return struct.pack("<d", x)


@pytest.fixture(scope="module")
def golden():
    with gzip.open(GOLDEN, "rb") as f:
        return json.loads(f.read())


def test_checker_reproduces_the_boundary_calls(golden):
    """Every addRecord call of (a): the cells the checker changes and their new values, bit for bit, and the final
    grid. The calls reach every row edge from both sides, every band edge, 360 - ulp, 360, zero and subnormal ranges."""
    grid = co.empty()
    for b, a, r, changed in golden["calls"]:
        before = [row[:] for row in grid]
        co.add(grid, b, a, r)
        got = [[i, j, grid[i][j]] for i in range(co.ROWS) for j in range(co.BANDS) if _bits(grid[i][j]) != _bits(before[i][j])]
        assert [(i, j, _bits(v)) for i, j, v in got] == [(i, j, _bits(v)) for i, j, v in changed], (b, a, r)
    assert [_bits(v) for row in grid for v in row] == [_bits(v) for row in golden["final"] for v in row]
    bearings = {c[0] for c in golden["calls"]}
    assert float(np.nextafter(2.5, 0.0)) in bearings and 357.5 in bearings and 360.0 in bearings
    assert co.cell(float(np.nextafter(2.5, 0.0)), 0)[0] == 1 and co.cell(357.5, 0)[0] == 0 and co.cell(360.0, 0)[0] == 0
    assert {c[2] for c in golden["calls"]} >= {0.0, 5e-324}


def _ulps(a: float, b: float) -> int:
    ia, ib = struct.unpack("<q", _bits(a))[0], struct.unpack("<q", _bits(b))[0]
    return abs(ia - ib)


def within_bounds(ours, ref):
    """DESIGN.md §8's bounds for a record's (bearing, altitude, range) against CPython's: range <= 2 ulp, bearing <= 1
    ulp, the same altitude."""
    return ours[1] == ref[1] and _ulps(ours[2], ref[2]) <= 2 and _ulps(ours[0], ref[0]) <= 1


def explain(grid, want, ours, ref, close=within_bounds):
    """Cells where `grid` (the checker's over our records) differs from `want` (the reference's), and whether each is
    explained: a counted record of the same message whose (bearing, altitude, range) is close(ours, ref) to the
    reference's and whose cell, ours or the reference's, is in that row. `ours` / `ref`: {message index: (bearing,
    altitude, range)} of the counted records."""
    assert set(ours) == set(ref)
    off = {k for k in ours if ours[k] != ref[k]}
    for k in off:
        assert close(ours[k], ref[k]), (k, ours[k], ref[k])
    rows = {co.cell(*ours[k][:2])[0] for k in off} | {co.cell(*ref[k][:2])[0] for k in off}
    cells = [(i, j) for i in range(co.ROWS) for j in range(co.BANDS) if _bits(float(grid[i][j])) != _bits(float(want[i][j]))]
    return cells, [c for c in cells if c[0] not in rows], sorted(off)


def test_checker_on_the_oracles_records_against_the_reference_scenes(golden):
    """(b): the checker over oracle/decode_oracle.py's records of every golden scene against az_map_output's grid. A
    cell may differ only where a counted record's range / bearing differs from CPython's within the §8 bounds; every
    such cell is listed, and none is expected."""
    scenes = {name: (loc, msgs) for name, loc, msgs in mcg.scenes()}
    assert len(golden["scenes"]) == len(scenes) >= 10
    for sc in golden["scenes"]:
        loc, msgs = scenes[sc["name"]]
        assert mcg.digest(msgs) == sc["digest"] and loc == sc["location"], sc["name"]
        recs = decode_oracle.decode_batch(msgs, loc)
        ours = {k: co.counted(r) for k, r in enumerate(recs) if co.counted(r) is not None}
        ref = {k: (b, a, r) for k, b, a, r in sc["records"]}
        cells, unexplained, records = explain(co.grid_of(recs), sc["grid"], ours, ref)
        assert not unexplained, (sc["name"], unexplained)
        assert cells == [] and records == [], (sc["name"], cells, records)
        assert sc["type_errors_without_location"] > 0
        assert not co.grid_of(decode_oracle.decode_batch(msgs, None)).any()   # nothing counts without a location
    assert sum(len(sc["records"]) for sc in golden["scenes"]) > 5000
    assert any(a >= 30000 for sc in golden["scenes"] for _, _, a, _ in sc["records"])


@pytest.mark.skipif(not os.path.isdir(mcg.mdg.REF), reason="reference tree not present")
def test_live_reference_on_fresh_seeds():
    """Where the reference tree is present: az_map_output over a fresh trajectory scene equals the checker."""
    import local_cpr_cases as lc
    mods = mcg.load_reference()
    try:
        msgs, _ = lc.trajectory_scene(23, n_aircraft=30, seconds=90.0, drop=0.3, surface_share=0.3)
        _, grid, te = mcg.run_output(mods, [48.0, 11.0], msgs)
    finally:
        mcg.mdg.unload_reference()
        for k in ("PyQt4", "PyQt4.QtCore", "PyQt4.QtGui"):
            sys.modules.pop(k, None)
    assert te == 0
    want = co.grid_of(decode_oracle.decode_batch(msgs, [48.0, 11.0]))
    assert np.array(grid).tobytes() == want.tobytes() and want.any()


def test_header_constants():
    from gr_air_modes_b200 import _lib, decode
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    assert re.search(r"#define AMB_COVERAGE_ROWS 72\b", hdr) and re.search(r"#define AMB_COVERAGE_BANDS 9\b", hdr)
    alts = re.search(r"#define AMB_COVERAGE_ALTITUDES \{([^}]*)\}", hdr).group(1)
    assert tuple(int(x) for x in alts.split(",")) == decode.COVERAGE_ALTITUDES == co.ALTITUDES
    assert (decode.COVERAGE_ROWS, decode.COVERAGE_BANDS) == (co.ROWS, co.BANDS) == (72, 9)
    assert len(decode.COVERAGE_ALTITUDES) == decode.COVERAGE_BANDS
    for sym in ("amb_decoder_coverage", "amb_decoder_coverage_device", "amb_decoder_coverage_reset"):
        assert any(s[0] == sym for s in _lib.SYMBOLS) and re.search(r"AMB_API int %s\(" % sym, hdr)


def test_option_validation_in_python():
    from gr_air_modes_b200 import decode
    for ok in (0, 1, True, False, np.bool_(True)):
        assert decode.check_coverage(ok) == int(ok)
    for bad in (2, -1, "1", 1.0, None):
        with pytest.raises(ValueError):
            decode.check_coverage(bad)


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


def test_option_validation_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder([48.0, 11.0])
    lib = d._lib
    buf = (C.c_double * 648)()
    assert lib.amb_decoder_coverage(d._h, buf) == ERR_STATE
    assert lib.amb_decoder_coverage_device(d._h, buf) == ERR_STATE
    assert lib.amb_decoder_coverage_reset(d._h) == ERR_STATE
    for v in (2, -1, 7):
        assert lib.amb_decoder_set_option(d._h, b"coverage", v) == ERR_INVALID
    assert lib.amb_decoder_coverage(None, buf) == ERR_INVALID
    for fn in (d.coverage, d.reset_coverage):
        with pytest.raises(RuntimeError):
            fn()
    with pytest.raises(ValueError):
        d.set_coverage(2)
    assert not d.get_coverage()
    d.set_coverage(True)
    assert d.get_coverage()
    got = d.coverage()                                   # on, nothing decoded yet: all zeros
    assert got.shape == (72, 9) and got.dtype == np.float64 and not got.any()
    d.reset_coverage()
    assert lib.amb_decoder_coverage(d._h, None) == ERR_INVALID
    d.close()


def test_a_stream_through_the_c_abi(emulated):
    """Records unchanged by the option, one launch more per decode, the grid equal to the checker's after every call;
    reset_coverage clears only the grid, amb_decoder_reset everything; off keeps the grid; a location change leaves it."""
    from gr_air_modes_b200 import decode
    loc, msgs = [48.0, 11.0], next(m for n, _, m, _ in tc.scenes() if n == "traj")
    frames = tc.frames_of(msgs)
    cuts = ((0, 100), (100, 1033), (1033, len(frames)))
    plain = decode.batch_decoder(loc, local_cpr=10)
    want = [plain.decode(frames[a:b]) for a, b in cuts]
    k_plain = plain.stats()[0]
    plain.close()
    d = decode.batch_decoder(loc, local_cpr=10, coverage=True)
    chk = co.CoverageChecker()
    for (a, b), w in zip(cuts, want):
        recs = d.decode(frames[a:b])
        assert recs.tobytes() == w.tobytes()
        assert d.coverage().tobytes() == chk.feed(recs).tobytes()
    assert d.stats()[0] == k_plain + len(cuts)
    assert chk.array().any()
    full = d.coverage()
    d.set_location([48.5, 11.5])                         # later ranges change, the grid stays
    assert d.coverage().tobytes() == full.tobytes()
    d.set_location(loc)
    d.reset_coverage()                                   # only the grid: the CPR state stays
    chk.reset()
    assert not d.coverage().any()
    other = decode.batch_decoder(loc, local_cpr=10)
    for a, b in cuts:
        other.decode(frames[a:b])
    tail = frames[-300:]
    r1, r2 = d.decode(tail), other.decode(tail)
    other.close()
    assert r1.tobytes() == r2.tobytes()
    assert d.coverage().tobytes() == chk.feed(r1).tobytes()
    d.set_coverage(False)                                # off: the grid is kept, decodes leave it alone
    d.decode(frames[:500])
    d.set_coverage(True)
    assert d.coverage().tobytes() == chk.array().tobytes()
    d.reset()
    assert not d.coverage().any()
    d.close()


def test_coverage_to_dict():
    from gr_air_modes_b200 import decode
    g = np.zeros((72, 9))
    g[0, 3:] = 12.5
    g[71, 8] = 5e-324
    d = decode.coverage_to_dict(g, (48.0, 11.0))
    assert json.loads(json.dumps(d)) == d
    assert d["location"] == [48.0, 11.0] and d["unit"] == "statute miles"
    assert d["altitudes"] == list(decode.COVERAGE_ALTITUDES)
    assert [b["altitude"] for b in d["bands"]] == [0, 1000, 2000, 5000, 10000, 15000, 20000, 25000, None]
    assert len(d["sectors"]) == 72
    assert d["sectors"][0] == {"bearing": 0.0, "from": 357.5, "to": 2.5}
    assert d["sectors"][1] == {"bearing": 5.0, "from": 2.5, "to": 7.5}
    assert d["sectors"][71] == {"bearing": 355.0, "from": 352.5, "to": 357.5}
    for i, s in enumerate(d["sectors"]):                 # each sector's own bearings land in its row ...
        for b in (s["bearing"], s["from"], s["from"] + 1e-9, s["to"] - 1e-9 if i else 2.0):
            assert co.cell(b, 0)[0] == i
        if 0 < i < 71:                                   # ... up to the rounding of bearing + 2.5 next to an edge
            assert co.cell(float(np.nextafter(s["to"], 0.0)), 0)[0] in (i, i + 1)
    assert np.array(d["ranges"]).tobytes() == g.tobytes()
    assert decode.coverage_to_dict(g, None)["location"] is None


def test_cli_arguments():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200 as m
    assert m.parse_args(["-s", "x.cfile", "-l", "1,2", "--coverage", "c.json"]).coverage == "c.json"
    assert m.parse_args(["-s", "x.cfile"]).coverage is None
    with pytest.raises(SystemExit):
        m.parse_args(["-s", "x.cfile", "--coverage", "c.json"])
    with pytest.raises(SystemExit):
        m.parse_args(["-s", "x.cfile", "--reports", "--coverage", "c.json"])


def test_cli_writes_the_grid_after_every_chunk(emulated, tmp_path):
    """The CLI's report_queue with coverage=PATH (what -l LAT,LON --coverage PATH builds): after every flush PATH holds
    coverage_to_dict of the checker's grid over the same records, written through a temporary file."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200 as m
    from gr_air_modes_b200 import decode
    loc, msgs = [48.0, 11.0], next(x for n, _, x, _ in tc.scenes() if n == "traj")
    texts = ["%s %06x 0.5 %d %r" % (h, e, s, f) for h, e, s, f in msgs]
    path = tmp_path / "cov.json"
    q = m.report_queue(loc, 0, out=None, coverage=str(path))
    chk = co.CoverageChecker()
    ref = decode.batch_decoder(loc)
    for a, b in ((0, 700), (700, len(texts))):
        for t in texts[a:b]:
            q.handle(type("msg", (), {"to_string": lambda self, t=t: t})())
        q.flush()
        chk.feed(ref.decode_messages(texts[a:b]))
        got = json.loads(path.read_text())
        assert got == json.loads(json.dumps(decode.coverage_to_dict(chk.array(), loc)))
        assert not [p for p in os.listdir(tmp_path) if ".tmp" in p]
    q.close()
    ref.close()
    assert chk.array().any() and not math.isnan(chk.array().sum())
