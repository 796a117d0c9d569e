"""The coverage stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_coverage.cuh, enqueued by the decoder's own
amb_decode_launch after the local CPR stage) on the host under the SIMT emulator (tests/simt/simt_emul.h), through the
decoder harness tests/simt/decode_emul.cc (with the coverage accessors of tests/simt/decode_coverage_emul.cc), against the sequential checker (tests/coverage_oracle.py) fed with the
decoder's own records: the grid byte for byte after every call, for single messages, cuts at 31/32/33 and random sizes,
with local_cpr on and off, across a reset; records chosen to fall all into one cell, onto every row edge and its
neighbouring doubles, onto every band edge, and records that must not count. Four mutants must fail: a kernel that
updates only the record's own band, a row from rint, a row from a comparison against 2.5, and a reset that leaves the
grid."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import coverage_oracle as co  # noqa: E402
import emul_build  # noqa: E402
import local_cpr_cases as lc  # noqa: E402
import track_cases as tc  # noqa: E402

LOC = (47.9, 11.1)
KERNEL = "gr_air_modes_b200/csrc/amb_decode_coverage.cuh"
HARNESS = os.path.join("tests", "simt", "decode_coverage_emul.cc")


def _bind(tmp_path_factory, src):
    """The decoder harness built from `src` (tests/simt/decode_coverage_emul.cc or a patched copy) and bound: the
    entry points of tests/emul_build.decode_emul plus the coverage accessors."""
    e = emul_build.decode_emul(tmp_path_factory, src)
    e.emul_set_coverage.argtypes = [C.c_void_p, C.c_int]
    e.emul_coverage.argtypes = [C.c_void_p, C.c_void_p]
    e.emul_coverage_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    return e


def _mutant(tmp_path, tmp_path_factory, rel, old, new):
    """The harness built from a copy of the sources under tmp_path in which the text `old`, which must occur exactly
    once in the file `rel`, reads `new`."""
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(emul_build.ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1, old
    p.write_text(src.replace(old, new))
    return _bind(tmp_path_factory, tmp_path / HARNESS)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(tmp_path_factory, os.path.join(emul_build.ROOT, HARNESS))


def _decode(e, h, frames, opts, coverage):
    """emul_decode of `frames` with the options `opts` and option coverage = `coverage`; returns the records."""
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    e.emul_set_coverage(h, coverage)
    assert e.emul_decode(h, C.c_void_p(frames.ctypes.data), len(frames), opts, C.c_void_p(recs.ctypes.data)) == 0
    return recs


def _grid(e, h):
    g = np.zeros((co.ROWS, co.BANDS), dtype=np.float64)
    e.emul_coverage(h, C.c_void_p(g.ctypes.data))
    return g


def _run(e, calls, loc, local_S=0, resets=()):
    """Decode the frame arrays `calls` one call each; the grid equal to the checker's after every call."""
    h = e.emul_new(17)
    assert h
    chk = co.CoverageChecker()
    for i, frames in enumerate(calls):
        if i in resets:
            e.emul_reset(h)
            chk.reset()
        recs = _decode(e, h, frames, emul_build.opts(loc, local_cpr=local_S), 1)
        want = chk.feed(recs)
        assert _grid(e, h).tobytes() == want.tobytes(), i
    e.emul_free(h)
    return chk.array()


def _cut(frames, splits):
    out, pos = [], 0
    for c in list(splits) + [len(frames)]:
        c = min(c, len(frames) - pos)
        if c > 0:
            out.append(frames[pos:pos + c])
            pos += c
    return out


def _scenes():
    for name, loc, msgs, _ in tc.scenes():
        if name in ("case11", "life", "traj", "burst"):
            yield name, loc if loc is not None else LOC, lc.remap_addresses(msgs)
    yield "chain", [48.0, 11.0], lc.chain_scene()


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


@pytest.mark.parametrize("local_S", [0, 10], ids=["global", "local_cpr"])
@pytest.mark.parametrize("name", ["case11", "life", "traj", "burst", "chain"])
def test_scene_in_batch_splits(emul, name, local_S):
    loc, msgs = next((lo, m) for nm, lo, m in _scenes() if nm == name)
    frames = tc.frames_of(msgs)
    grids = [_run(emul, _cut(frames, s), loc, local_S) for s in SPLITS]
    assert grids[0].tobytes() == grids[1].tobytes() and grids[0].any()


def test_random_batch_sizes_and_a_reset(emul):
    loc, msgs = next((lo, m) for nm, lo, m in _scenes() if nm == "traj")
    frames = tc.frames_of(msgs)
    rng = np.random.default_rng(7)
    calls = _cut(frames, [int(x) for x in rng.integers(1, 300, 12)])
    _run(emul, calls + calls[:3], loc, 10, resets=(len(calls),))


def _rec(bearing, rng, alt=5000, bds=0x05, df=17, status=0x30):
    from gr_air_modes_b200 import decode
    r = np.zeros(1, dtype=decode.FIELDS_DTYPE)
    r["df"], r["bds"], r["status"], r["altitude"], r["bearing"], r["range"] = df, bds, status, alt, bearing, rng
    return r


def _crafted(e, recs, h=None):
    """The stage alone over the records `recs` (one call); the grid must equal the checker's. Returns the grid."""
    own = h is None
    h = h or e.emul_new(10)
    recs = np.ascontiguousarray(np.concatenate(recs))
    assert e.emul_coverage_records(h, C.c_void_p(recs.ctypes.data), len(recs)) == 0
    got = _grid(e, h)
    if own:
        e.emul_free(h)
    return got, co.grid_of(recs)


def edge_records():
    """Every row edge 5i + 2.5, its neighbouring doubles, 0, 360 - ulp and 360, at altitudes cycling over every band
    edge and its neighbours; ranges increasing so that the last record of a cell shows in the grid."""
    bearings = [0.0, float(np.nextafter(360.0, 0.0)), 360.0]
    for i in range(72):
        e = 5.0 * i + 2.5
        bearings += [float(np.nextafter(e, 0.0)), e, float(np.nextafter(e, 400.0))]
    alts = sorted({-1300, -1000, 0, 1, 100000} | {a + d for a in co.ALTITUDES for d in (-1, 0, 1)})
    out, r = [], 1.0
    for k, b in enumerate(bearings):
        for j in range(3):
            r += 0.25
            out.append(_rec(b, r, alt=alts[(3 * k + j) % len(alts)], bds=0x06 if (k + j) % 7 == 0 else 0x05))
    return out


def test_records_on_every_row_and_band_edge(emul):
    got, want = _crafted(emul, edge_records())
    assert got.tobytes() == want.tobytes()
    assert (want > 0).sum() > 500


def test_a_block_whose_records_all_fall_into_one_cell(emul):
    rng = np.random.default_rng(3)
    ranges = rng.uniform(1, 300, 1024)
    recs = [_rec(float(b), float(r), alt=7000) for b, r in zip(rng.uniform(92.5, 97.5 - 1e-9, 1024), ranges)]
    got, want = _crafted(emul, recs)
    assert got.tobytes() == want.tobytes()
    assert (got[19, 4:] == ranges.max()).all() and not got[19, :4].any() and np.count_nonzero(got) == 5


def test_records_that_change_nothing(emul):
    """Not queued, no handler, not DF17, not a position, no range; ranges 0, -0.0, NaN: the grid stays all zeros."""
    recs = [_rec(10.0, 50.0, status=0x30 | 0x80), _rec(10.0, 50.0, status=0x30 | 0x01), _rec(10.0, 50.0, df=18),
            _rec(10.0, 50.0, bds=0x08), _rec(10.0, 50.0, bds=0x09), _rec(10.0, 50.0, status=0x10),
            _rec(10.0, 0.0), _rec(10.0, -0.0), _rec(10.0, float("nan"))]
    got, want = _crafted(emul, recs)
    assert not got.any() and got.tobytes() == want.tobytes()


def test_off_allocates_nothing_and_changes_no_record(emul):
    loc, msgs = next((lo, m) for nm, lo, m in _scenes() if nm == "life")
    frames = tc.frames_of(msgs)
    out = []
    for cov in (0, 1):
        h = emul.emul_new(17)
        recs = _decode(emul, h, frames, emul_build.opts(loc, local_cpr=10, track=20), cov)
        assert emul.emul_coverage(h, C.c_void_p(np.zeros(648).ctypes.data)) == cov
        emul.emul_free(h)
        out.append(recs.tobytes())
    assert out[0] == out[1]


def _caught(e):
    """Whether the harness `e` departs from the checker on the crafted records or on a scene across a reset."""
    try:
        got, want = _crafted(e, edge_records())
        assert got.tobytes() == want.tobytes()
        loc, msgs = next((lo, m) for nm, lo, m in _scenes() if nm == "traj")
        calls = _cut(tc.frames_of(msgs), [800, 800])
        _run(e, calls, loc, 0, resets=(2,))
    except AssertionError:
        return True
    return False


def test_the_harness_itself_passes(emul):
    assert not _caught(emul)


def test_a_kernel_updating_only_its_own_band_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, KERNEL, "for (int j = row0; j <= i; j++)", "for (int j = i; j <= i; j++)")
    assert _caught(e)


def test_a_row_from_rint_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, KERNEL, "const long long t = (long long)(r.bearing + 2.5);",
               "const long long t = (long long)rint(r.bearing / 5.0) * 5;")
    assert _caught(e)


def test_a_row_from_a_comparison_against_2_5_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, KERNEL, "const long long t = (long long)(r.bearing + 2.5);",
               "const long long f5 = (long long)r.bearing - (long long)r.bearing % 5; "
               "const long long t = f5 + (r.bearing - (double)f5 >= 2.5 ? 5 : 0);")
    assert _caught(e)


def test_a_reset_that_leaves_the_grid_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_kernels.cuh",
               "    if (st->cgrid)\n", "    if (false)\n")
    assert _caught(e)
