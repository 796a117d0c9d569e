"""The multilateration stage's kernels and C ABI (amb_mlat) on the CPU box: the emulated build of the library
(tests/simt/library_emul.cc, which takes amb_mlat.cuh in through amb_decode.cu) driven through gr_air_modes_b200.mlat,
against the CPU checker tests/mlat_oracle.py - the same groups exactly, the same statuses, positions within 1e-6 m
where the step counts agree - plus the grouping rules at their edges, batch-split invariance bit for bit, and the
argument checks. TEST INFRASTRUCTURE ONLY: sequential, like tests/test_library_simt.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from gr_air_modes_b200 import _lib
from gr_air_modes_b200 import mlat as ml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import mlat_cases as mc  # noqa: E402
import mlat_oracle as mo  # noqa: E402

T0 = (1_700_000_000, 0.125)


@pytest.fixture(scope="module", autouse=True)
def emulated_library(tmp_path_factory):
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def planes(rng, center, n=6):
    """Aircraft over the network (outside it, far from every baseline, a least-squares minimum need not be the truth)."""
    return [(0x400000 + i, center[0] + rng.uniform(-0.15, 0.15), center[1] + rng.uniform(-0.15, 0.15),
             int(rng.integers(40, 1800)) * 25) for i in range(n)]


def check(got, want):
    bad = mo.compare(got, want)
    assert not bad, bad[:5]


@pytest.mark.parametrize("seed,K,rate", [(1, 3, None), (5, 6, None), (2, 5, 20e6), (3, 8, 4e6), (4, 4, 20e6)])
def test_device_fixes_match_the_checker(seed, K, rate):
    rng = np.random.default_rng(seed)
    st, c = mc.random_geometry(rng, K, 150)
    frames, truth = mc.scene_frames(st, planes(rng, c), 40, rng, rate=rate, t0=T0, drop=0.15)
    m = ml.mlat_solver(st)
    got = m.process(frames, flush=True)
    ck = mo.Checker(st)
    want = ck.process(frames, flush=True)
    check(got, want)
    assert len(got) > 10
    s = m.stats()
    for k in ("eligible", "carried", "solved", "no_convergence", "degenerate", "too_few", "duplicate", "span"):
        assert s[k] == ck.counts[k], k
    if rate is None:                                  # exact stamps: every SOLVED fix within 1 cm of the truth
        where = {t["payload"]: t["ecef"] for t in truth}          # one payload: one aircraft at one place
        for f in got:
            if f["status"] == mo.SOLVED and f["n"] == 3:
                assert f["rms"] < 1e-3                    # three stations: the truth or its mirror, both exact
            elif f["status"] == mo.SOLVED:
                d = np.linalg.norm(np.array([f["x"], f["y"], f["z"]]) - where[bytes(f["data"][:f["nbits"] // 8])])
                assert d < 1e-2, d


def test_batch_split_invariance_bit_for_bit():
    rng = np.random.default_rng(7)
    st, c = mc.random_geometry(rng, 5, 100)
    frames, _ = mc.scene_frames(st, planes(rng, c), 60, rng, rate=20e6, t0=T0, spacing=1e-3, drop=0.1)
    one = ml.mlat_solver(st).process(frames, flush=True)
    m = ml.mlat_solver(st)
    parts = [m.process(p, end=e, flush=e is None) for p, e in mc.split(frames, T0, sorted(rng.uniform(0.01, 0.07, 4)))]
    assert np.concatenate(parts).tobytes() == one.tobytes()
    assert m.stats()["carried"] == 0


def _edge_case(W, gaps, stations=(0, 1, 2), secs=1_700_000_000):
    """Frames of one payload at stations[i], t_0 = (secs, 0.5), t_{i+1} = t_i + gaps[i] (exact)."""
    rng = np.random.default_rng(0)
    pl, ov = mc.payload(4, 0xABCDEF, 10000, rng)
    per = [[] for _ in range(4)]
    t = 0.5
    for i, k in enumerate(stations):
        per[k].append(mc.frame(pl, secs, t, ov))
        if i < len(gaps):
            t = t + gaps[i]
    return [np.array(p, mc.FRAME) if p else np.zeros(0, mc.FRAME) for p in per]


ST4 = [(52.0, 4.0, 10.0), (52.1, 4.2, 10.0), (51.9, 4.3, 10.0), (52.05, 4.05, 10.0)]


def _both(frames, W_us, end=None, flush=True):
    m = ml.mlat_solver(ST4, window_us=W_us)
    got = m.process(frames, end=end, flush=flush)
    ck = mo.Checker(ST4, window_us=W_us)
    want = ck.process(frames, end=end or (0, 0.0), flush=flush)
    check(got, want)
    s = m.stats()
    assert {k: s[k] for k in ck.counts} == ck.counts
    return got, s


def test_grouping_edges():
    W_us = 2.0 ** -11 * 1e6                           # W = 2^-11 s, exactly representable
    W = W_us / 1e6
    assert W == 2.0 ** -11
    # gap = W joins; gap = W + one ulp splits
    _, s = _both(_edge_case(W, [W, W / 2]), W_us)
    assert s["span"] == 1                             # joined: 3 frames, span 1.5 W
    _, s = _both(_edge_case(W, [W / 2, W / 2]), W_us)
    assert s["solved"] + s["no_convergence"] + s["degenerate"] == 1
    up = np.nextafter(0.5 + W, 1.0) - 0.5
    _, s = _both(_edge_case(W, [up, 0.0]), W_us)
    assert s["too_few"] == 2                          # split into a single and a pair
    # two stations; a duplicate station
    _, s = _both(_edge_case(W, [W / 4], stations=(0, 1)), W_us)
    assert s["too_few"] == 1
    _, s = _both(_edge_case(W, [W / 4, W / 4, W / 4], stations=(0, 1, 1, 2)), W_us)
    assert s["duplicate"] == 1


def test_completeness_edge_and_carry():
    W_us = 2.0 ** -11 * 1e6
    W = W_us / 1e6
    f = _edge_case(W, [W / 4, W / 4])
    t_last = 0.5 + W / 2
    secs = 1_700_000_000
    _, s = _both(f, W_us, end=(secs, t_last + W), flush=False)       # t_last + W = end: complete
    assert s["carried"] == 0 and s["solved"] + s["no_convergence"] + s["degenerate"] == 1
    _, s = _both(f, W_us, end=(secs, np.nextafter(t_last + W, 0.0)), flush=False)   # one ulp short: carried
    assert s["carried"] == 3
    m = ml.mlat_solver(ST4, window_us=W_us)
    assert len(m.process(f, end=(secs, t_last), flush=False)) == 0 and m.stats()["carried"] == 3
    m.reset()
    assert m.stats()["carried"] == 0
    assert len(m.process([np.zeros(0, mc.FRAME)] * 4, flush=True)) == 0


def test_nanosecond_differences_at_utc_magnitudes():
    """secs ~ 1.7e9: a 1 ns difference survives (secs + frac as one double would keep only ~2.4e-7 s)."""
    W_us = 2.0 ** -11 * 1e6
    f = _edge_case(None, [1e-9, 1e-9], secs=1_700_000_000)
    got, _ = _both(f, W_us)
    assert len(got) == 1


def test_argument_checks():
    with pytest.raises(ValueError):
        ml.mlat_solver(ST4[:2])
    with pytest.raises(ValueError):
        ml.mlat_solver(ST4 * 9)
    m = ml.mlat_solver(ST4)
    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError):
            m.set_window_us(bad)
    with pytest.raises(ValueError):
        m.set_offset(4, 0.0)
    with pytest.raises(ValueError):
        m.process([np.zeros(0, mc.FRAME)] * 3, flush=True)
    with pytest.raises(ValueError):
        m.process([np.zeros(0, mc.FRAME)] * 4)                       # neither end nor flush
    lib = _lib.load()
    # overflow: nothing changes, *n_out = the number due
    rng = np.random.default_rng(3)
    frames, _ = mc.scene_frames(ST4, planes(rng, (52.0, 4.1)), 5, rng, t0=T0)
    bufs = [(C.c_char * max(1, f.nbytes)).from_buffer_copy(f.tobytes() or b"\0") for f in frames]
    ptrs = (C.c_void_p * 4)(*[C.addressof(b) for b in bufs])
    counts = (C.c_int * 4)(*[len(f) for f in frames])
    n = C.c_int()
    out = np.zeros(8, ml.FIX_DTYPE)
    assert lib.amb_mlat_process(m._h, ptrs, counts, 0, 0.0, 1, out.ctypes.data, 2, C.byref(n)) == _lib.ERR_OVERFLOW
    assert n.value == 5 and m.stats()["eligible"] == 0
    assert lib.amb_mlat_process(m._h, ptrs, counts, 0, 0.0, 1, out.ctypes.data, 8, C.byref(n)) == 0 and n.value == 5
    # a station's frames out of time order
    rev = [f[::-1].copy() for f in frames]
    with pytest.raises(ValueError):
        m.process(rev, flush=True)
    assert m.stats()["eligible"] == 20


def test_offsets_shift_the_stamps():
    rng = np.random.default_rng(11)
    frames, _ = mc.scene_frames(ST4, planes(rng, (52.0, 4.1)), 10, rng, t0=T0)
    shifted = [f.copy() for f in frames]
    shifted[2]["frac"] += 3e-7
    a = ml.mlat_solver(ST4).process(frames, flush=True)
    b = ml.mlat_solver(ST4, offsets=[0, 0, 3e-7, 0]).process(shifted, flush=True)
    ck = mo.Checker(ST4, offsets=[0, 0, 3e-7, 0])
    check(b, ck.process(shifted, flush=True))
    assert len(a) == len(b) == 10
    assert np.allclose(a["x"], b["x"], atol=1e-3)


def test_carry_that_grows_across_calls():
    """An `end` that completes nothing carries almost every frame, twice: the scan buffers grow with the carry while
    the count's offsets are still to be read (they must be sized before the count)."""
    rng = np.random.default_rng(21)
    st, c = mc.random_geometry(rng, 3, 150)
    a, _ = mc.scene_frames(st, planes(rng, c), 200, rng, rate=20e6, t0=T0, spacing=2e-4)
    b, _ = mc.scene_frames(st, planes(rng, c), 200, rng, rate=20e6, t0=(T0[0], T0[1] + 0.05), spacing=2e-4)
    m, ck = ml.mlat_solver(st), mo.Checker(st)
    got = []
    for part in (a, b):
        got.append(m.process(part, end=(T0[0], 0.0), flush=False))
        check(got[-1], ck.process(part, end=(T0[0], 0.0)))
        assert len(got[-1]) == 0
    assert m.stats()["carried"] == ck.counts["carried"] == sum(len(f) for f in a + b)
    got.append(m.process([np.zeros(0, mc.FRAME)] * 3, flush=True))
    check(got[-1], ck.process([np.zeros(0, mc.FRAME)] * 3, flush=True))
    one = ml.mlat_solver(st).process([np.concatenate([x, y]) for x, y in zip(a, b)], flush=True)
    assert len(one) > 300 and np.concatenate(got).tobytes() == one.tobytes()


def test_rehearsal_at_the_gpu_tests_size():
    """tests/test_mlat_gpu.py's geometry and size (five stations, 80 transmissions, 20 Msps stamps) without the IQ; the
    derived fields against the truth: position, lat / lon / height and the emission time."""
    import test_mlat_gpu as tg
    from gr_air_modes_b200.mlat import ecef2llh
    rng = np.random.default_rng(8)
    planes80 = [(a, la, lo, int(round(h / 0.3048 / 25)) * 25) for a, la, lo, h in tg.AIRCRAFT]
    frames, _ = mc.scene_frames(tg.STATIONS, planes80, 80, rng, rate=20e6, t0=T0, spacing=1.2e-3)
    m = ml.mlat_solver(tg.STATIONS)
    got = m.process(frames, flush=True)
    check(got, mo.Checker(tg.STATIONS).process(frames, flush=True))
    assert len(got) == 80
    exact, truth = mc.scene_frames(tg.STATIONS, planes80, 80, np.random.default_rng(8), t0=T0, spacing=1.2e-3)
    fx = ml.mlat_solver(tg.STATIONS).process(exact, flush=True)
    assert len(fx) == 80
    for f, tr in zip(fx, truth):                      # one transmission per group, in time order
        assert f["status"] == mo.SOLVED and f["n"] == 5
        p = np.array([f["x"], f["y"], f["z"]])
        assert np.linalg.norm(p - tr["ecef"]) < 1e-2
        la, lo, h = ecef2llh(tr["ecef"])
        assert abs(f["lat"] - la) < 1e-9 and abs(f["lon"] - lo) < 1e-9 and abs(f["height"] - h) < 1e-2
        assert abs(mo.diff((int(f["secs"]), float(f["frac"])), (T0[0], T0[1] + tr["T"]))) < 1e-10
        assert f["rms"] < 1e-3 and f["dop"] > 0
