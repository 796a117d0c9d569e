"""Every comparison that carries the chain's bit-exactness claim, tested at its decision boundary and across every
instantiation of the scan, exact and slice kernels. Need an H100.

Random scenes at round thresholds almost never put a comparison within a few ulps of its threshold, so a contracted
FMA, a single-precision constant or a guard one rounding short in the kernels would go unnoticed by the other parity
tests. Here:
  A. every (samples per chip, PMF, pulse-offset) instantiation runs once against the oracle, in all chain forms;
  B. thresholds are bisected on their float32 bit pattern down to the two adjacent values between which the oracle's
     output changes, and the chain must equal the oracle on both sides (preamble_impl.cc:173-209);
  C. scenes of flat-topped int16-grid pulses make the comparisons tie exactly (peak test, late gate, quiet zone);
  D. 240-chip packets put chips exactly on llslicer's limits and on the packet rules' boundaries (slicer_impl.cc).
The oracle is pinned against the unmodified reference at the same points in tests/test_oracle_vs_ref.py.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

from helpers import EDGE_MATRIX, constructed_tie_cases, edge_scene, first_four, knife_edges, slicer_edge_packets
from test_gpu_parity import run_cuda

pytestmark = pytest.mark.gpu

_PORT = co.Port()


# ---- which kernel instantiation a rate runs (amb_launch_scan, amb_launch_exact, amb_launch_slice) --------------------
def scan_variant(p, pmf):
    """(SPC, PMF, PREF) of amb_scan_kernel: integer samples per chip (pulse offsets 2, 7, 9 x spc_i) use PREF 2 (spc <= 3)
    or 1 (spc >= 4) with PMF, 2 without; fractional ones PREF 0."""
    k = int(p.spc)
    integral = p.po[1] == 2 * k and p.po[2] == 7 * k and p.po[3] == 9 * k
    if not integral:
        return k, pmf, 0
    return k, pmf, ((2 if k <= 3 else 1) if pmf else 2)


def exact_variant(p, pmf):
    """SPC of amb_exact_kernel / amb_exact_warp_kernel / amb_slice_kernel: 1, 2, 5, 10 or the generic 0."""
    k = int(p.spc)
    return (k if p.spc == k and k in (1, 2, 5, 10) else 0), pmf


SCAN_TEMPLATES = {(k, pmf, pref) for k in range(1, 11) for pmf in (True, False)
                  for pref in (((2 if k <= 3 else 1) if pmf else 2), 0)}
# spc_f <= AMB_MAX_SPC = 10 (compute_params), so spc_i == 10 only at exactly 20 Msps: never fractional
SCAN_UNREACHABLE = {(10, True, 0), (10, False, 0)}
_SCAN_RUN = {scan_variant(_PORT.params(r, 7.0), pmf) for r, pmf in EDGE_MATRIX}
_EXACT_RUN = {exact_variant(_PORT.params(r, 7.0), pmf) for r, pmf in EDGE_MATRIX}
assert len(SCAN_TEMPLATES) == 40
assert _SCAN_RUN == SCAN_TEMPLATES - SCAN_UNREACHABLE, sorted(SCAN_TEMPLATES - SCAN_UNREACHABLE - _SCAN_RUN)
assert _EXACT_RUN == {(k, pmf) for k in (0, 1, 2, 5, 10) for pmf in (True, False)}, sorted(_EXACT_RUN)


def _bits(x):
    return int(np.array(x, np.float32).view(np.uint32))


def assert_frames(frames, want, where):
    """Every amb_frame field as test_frames_bit_exact_vs_oracle compares them; the reference level as bits."""
    assert [f.sample_index for f in frames] == [int(x) for x in want.index], where
    for f, g in zip(frames, want.frames):
        assert bytes(f.data) == bytes(g.data) and f.crc == g.crc and f.nbits == g.nbits, where
        assert f.numlowconf == g.numlowconf and bytes(f.lowconfbits) == bytes(g.lowconfbits), where
        assert f.passed == g.passed and _bits(f.ref_level) == _bits(g.ref_level), where
        assert f.secs == g.secs and f.frac == g.frac, where


def check_chain(iq, rate, t, pmf, where, chunks=None):
    """The fused chain one-shot, with the parallel resolver, with the row-based exact kernel forced and (if given) in
    ragged chunks: each equals the oracle frame for frame. Returns the oracle's result."""
    want = _PORT.run_iq(iq, rate, t, pmf, co.MA_CANONICAL)
    runs = [{}, dict(resolver=1), dict(exact_dense=0)] + ([dict(chunks=chunks)] if chunks else [])
    for kw in runs:
        msgs, frames, rx = run_cuda(iq, rate, t, pmf, **kw)
        assert msgs == want.msgs, (where, kw)
        assert_frames(frames, want, (where, kw))
        rx.close()
    return want


def check_split_form(bb, avg, rate, t, where):
    """amb_preamble_process on the float streams (amb_exact_streams_kernel): packets and tags bit-exact."""
    want = _PORT.run_streams(bb, avg, rate, t)
    chips, tags = am.preamble(rate, t).process(bb, avg)
    assert [x[0] for x in tags] == [int(x) for x in want.index], where
    assert np.array_equal(chips.view(np.uint32), np.asarray(want.chips, np.float32).reshape(-1, 240).view(np.uint32)), where


def candidates(iq, rate, t, pmf):
    """(scan candidates, exact verdicts) of one flushed one-shot call (amb_debug_candidates)."""
    rx = am.rx_path(rate, t, am.msg_queue(), use_pmf=pmf)
    rx.process(iq, flush=True)
    idx = (C.c_uint64 * (1 << 20))(); info = (C.c_uint32 * (1 << 20))()
    n = rx._ctx.call("amb_debug_candidates", idx, info, 1 << 20)
    cand = {int(idx[k]) for k in range(n)}
    real = {int(idx[k]) for k in range(n) if info[k] & 0x100}
    rx.close()
    return cand, real


@functools.lru_cache(maxsize=None)
def scene_edges(rate, pmf):
    sc = edge_scene(rate, pmf)
    bb, avg = _PORT.frontend(sc.iq, rate, pmf, co.MA_CANONICAL)
    return sc, bb, avg, knife_edges(_PORT, bb, avg, rate)[0]


# ---- A: the rate x PMF matrix --------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,pmf", EDGE_MATRIX)
def test_every_kernel_instantiation_matches_the_oracle(rate, pmf):
    sc = edge_scene(rate, pmf)
    rng = np.random.default_rng(int(rate) // 1000 + pmf)
    chunks = [int(c) for c in rng.integers(1, 40_000, 400)]
    want = check_chain(sc.iq, rate, 7.0, pmf, (rate, pmf), chunks=chunks)
    assert len(want.index) > 0


def test_rates_above_20_msps_are_refused():
    """Why SCAN_UNREACHABLE is unreachable: spc_i == 10 with a fractional spc would need a rate above 20 Msps."""
    for rate in (20e6 + 2, 20.5e6, 21e6):
        with pytest.raises(RuntimeError):
            am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)


# ---- B: threshold knife edges --------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,pmf", EDGE_MATRIX)
def test_threshold_knife_edges(rate, pmf):
    sc, bb, avg, edges = scene_edges(rate, pmf)
    assert edges, (rate, pmf)
    for lo, hi, kind in edges:
        for t in (lo, hi):
            where = (rate, pmf, t, kind)
            check_chain(sc.iq, rate, t, pmf, where)
            check_split_form(bb, avg, rate, t, where)
            if kind != "pulse":
                continue
            # the scan kernel is a filter with lowered thresholds: at the pulse test's margin it must still report
            # every candidate that passes :173-179, and the exact stage must decide each exactly as they do
            want = {int(x) for x in first_four(bb, avg, rate, t, _PORT)}
            cand, real = candidates(sc.iq, rate, t, pmf)
            assert want <= cand, (where, sorted(want - cand))
            assert real == want, (where, sorted(real ^ want))


def test_both_kinds_of_knife_edge_are_reached():
    """A seed or scene change must not quietly leave one kind of edge untested."""
    kinds = [e[2] for r, pmf in EDGE_MATRIX for e in scene_edges(r, pmf)[3]]
    n_pulse, n_quiet = kinds.count("pulse"), kinds.count("quiet")
    print("knife edges: %d pulse, %d quiet-zone / late-gate" % (n_pulse, n_quiet))
    assert n_pulse >= 100 and n_quiet >= 100, (n_pulse, n_quiet)


# ---- C: constructed ties -------------------------------------------------------------------------------------------
def test_constructed_ties(port):
    """Exact ties (asserted on the oracle's bb and avg while the cases are built): the chain must decide them as the
    reference does - equal is not greater at :175, :188, :206 and :208."""
    cases, seen = constructed_tie_cases(port)
    assert seen == {"peak": {False, True}, "late_tie": {False, True}, "quiet": {False, True}}, seen
    for case in cases:
        check_chain(case.iq, case.rate, case.threshold_db, case.pmf, case.name)
        bb, avg = port.frontend(case.iq, case.rate, case.pmf, co.MA_CANONICAL)
        check_split_form(bb, avg, case.rate, case.threshold_db, case.name)
    assert len(cases) >= 12, [c.name for c in cases]


# ---- D: slicer knife edges -----------------------------------------------------------------------------------------
def test_slicer_knife_edges(port):
    chips, facts = slicer_edge_packets()
    n = chips.shape[0]
    secs = np.arange(n, dtype=np.uint64)
    frac = np.linspace(0.0, 0.999, n)
    want = port.run_slicer(chips, secs, frac)
    q = am.msg_queue()
    frames = am.slicer(q).process(chips, list(zip(secs, frac)))
    assert len(frames) == len(want.frames) == n
    for k, (f, g) in enumerate(zip(frames, want.frames)):
        assert bytes(f.data) == bytes(g.data) and f.crc == g.crc and f.nbits == g.nbits, k
        assert f.numlowconf == g.numlowconf and bytes(f.lowconfbits) == bytes(g.lowconfbits), k
        assert f.passed == g.passed, k
        # NaN payloads differ between x86 and the GPU; every other level is compared bit for bit
        assert _bits(f.ref_level) == _bits(g.ref_level) or (np.isnan(f.ref_level) and np.isnan(g.ref_level)), k
    assert q.strings() == want.msgs
    # the construction does what it claims: a single-precision 1.414 or 0.707 gives another limit at these levels ...
    for r, const in ((facts["ref_1414"], 1.414), (facts["ref_0707"], 0.707)):
        assert np.float32(np.float64(r) * const) != np.float32(np.float64(r) * np.float64(np.float32(const)))
    assert facts["order_ref"] == 0.25
    # ... and the packet rules decide both ways
    assert {g.passed for g in want.frames} == {0, 1} and {g.numlowconf for g in want.frames} >= {9, 10, 0, 1}
