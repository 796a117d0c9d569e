"""Parity tests proper: the CUDA path through the C ABI vs the CPU oracle / reference goldens. Need an H100."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

from helpers import first_four, load_golden, parse_msg

pytestmark = pytest.mark.gpu


def device_resident(iq):
    """The recording as ONE device-resident buffer (read in place, one pass of the chain). Under the emulated build of
    tests/test_emulated_gpu_suite.py "device" memory is host memory, so the numpy buffer itself plays that part."""
    if os.environ.get("AMB_TEST_EMULATED_LIB"):
        class _Dev:                                             # what blocks._as_iq needs from a CUDA tensor
            def __init__(self, a):
                self.a = np.ascontiguousarray(a, dtype=np.float32)
        return _Dev(iq)
    import torch
    return torch.from_numpy(np.ascontiguousarray(iq, dtype=np.float32)).cuda()


def run_cuda(iq, rate, thr, pmf, chunks=None, resolver=0, keep=False, one_pass=False, exact_dense=None):
    q = am.msg_queue()
    rx = am.rx_path(rate, thr, q, use_pmf=pmf)
    rx._ctx.call("amb_set_option", b"resolver", resolver)
    if exact_dense is not None:        # 0: the row-based exact kernel decides every call (dense-traffic regime)
        rx.set_option("exact_dense", exact_dense)
    frames = []
    if one_pass:
        d = device_resident(iq)
        if hasattr(d, "a"):
            import ctypes as C
            from gr_air_modes_b200 import _lib
            rx._ctx.call("amb_process", C.c_void_p(d.a.ctypes.data), d.a.size // 2, _lib.MEM_DEVICE, 1)
            rx.drain()
        else:
            rx.process(d, flush=True)
        frames += rx.frames
    elif chunks is None:
        rx.process(iq, flush=True)
        frames += rx.frames
    else:
        pos, n = 0, iq.size // 2
        for c in chunks:
            c = int(min(c, n - pos))
            last = pos + c >= n
            rx.process(iq[2 * pos: 2 * (pos + c)], flush=last)
            frames += rx.frames
            pos += c
            if last:
                break
    return q.strings(), frames, rx


@pytest.mark.parametrize("rate,n,nb,pmf,thr,seed", [
    (2e6, 600_000, 40, True, 7.0, 1), (4e6, 800_000, 50, True, 7.0, 2), (4e6, 800_000, 50, False, 7.0, 3),
    (10e6, 1_200_000, 40, True, 7.0, 4), (20e6, 2_000_000, 30, True, 7.0, 5), (4e6, 800_000, 50, True, 4.0, 6),
    (5e6, 600_000, 30, True, 7.0, 7), (3e6, 600_000, 30, True, 7.0, 8), (2.4e6, 600_000, 30, True, 6.0, 9),
    (6e6, 600_000, 30, True, 7.0, 10), (8e6, 800_000, 30, True, 7.0, 11), (16e6, 1_600_000, 20, True, 7.0, 12),
    (4e6, 600_000, 700, True, 6.0, 13), (10e6, 1_000_000, 30, False, 7.0, 14), (20e6, 1_600_000, 20, False, 8.0, 15),
    (7e6, 700_000, 30, True, 7.0, 16), (18e6, 1_500_000, 20, True, 7.0, 17),
])
def test_frames_bit_exact_vs_oracle(port, rate, n, nb, pmf, thr, seed):
    """Payload, CRC, timestamp, reference level: every queue message identical to the oracle's."""
    dense = nb > 100
    sc = synth.make_scene(rate, n, nb, seed, garble_frac=0.2 if dense else 0.0, fruit=80 if dense else 0)
    want = port.run_iq(sc.iq, rate, thr, pmf, co.MA_CANONICAL)
    msgs, frames, rx = run_cuda(sc.iq, rate, thr, pmf)
    assert len(want.index) > 0
    assert [f.sample_index for f in frames] == [int(x) for x in want.index]      # detected preamble offsets
    assert msgs == want.msgs
    for f, g in zip(frames, want.frames):
        assert bytes(f.data) == bytes(g.data) and f.crc == g.crc and f.nbits == g.nbits
        assert f.numlowconf == g.numlowconf and bytes(f.lowconfbits) == bytes(g.lowconfbits)
        assert f.passed == g.passed and f.ref_level == g.ref_level and f.secs == g.secs and f.frac == g.frac
    # both resolvers agree, and so do both kernels of the exact stage (row-based for dense traffic forced here)
    msgs1, _, _ = run_cuda(sc.iq, rate, thr, pmf, resolver=1)
    assert msgs1 == want.msgs
    msgs2, frames2, _ = run_cuda(sc.iq, rate, thr, pmf, exact_dense=0)
    assert msgs2 == want.msgs and [f.sample_index for f in frames2] == [int(x) for x in want.index]


def test_golden_fixtures_from_unmodified_reference():
    """tests/golden was produced by the reference's own preamble_impl/slicer_impl/modes_crc objects."""
    meta, scenes = load_golden()
    for s, iq in scenes:
        assert hashlib.sha256(iq.tobytes()).hexdigest() == s["iq_sha256"]
        msgs, frames, rx = run_cuda(iq, s["rate"], s["threshold_db"], s["use_pmf"])
        assert [f.sample_index for f in frames] == s["det_index"], s["name"]
        assert msgs == s["msgs"], s["name"]


def test_against_live_reference_if_present(port, ref):
    sc = synth.make_scene(4e6, 700_000, 60, 31)
    bb, avg = port.frontend(sc.iq, 4e6, True, co.MA_CANONICAL)
    r = ref.run_streams(bb, avg, 4e6, 7.0)
    msgs, frames, _ = run_cuda(sc.iq, 4e6, 7.0, True)
    assert msgs == r.msgs and [f.sample_index for f in frames] == [int(x) for x in r.index]


def test_streaming_equals_one_shot(port):
    """Ragged chunking (down to 1 sample) must not change a single frame: history, scan position and the
    'no room' rules carry across calls."""
    rng = np.random.default_rng(7)
    for rate, n in ((4e6, 600_000), (10e6, 900_000), (2e6, 400_000)):
        sc = synth.make_scene(rate, n, 40, int(rate / 1e6) + 40)
        want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL)
        for chunks in (list(rng.integers(1, 50_000, 2000)), [1, 2, 3, 255, 256, 257, 100_000] * 200, [n // 3] * 4):
            msgs, frames, _ = run_cuda(sc.iq, rate, 7.0, True, chunks=chunks)
            assert msgs == want.msgs
            assert [f.sample_index for f in frames] == [int(x) for x in want.index]


def test_end_of_stream_rules(port):
    """Bursts cut by the end of the stream: preamble_impl.cc:150 and :212-216."""
    rate = 4e6
    for cut in range(0, 700, 41):
        sc = synth.make_scene(rate, 60_000, 0, 11, starts=[20_000.3, 59_200.0 - cut], amplitude=0.3)
        want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL)
        for resolver in (0, 1):
            msgs, frames, _ = run_cuda(sc.iq, rate, 7.0, True, resolver=resolver)
            assert msgs == want.msgs and [f.sample_index for f in frames] == [int(x) for x in want.index]


def test_empty_tiny_and_silent_inputs(port):
    for n in (0, 1, 2, 5, 255, 256, 257, 1000):
        iq = np.zeros(2 * n, np.float32)
        msgs, frames, _ = run_cuda(iq, 4e6, 7.0, True)
        assert msgs == [] and frames == []
    iq = (np.random.default_rng(0).standard_normal(2 * 3000) * 0.01).astype(np.float32)
    want = port.run_iq(iq, 4e6, 7.0, True, co.MA_CANONICAL)
    msgs, _, _ = run_cuda(iq, 4e6, 7.0, True)
    assert msgs == want.msgs


def test_candidate_prefilter_is_a_superset_and_exact_stage_is_exact(port):
    """The streaming kernel may over-report candidates but never miss one; the exact stage's verdicts are
    the reference's first four tests (preamble_impl.cc:173-179)."""
    for rate, pmf in ((4e6, True), (2e6, True), (10e6, True), (4e6, False)):
        sc = synth.make_scene(rate, 500_000, 60, 77)
        bb, avg = port.frontend(sc.iq, rate, pmf, co.MA_CANONICAL)
        want = set(int(x) for x in first_four(bb, avg, rate, 7.0, port))
        q = am.msg_queue()
        rx = am.rx_path(rate, 7.0, q, use_pmf=pmf)
        rx.process(sc.iq, flush=True)
        idx = (C.c_uint64 * (1 << 20))(); info = (C.c_uint32 * (1 << 20))()
        n = rx._ctx.call("amb_debug_candidates", idx, info, 1 << 20)
        cand = {int(idx[k]) for k in range(n)}
        real = {int(idx[k]) for k in range(n) if info[k] & 0x100}
        limit = max(want) if want else 0
        assert {w for w in want if w < limit - 1000} <= cand
        assert {r for r in real if r < limit - 1000} == {w for w in want if w < limit - 1000}
        assert len(cand) <= 1.05 * len(real) + 8           # and it is tight


def test_long_gap_float_rounding_falls_back_to_sequential(port):
    """> 2^24 samples between packets: :237 adds 240*spc in float; the parallel resolver must notice."""
    rate = 10e6
    sc = synth.make_scene(rate, (1 << 25) + 5_000_001, 0, 3,
                          starts=[1_000_000.4, 1_000_000.4 + (1 << 24) + 4_000_001, 33_000_000.2], amplitude=0.3)
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_SLIDING64)
    msgs, frames, rx = run_cuda(sc.iq, rate, 7.0, True, one_pass=True)     # one device-resident pass over the whole gap
    assert [f.sample_index for f in frames] == [int(x) for x in want.index] and len(frames) == 3
    assert [m.split()[:2] for m in msgs] == [m.split()[:2] for m in want.msgs]
    assert rx.stats().resolver_fallback == 1
    # host memory goes through the ingest ring in 2^22-sample chunks: the packet behind the gap is then the first
    # cluster of its chunk, whose entry state is known exactly - same frames, no fallback needed
    msgs, frames, rx = run_cuda(sc.iq, rate, 7.0, True)
    assert [f.sample_index for f in frames] == [int(x) for x in want.index] and len(frames) == 3
    assert [m.split()[:2] for m in msgs] == [m.split()[:2] for m in want.msgs]


def test_device_crc_and_slicer_block(port):
    rng = np.random.default_rng(9)
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    for length in (4, 11):
        data = rng.integers(0, 256, (500, length), dtype=np.uint8)
        out = (C.c_uint32 * 500)()
        rx._ctx.call("amb_device_crc", data.tobytes(), 500, length, out)
        assert [out[k] for k in range(500)] == [port.crc24(data[k].tobytes()) for k in range(500)]
    chips = rng.normal(0.0, 0.3, (400, 240)).astype(np.float32)
    chips[:, [0, 2, 7, 9]] += 1.0
    chips[::3, 16:240:2] += 1.0
    secs = np.arange(400, dtype=np.uint64); frac = rng.random(400)
    want = port.run_slicer(chips, secs, frac)
    q2 = am.msg_queue()
    s = am.slicer(q2)
    s.process(chips, list(zip(secs, frac)))
    assert q2.strings() == want.msgs and len(want.msgs) > 10


def test_setters_and_errors():
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    assert rx.get_threshold() == 7.0 and rx.get_pmf() is True
    rx.set_threshold(5.5)
    assert rx.get_threshold() == 5.5
    rx.set_rate(10e6)
    with pytest.raises(RuntimeError):
        rx.set_rate(1e6)                         # int(spc) == 0 crashes the reference (% 0); we refuse
    rx.process(np.zeros(2000, np.float32), flush=True)
    with pytest.raises(RuntimeError):
        rx.process(np.zeros(2000, np.float32))  # flushed stream needs reset()
    rx.reset()
    rx.process(np.zeros(2000, np.float32))


def test_threshold_change_takes_effect(port):
    sc = synth.make_scene(4e6, 400_000, 40, 91)
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    for thr in (7.0, 3.0, 10.0):
        rx.reset(); q.flush(); rx.set_threshold(thr)
        rx._slicer._first = True
        rx.process(sc.iq, flush=True)
        assert q.strings() == port.run_iq(sc.iq, 4e6, thr, True, co.MA_CANONICAL).msgs


def test_full_size_properties():
    """BASELINE size (2^28 samples at 4 Msps) through size-independent properties: idempotence, payloads
    invariant under a power-of-two gain with levels scaling by its square, and every strong burst decoded."""
    import torch
    n = 1 << 28
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    iq = torch.randn(2 * n, device="cuda", generator=g) * 0.01
    rng = np.random.Generator(np.random.PCG64(5))
    sent = []
    for s in np.sort(rng.uniform(1000, n - 2000, 300)):
        frame = synth.make_frame((11, 17)[int(rng.integers(0, 2))], rng)
        n0, w = synth.burst_waveform(synth.Burst(float(s), frame, 0.2, float(rng.uniform(0, 6.28))), 2.0)
        iq[2 * n0: 2 * n0 + 2 * w.size] += torch.from_numpy(np.ascontiguousarray(w).view(np.float32)).cuda()
        sent.append(frame.hex())
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    rx.process(iq, flush=True)
    a = q.strings(); q.flush()
    rx.reset(); rx._slicer._first = True
    rx.process(iq, flush=True)
    b = q.strings(); q.flush()
    assert a == b and len(a) >= 300
    decoded = set(sent) & {m.split()[0] for m in a}
    assert len(decoded) >= 0.97 * len(sent)      # a noise false alarm within 120 us before a burst blanks it (reference dead time)
    assert all(int(m.split()[1], 16) == 0 for m in a if m.split()[0] in decoded)
    iq *= 4.0
    rx.reset(); rx._slicer._first = True
    rx.process(iq, flush=True)
    c = q.strings()
    assert [m.split()[:2] for m in c] == [m.split()[:2] for m in a]
    assert [m.split()[3:] for m in c] == [m.split()[3:] for m in a]
    for x, y in zip(a, c):
        assert abs(parse_msg(y)[2] / parse_msg(x)[2] - 16.0) < 1e-5


def test_split_form_preamble_and_slicer_blocks(port):
    """The two reference blocks used separately: preamble(in0, in1) -> 240-chip packets + tags -> slicer."""
    for rate, pmf in ((4e6, True), (10e6, True), (2e6, False), (5e6, True)):
        sc = synth.make_scene(rate, 500_000, 40, 55)
        bb, avg = port.frontend(sc.iq, rate, pmf, co.MA_CANONICAL)
        want = port.run_streams(bb, avg, rate, 7.0)
        pre = am.preamble(rate, 7.0)
        assert pre.get_rate() == float(int(rate)) and pre.get_threshold() == 7.0
        chips, tags = pre.process(bb, avg)
        assert [t[0] for t in tags] == [int(x) for x in want.index]
        assert np.array_equal(chips, want.chips)                       # bit-exact soft symbols
        assert [(t[1], t[2]) for t in tags] == list(zip([int(x) for x in want.secs], [float(x) for x in want.frac]))
        q = am.msg_queue()
        am.slicer(q).process(chips, [(t[1], t[2]) for t in tags])
        assert q.strings() == want.msgs


def test_dense_traffic_threshold_sweep_matches_reference(port):
    """BASELINE configs[4]: ~10 k overlapping squitters/s with garbled CRCs and Mode A/C-like FRUIT; detection
    sets and messages (hence P_d / P_fa at every threshold) must equal the reference's."""
    rate, n = 4e6, 2_000_000
    sc = synth.make_scene(rate, n, 5000, 99, garble_frac=0.2, fruit=2000, snr_db=(4.0, 30.0))
    sent = {b.frame.hex() for b in sc.bursts}
    roc = []
    for thr in (3.0, 5.0, 7.0, 9.0, 12.0):
        want = port.run_iq(sc.iq, rate, thr, True, co.MA_CANONICAL)
        msgs, frames, rx = run_cuda(sc.iq, rate, thr, True)
        assert [f.sample_index for f in frames] == [int(x) for x in want.index]
        assert msgs == want.msgs
        got = {m.split()[0] for m in msgs}
        roc.append((thr, len(frames), len(got & sent), len(got - sent)))
    assert roc[0][1] > roc[-1][1]                                       # fewer detections at higher thresholds
    # streaming over the same dense scene
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL)
    msgs, _, _ = run_cuda(sc.iq, rate, 7.0, True, chunks=[123_457] * 40)
    assert msgs == want.msgs
    msgs, _, _ = run_cuda(sc.iq, rate, 7.0, True, chunks=[123_457] * 40, exact_dense=0)
    assert msgs == want.msgs


def test_device_side_drain_equals_host_poll(port):
    """amb_drain_device (rx_path.drain_device): the frames of several calls, put into stream order and stamped ON THE
    DEVICE, are byte for byte the records amb_poll_frames copies to the host - on dense traffic (1.7 k frames over
    tiles of 256: the ordering network needs its global stages; tools/prof_chain.py checks 2.4 x 10^5 frames with the
    default tile) and on a sparse 10 Msps scene, with a start time and a later rx_time
    tag in force."""
    import torch
    cases = [(4e6, 2_000_000, 5000, 99, dict(garble_frac=0.2, fruit=2000, snr_db=(4.0, 30.0))), (10e6, 1_200_000, 40, 4, {})]
    for rate, n, nb, seed, kw in cases:
        sc = synth.make_scene(rate, n, nb, seed, **kw)
        cuts = [0, 300_000, 300_000 + 123_456, n]

        def ctx():
            rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
            rx.set_start_time(77, 0.5)
            rx.add_time_tag(n // 2, 9000, 0.25)
            if nb == 5000:
                rx.set_option("order_tile", 256)      # 1.7 k frames: several tiles, so the network's global stages run too
            return rx

        rx = ctx()
        for a, b in zip(cuts[:-1], cuts[1:]):
            rx.process(sc.iq[2 * a: 2 * b], flush=(b == n), collect=False)
        buf, got = rx._ctx.poll_array()
        want = bytes(buf)[:got * 80]
        idx = [int(buf[k].sample_index) for k in range(got)]
        assert idx == [int(x) for x in port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL).index]
        rx.close()
        if nb == 5000:
            assert got > 1024

        rx = ctx()
        dev = torch.from_numpy(sc.iq).cuda()
        for a, b in zip(cuts[:-1], cuts[1:]):
            rx.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
        fr = rx.drain_device()
        assert fr.is_cuda and fr.numel() == got * 80
        assert fr.cpu().numpy().tobytes() == want
        assert rx.drain_device().numel() == 0
        rx.close()


def test_overlap_off_is_identical(port):
    sc = synth.make_scene(4e6, 700_000, 50, 17)
    want = port.run_iq(sc.iq, 4e6, 7.0, True, co.MA_CANONICAL).msgs
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    rx._ctx.call("amb_set_option", b"overlap", 0)
    for k in range(0, 700_000, 100_000):
        rx.process(sc.iq[2 * k: 2 * (k + 100_000)], flush=(k + 100_000 >= 700_000), collect=False)
    rx.drain()
    assert q.strings() == want


def test_config0_pr1_golden_single_df17(port, tmp_path):
    """BASELINE configs[0]: 10 s at 2 Msps, one injected DF17 8D4840D6202CC371C32CE0576098, noise sigma 0.01.
    (A) fed to rx_path at 2 Msps directly, (B) the same scene rendered at 4 Msps (what modes_rx runs after its
    2->4 Msps resampler). The oracle's message list is the golden; the CLI tool must print the same lines."""
    import subprocess, sys, os
    frame = bytes.fromhex("8D4840D6202CC371C32CE0576098")
    for rate, n in ((2e6, 20_000_000), (4e6, 40_000_000)):
        rng = np.random.Generator(np.random.PCG64(1))
        iq = (rng.standard_normal(2 * n, dtype=np.float32) * np.float32(0.01))
        n0, w = synth.burst_waveform(synth.Burst(n / 2 + 0.37, frame, 0.5, 1.0), rate / 2e6)
        iq[2 * n0: 2 * (n0 + w.size)] += w.view(np.float32)
        want = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL)
        assert any(m.startswith(frame.hex() + " 000000") for m in want.msgs)
        msgs, frames, _ = run_cuda(iq, rate, 7.0, True)
        assert msgs == want.msgs and [f.sample_index for f in frames] == [int(x) for x in want.index]
        if rate == 2e6:
            path = tmp_path / "pr1.cfile"
            iq.tofile(path)
            root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
            out = subprocess.run([sys.executable, os.path.join(root, "tools", "modes_rx_b200.py"), "-s", str(path), "-r", "2e6",
                                  "--chunk", "3000001"], capture_output=True, text=True, check=True).stdout.split("\n")
            assert [ln for ln in out if ln] == want.msgs


def test_rx_time_start_tag(port):
    sc = synth.make_scene(4e6, 400_000, 30, 3)
    for st in ((1234567, 0.25), (7, 0.9999999)):
        port.set_start_time(*st)
        try:
            want = port.run_iq(sc.iq, 4e6, 7.0, True, co.MA_CANONICAL)
        finally:
            port.set_start_time(0, 0.0)
        q = am.msg_queue()
        rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
        rx.set_start_time(*st)
        rx.process(sc.iq, flush=True)
        assert q.strings() == want.msgs


def test_dc_blocker_option(port):
    """rx_path(..., use_dcblock=True): filter.dc_blocker_cc(100*spc, False) in front of the demodulator
    (rx_path.py:39-41). GNU Radio code - restated, parity unpinned - but CUDA and the CPU restatement agree bit
    for bit, one-shot and streamed, and a DC offset that swamps detection without it is removed with it."""
    for rate, n in ((4e6, 400_000), (2e6, 300_000), (10e6, 600_000)):
        sc = synth.make_scene(rate, n, 30, 61)
        iq = sc.iq.copy(); iq[0::2] += np.float32(0.05); iq[1::2] -= np.float32(0.03)
        want = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL, use_dcblock=True)
        for chunks in (None, [77_777] * 20):
            q = am.msg_queue()
            rx = am.rx_path(rate, 7.0, q, use_pmf=True, use_dcblock=True)
            frames = []
            if chunks is None:
                rx.process(iq, flush=True); frames = rx.frames
            else:
                pos = 0
                for c in chunks:
                    c = min(c, n - pos); last = pos + c >= n
                    rx.process(iq[2 * pos: 2 * (pos + c)], flush=last); frames += rx.frames
                    pos += c
                    if last: break
            assert [f.sample_index for f in frames] == [int(x) for x in want.index]
            assert q.strings() == want.msgs
        without = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL).index
        clean = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL).index
        assert len(want.index) > 0 and len(without) <= len(clean)


def test_two_contexts_with_different_rates_coexist(port):
    """Contexts are independent: interleaving calls at 4 and 10 Msps on one device changes nothing."""
    a = synth.make_scene(4e6, 400_000, 30, 71)
    b = synth.make_scene(10e6, 600_000, 30, 72)
    wa = port.run_iq(a.iq, 4e6, 7.0, True, co.MA_CANONICAL).msgs
    wb = port.run_iq(b.iq, 10e6, 7.0, True, co.MA_CANONICAL).msgs
    qa, qb = am.msg_queue(), am.msg_queue()
    ra = am.rx_path(4e6, 7.0, qa, use_pmf=True)
    rb = am.rx_path(10e6, 7.0, qb, use_pmf=True)
    for k in range(4):
        ra.process(a.iq[2 * k * 100_000: 2 * (k + 1) * 100_000], flush=(k == 3), collect=False)
        rb.process(b.iq[2 * k * 150_000: 2 * (k + 1) * 150_000], flush=(k == 3), collect=False)
    ra.drain(); rb.drain()
    assert qa.strings() == wa and qb.strings() == wb


def test_randomised_stress_including_pathological_inputs():
    """tests/tools/stress_parity.py: random rates / thresholds / PMF / chunkings / resolvers plus inputs scaled to the
    denormal range or near overflow, stretches of exact zeros, NaN / Inf samples, DC offsets, dense bursts."""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tests", "tools", "stress_parity.py"), "3", "40"],
                         capture_output=True, text=True, timeout=900).stdout
    assert "40 cases, 0 mismatches" in out, out[-2000:]


def test_c_abi_example_program(port, tmp_path):
    """examples/modes_rx_c.c (C only, no Python in the loop) prints the oracle's message list."""
    import subprocess
    from gr_air_modes_b200 import build
    exe = build.build_c_example()
    sc = synth.make_scene(4e6, 600_000, 40, 81)
    path = tmp_path / "c.cfile"
    sc.iq.tofile(path)
    want = port.run_iq(sc.iq, 4e6, 7.0, True, co.MA_CANONICAL).msgs
    out = subprocess.run([exe, str(path), "4e6", "7.0", "100003"], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [ln for ln in out if ln] == want


def test_split_form_preamble_streaming(port):
    """preamble.process(in0, in1, flush=False) in ragged chunks: same packets and tags as one call."""
    rng = np.random.default_rng(3)
    for rate in (4e6, 10e6, 2e6):
        sc = synth.make_scene(rate, 400_000, 40, 56)
        bb, avg = port.frontend(sc.iq, rate, True, co.MA_CANONICAL)
        want = port.run_streams(bb, avg, rate, 7.0)
        pre = am.preamble(rate, 7.0)
        chips, tags, pos, n = [], [], 0, bb.size
        for c in list(rng.integers(1, 60_000, 60)) + [n]:
            c = int(min(c, n - pos)); last = pos + c >= n
            ch, tg = pre.process(bb[pos:pos + c], avg[pos:pos + c], flush=last)
            chips.append(ch); tags += tg; pos += c
            if last: break
        assert [t[0] for t in tags] == [int(x) for x in want.index]
        assert np.array_equal(np.concatenate(chips), want.chips)
        # the block starts a new stream after a flush
        ch, tg = pre.process(bb, avg)
        assert [t[0] for t in tg] == [int(x) for x in want.index]


# ---- one stream time-sharded over several contexts (SURVEY.md 8e secondary mode; amb_seek / amb_resolve) --------
def run_time_sharded(iq, rate, thr, pmf, spans=None, boundaries=None, resolver=0):
    """All spans on cuda:0, one rx_path each: dense stages of every span first, then the state chain."""
    from gr_air_modes_b200 import shard
    n = iq.size // 2
    plan = shard.time_shard_plan(n, spans or (len(boundaries) + 1), am.query_geometry(rate, thr, pmf), boundaries=boundaries)
    q = am.msg_queue()
    rxs = [am.rx_path(rate, thr, q, use_pmf=pmf) for _ in plan]
    for rx, sp in zip(rxs, plan):                       # what the ranks do concurrently
        rx._ctx.call("amb_set_option", b"resolver", resolver)
        rx.defer_resolve(True)
        rx.seek(sp.first_sample, sp.first_decision)
        rx.process(iq[2 * sp.first_sample: 2 * sp.end], flush=sp.flush, collect=False)
    frames, state, queued = [], (0, 0), 0
    for rx, sp in zip(rxs, plan):                       # the chain
        rx.resolve(state)
        if not sp.flush:
            state = rx.walk_state()
        rx._slicer._first = queued == 0
        queued += rx.drain()
        frames += rx.frames
    for rx in rxs:
        rx.close()
    return q.strings(), frames, plan


@pytest.mark.parametrize("rate,n,nb,pmf", [(4e6, 1_500_000, 120, True), (2e6, 900_000, 80, True),
                                           (10e6, 2_500_000, 80, True), (20e6, 4_000_000, 60, False)])
def test_time_sharded_equals_one_shot(port, rate, n, nb, pmf):
    sc = synth.make_scene(rate, n, nb, int(rate / 1e6) + 70)
    want = port.run_iq(sc.iq, rate, 7.0, pmf, co.MA_CANONICAL)
    assert len(want.msgs) > 10
    for spans in (2, 3, 8):
        for resolver in (0, 1):
            msgs, frames, plan = run_time_sharded(sc.iq, rate, 7.0, pmf, spans=spans, resolver=resolver)
            assert len(plan) == spans
            assert [f.sample_index for f in frames] == [int(x) for x in want.index]
            assert msgs == want.msgs
            for f, g in zip(frames, want.frames):
                assert bytes(f.data) == bytes(g.data) and f.ref_level == g.ref_level and f.secs == g.secs and f.frac == g.frac


def test_time_shard_cut_inside_packets_and_dense_traffic(port):
    """Cuts placed on, just before and just after accepted preambles (the previous span's packet skip then
    reaches into the next span: the handed-over `p` matters), and cuts through one long cluster of a dense scene."""
    rate = 4e6
    sc = synth.make_scene(rate, 1_200_000, 150, 404)
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL)
    idx = [int(x) for x in want.index if 300_000 < int(x) < 1_100_000]
    rng = np.random.default_rng(5)
    for trial in range(6):
        picks = sorted(rng.choice(len(idx), 3, replace=False))
        cuts = [idx[picks[0]] + int(rng.integers(-3, 4)), idx[picks[1]] + int(rng.integers(1, 480)), idx[picks[2]] + 481]
        msgs, frames, _ = run_time_sharded(sc.iq, rate, 7.0, True, boundaries=cuts, resolver=trial & 1)
        assert [f.sample_index for f in frames] == [int(x) for x in want.index], cuts
        assert msgs == want.msgs
    dense = synth.make_scene(rate, 2_000_000, 5000, 99, garble_frac=0.2, fruit=2000, snr_db=(4.0, 30.0))
    want = port.run_iq(dense.iq, rate, 5.0, True, co.MA_CANONICAL)
    for spans in (2, 5):
        msgs, frames, _ = run_time_sharded(dense.iq, rate, 5.0, True, spans=spans)
        assert [f.sample_index for f in frames] == [int(x) for x in want.index]
        assert msgs == want.msgs


def test_time_shard_api_errors():
    q = am.msg_queue()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    g = am.query_geometry(4e6, 7.0, True)
    assert g.shard_back == g.history - 1 + g.floor_len + g.pmf_len and g.shard_fwd > g.packet_skip - g.history
    with pytest.raises(RuntimeError):
        rx.seek(4096, 4096 + g.shard_back - 1)            # halo too short
    with pytest.raises(RuntimeError):
        rx.resolve((0, 0))                                  # nothing deferred
    rx.defer_resolve(True)
    rx.seek(0, 0)
    iq = synth.make_scene(4e6, 100_000, 5, 3).iq
    rx.process(iq, flush=False, collect=False)
    with pytest.raises(RuntimeError):
        rx.process(iq, flush=False, collect=False)          # one call per span in deferred mode
    with pytest.raises(RuntimeError):
        rx.walk_state()
    rx.resolve((0, 0))
    pos, p = rx.walk_state()
    assert p >= 100_000 + g.history - 1 - (g.shard_fwd + g.history - 1)
    rx.defer_resolve(False)
    rx.reset()
    assert rx.process(iq, flush=True) >= 5                  # normal operation afterwards
    rx.close()


@pytest.mark.parametrize("rate,pmf", [(2e6, True), (4e6, True), (4e6, False), (10e6, True), (20e6, True), (5e6, True)])
def test_front_end_streams_bit_exact_at_every_sample(port, rate, pmf):
    """SURVEY 8c pin (iii): m2, the preamble block's in0 (bb) and in1 (avg) at EVERY sample, not only at candidates,
    equal the oracle's canonical front end bit for bit - including the zero history at the stream start, strong
    bursts inside the floor window and denormal-range noise."""
    n = 200_000
    sc = synth.make_scene(rate, n, 25, int(rate / 1e6) + 300)
    iq = sc.iq.copy()
    iq[2 * 150_000: 2 * 150_400] *= np.float32(1e-18)         # m2 in the denormal range
    iq[2 * 160_000: 2 * 160_100] = 0.0
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=pmf)
    bb, avg = port.frontend(iq, rate, pmf, co.MA_CANONICAL)
    assert np.array_equal(rx.dump_stage("m2", iq).view(np.uint32), port.mag2(iq).view(np.uint32))
    assert np.array_equal(rx.dump_stage("bb", iq).view(np.uint32), bb.view(np.uint32))
    assert np.array_equal(rx.dump_stage("avg", iq).view(np.uint32), avg.view(np.uint32))
    rx.close()


def test_cli_udp_source_zmq_feed_and_dcblock(port, tmp_path):
    """Row f1: tools/modes_rx_b200.py with the reference's other offline source (UDP datagrams of gr_complex,
    radio.py:221-228), the -t ZMQ dl_data feed (radio.py:79-87) and -d; the lines are the oracle's."""
    import os, socket, subprocess, sys, threading, time
    zmq = pytest.importorskip("zmq")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = os.path.join(root, "tools", "modes_rx_b200.py")
    sc = synth.make_scene(4e6, 300_000, 25, 808)
    want = port.run_iq(sc.iq, 4e6, 7.0, True, co.MA_CANONICAL).msgs
    assert len(want) > 5

    def free_port(kind):
        s = socket.socket(socket.AF_INET, kind); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p

    uport, zport = free_port(socket.SOCK_DGRAM), free_port(socket.SOCK_STREAM)
    proc = subprocess.Popen([sys.executable, cli, "-s", "127.0.0.1:%d" % uport, "-r", "4e6", "-t", str(zport),
                             "--udp-idle", "1.5", "--chunk", "70001"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    ctx = zmq.Context()
    sub = ctx.socket(zmq.SUB); sub.connect("tcp://127.0.0.1:%d" % zport); sub.setsockopt(zmq.SUBSCRIBE, b"dl_data")
    got = []

    def listen():
        sub.RCVTIMEO = 15000
        try:
            while len(got) < len(want):
                key, val = sub.recv_multipart()
                assert key == b"dl_data"
                got.append(val.decode())
        except zmq.Again:
            pass

    th = threading.Thread(target=listen); th.start()
    # wait until the receiver has bound its sockets (it prints "Rate is" after constructing rx_path)
    deadline = time.time() + 120
    rcvbuf = 0
    while time.time() < deadline:
        line = proc.stderr.readline()
        if line.startswith("UDP receive buffer"):
            rcvbuf = int(line.split()[3])
        if line.startswith("Rate is") or not line:
            break
    time.sleep(0.5)
    tx = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    raw = sc.iq.tobytes()
    # Loss is made impossible rather than tolerated: if the receiver's socket buffer (Linux reports twice the usable
    # size, and skb overhead roughly doubles a 1.4 kB datagram's footprint) holds the whole recording, send at full
    # speed; otherwise pace the sender far below what the receive loop sustains (2 MB/s against > 500 MB/s).
    fits = rcvbuf // 4 >= len(raw)
    step = 1472 // 8 * 8                                              # 184 complex items per datagram
    t0 = time.time()
    for a in range(0, len(raw), step):
        tx.sendto(raw[a: a + step], ("127.0.0.1", uport))
        if not fits:
            while (a + step) / 2e6 > time.time() - t0:
                time.sleep(0.001)
    out, err = proc.communicate(timeout=180)
    th.join()
    assert proc.returncode == 0, err
    lines = [ln for ln in out.split("\n") if ln]
    assert lines == want
    assert got == want
    # -d on a cfile
    iq = sc.iq.copy(); iq[0::2] += np.float32(0.05)
    path = tmp_path / "dc.cfile"; iq.tofile(path)
    wantd = port.run_iq(iq, 4e6, 7.0, True, co.MA_CANONICAL, use_dcblock=True).msgs
    out = subprocess.run([sys.executable, cli, "-s", str(path), "-r", "4e6", "-d"], capture_output=True, text=True, check=True).stdout
    assert [ln for ln in out.split("\n") if ln] == wantd
    # -n prints nothing
    out = subprocess.run([sys.executable, cli, "-s", str(path), "-n"], capture_output=True, text=True, check=True).stdout
    assert out.strip() == ""


def run_time_sharded_speculative(iq, rate, thr, pmf, spans=None, boundaries=None):
    """One thread per span, each with its own rx_path on cuda:0, running shard.process_time_sharded_speculative with
    an in-process all-gather and mailboxes for the fallback chain. Returns (messages, frames, first_bad)."""
    import queue, threading
    from gr_air_modes_b200 import shard
    n = iq.size // 2
    plan = shard.time_shard_plan(n, spans or (len(boundaries) + 1), am.query_geometry(rate, thr, pmf), boundaries=boundaries)
    world = len(plan)
    table, bar = [None] * world, threading.Barrier(world)
    boxes = [queue.Queue() for _ in range(world)]
    qs = [am.msg_queue() for _ in range(world)]
    out, errs, bad = [None] * world, [], [None]

    def work(rank):
        try:
            rx = am.rx_path(rate, thr, qs[rank], use_pmf=pmf)

            def all_gather(vals):
                table[rank] = list(vals)
                bar.wait(60)
                res = [list(r) for r in table]
                bar.wait(60)
                if rank == 0:
                    bad[0] = shard.compose_entries(plan, res)[2]
                return res

            sp = plan[rank]
            shard.process_time_sharded_speculative(rx, iq[2 * sp.first_sample: 2 * sp.end], plan, rank, all_gather,
                                                   lambda: boxes[rank].get(timeout=60), lambda st: boxes[rank + 1].put(st))
            out[rank] = list(rx.frames)
            rx.close()
        except Exception as e:                       # noqa: BLE001 - reported by the caller
            errs.append((rank, repr(e)))
            bar.abort()

    ths = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert not errs, errs
    return [m for q in qs for m in q.strings()], [f for fr in out for f in fr], bad[0], world


def test_time_sharded_speculative_resolution(port):
    """The chain-free variant: speculative resolution + one all-gather; spans whose speculation cannot be proven fall
    back to the chain. Both outcomes must give the one-shot result."""
    rate = 4e6
    sc = synth.make_scene(rate, 1_500_000, 120, 74)
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_CANONICAL)
    for spans in (2, 3, 8):
        msgs, frames, bad, world = run_time_sharded_speculative(sc.iq, rate, 7.0, True, spans=spans)
        assert bad == world - 1                                           # every speculation held
        assert [f.sample_index for f in frames] == [int(x) for x in want.index] and msgs == want.msgs
    # cuts just after accepted preambles: the previous packet's skip covers real candidates of the next span
    idx = [int(x) for x in want.index if 300_000 < int(x) < 1_200_000]
    rng = np.random.default_rng(11)
    fell_back = 0
    for trial in range(8):
        picks = sorted(rng.choice(len(idx), 3, replace=False))
        cuts = [idx[k] + int(rng.integers(1, 12)) for k in picks]
        msgs, frames, bad, world = run_time_sharded_speculative(sc.iq, rate, 7.0, True, boundaries=cuts)
        fell_back += bad < world - 1
        assert [f.sample_index for f in frames] == [int(x) for x in want.index], cuts
        assert msgs == want.msgs
    assert fell_back > 0                                                  # the fallback chain was exercised
    dense = synth.make_scene(rate, 2_000_000, 5000, 99, garble_frac=0.2, fruit=2000, snr_db=(4.0, 30.0))
    want = port.run_iq(dense.iq, rate, 5.0, True, co.MA_CANONICAL)
    for spans in (2, 6):
        msgs, frames, bad, world = run_time_sharded_speculative(dense.iq, rate, 5.0, True, spans=spans)
        assert [f.sample_index for f in frames] == [int(x) for x in want.index] and msgs == want.msgs


def test_dc_blocker_output_bit_exact_both_paths(port):
    """The DC blocker kernel takes an O(1) prefix-sum path on tiles whose exponent spread proves every fp64 sum exact
    and the literal ascending sum elsewhere; its complex output equals the CPU restatement bit for bit on inputs that
    force both: plain noise, strong bursts next to near-zero samples, zeros, denormals, huge dynamic range, Inf/NaN."""
    rng = np.random.default_rng(3)
    for rate in (2e6, 4e6, 10e6, 20e6):
        n = 120_000
        sc = synth.make_scene(rate, n, 20, int(rate / 1e6) + 500, snr_db=(10.0, 45.0))
        iq = sc.iq.copy()
        iq[0::2] += np.float32(0.03)
        iq[2 * 20_000: 2 * 23_000] = 0.0                                      # silence
        iq[2 * 30_000: 2 * 33_000] *= np.float32(1e-38)                       # denormals
        iq[2 * 40_000: 2 * 40_002] = np.float32(1e-30)                        # tiny samples inside ordinary noise
        iq[2 * 50_000: 2 * 53_000: 7] *= np.float32(1e12)                     # 40 binades of spread
        iq[2 * 60_000] = np.inf; iq[2 * 61_000 + 1] = np.nan; iq[2 * 62_000] = -np.inf
        iq[2 * 70_000: 2 * 74_000] = rng.integers(-3, 4, 8000).astype(np.float32)   # small integers: exact with cancellation
        q = am.msg_queue()
        rx = am.rx_path(rate, 7.0, q, use_pmf=True, use_dcblock=True)
        got = rx.dump_stage("dc", iq)
        want = port.dc_blocker(iq, 100 * int(rate / 2e6), co.MA_CANONICAL)
        nan = np.isnan(want)                                                  # NaN payloads differ between x86 and the GPU
        assert nan.any() and np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]), rate
        rx.close()


# ---- host ingest pipeline on the device (chunk ring, copy stream, 16-bit IQ, non-blocking poll) -----------------------
def test_host_ingest_paths_pinned_pageable_small_calls(port):
    """The same recording as pinned host memory (DMA'd from where it lies, chunk by chunk), as pageable memory
    (gathered into the library's pinned ring by its copy threads) and as GNU Radio-sized calls with the non-blocking
    poll: identical messages = the oracle's. Chunks far smaller than the recording force many ring wrap-arounds with
    the H2D copy of one chunk running under the kernels of the previous one."""
    import torch
    rate = 4e6
    sc = synth.make_scene(rate, 3_000_000, 300, 1201)
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_SLIDING64)
    assert len(want.msgs) > 200
    pinned = torch.from_numpy(sc.iq).pin_memory()
    for chunk in (1 << 16, 1 << 22):
        for src in (pinned, sc.iq):
            q = am.msg_queue()
            rx = am.rx_path(rate, 7.0, q, use_pmf=True)
            rx.set_option("ingest_chunk", chunk)
            rx.process(src, flush=True)
            assert q.strings() == want.msgs, (chunk, type(src))
            assert [f.sample_index for f in rx.frames] == [int(x) for x in want.index]
            rx.close()
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    early, n = 0, sc.iq.size // 2
    for a in range(0, n, 32768):                                 # what a GNU Radio sink's work() hands over
        rx.process(sc.iq[2 * a: 2 * min(a + 32768, n)], collect=False)
        early += rx.poll_ready()
    rx.process(sc.iq[:0], flush=True)
    assert q.strings() == want.msgs and early > 0
    rx.close()


def test_sc16_input_equals_its_float32_widening_on_the_device(port):
    """AMB_MEM_HOST_SC16 / AMB_MEM_DEVICE_SC16: 16-bit IQ widened on the device with x * 2^-15 gives the very messages
    of feeding the float32 array a host-side conversion would have produced (radio.py:163-173, cpu_format fc32)."""
    import torch
    rate = 4e6
    sc = synth.make_scene(rate, 2_000_000, 200, 1202)
    i16 = np.clip(np.rint(sc.iq * 32768.0), -32768, 32767).astype(np.int16)
    f32 = i16.astype(np.float32) * np.float32(1.0 / 32768.0)
    want = port.run_iq(f32, rate, 7.0, True, co.MA_SLIDING64)
    assert len(want.msgs) > 100
    ref_msgs, _, _ = run_cuda(f32, rate, 7.0, True)
    assert ref_msgs == want.msgs
    for src in (i16, torch.from_numpy(i16).pin_memory(), torch.from_numpy(i16).cuda()):
        q = am.msg_queue()
        rx = am.rx_path(rate, 7.0, q, use_pmf=True)
        rx.set_option("ingest_chunk", 1 << 18)
        rx.process(src[: 2 * 777_777], collect=False)
        rx.process(src[2 * 777_777:], flush=True)
        assert q.strings() == want.msgs, type(src)
        rx.close()


def test_torch_input_is_ordered_after_its_producer(port):
    """A CUDA tensor written asynchronously on torch's stream just before process(): the context's streams wait for
    that stream (amb_wait_stream), and the tensor is kept alive until drain()."""
    import torch
    rate = 4e6
    sc = synth.make_scene(rate, 1_500_000, 120, 1203)
    want = port.run_iq(sc.iq, rate, 7.0, True, co.MA_SLIDING64).msgs
    host = torch.from_numpy(sc.iq).pin_memory()
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    for _ in range(3):
        q.flush(); rx.reset(); rx._slicer._first = True
        junk = torch.randn(1 << 26, device="cuda")             # keeps torch's stream busy in front of the copy
        junk = junk * 2 + 1
        dev = torch.empty(host.numel(), device="cuda")
        dev.copy_(host, non_blocking=True)                      # still in flight when process() is called
        rx.process(dev, flush=True, collect=False)
        del dev, junk                                           # the block must not go back to the allocator yet
        torch.empty(host.numel(), device="cuda").fill_(7.0)     # would overwrite it if it did
        rx.drain()
        assert q.strings() == want
