"""Mode A/C replies (option "modeac") through the library's own sources under the SIMT emulator (tests/simt/library_emul.cc):
the tile and emit kernels, the chain's launch sequence and the C ABI, record for record against tests/modeac_oracle.py,
peak and floor bit for bit, under cuts into calls, with the DC blocker, from float32 and int16 IQ; Mode S frames
unchanged by the option; launch counts; the C ABI's error returns."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import _lib, synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import modeac_oracle as mo  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def launches(tmp_path_factory):
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        lib = C.CDLL(out)
        lib.simt_launch_count.restype = C.c_ulonglong
        yield lib.simt_launch_count
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def scene(rate, n, n_replies, seed, n_bursts=2):
    return synth.make_modeac_scene(rate, n, n_replies, seed, n_bursts=n_bursts)[0]


def run(iq, rate, chunks=(), modeac=True, dcblock=False, sc16=False):
    """(replies, frames, stats) of the stream iq cut after the sample counts in chunks, flushed at the end."""
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, use_dcblock=dcblock, modeac=modeac)
    n = iq.size // 2
    data = np.clip(np.rint(iq * 32768.0), -32768, 32767).astype(np.int16) if sc16 else iq
    frames, pos = [], 0
    for c in list(chunks) + [n]:
        c = int(min(c, n - pos))
        last = pos + c >= n
        rx.process(data[2 * pos: 2 * (pos + c)], flush=last)
        frames += [bytes(f) for f in rx.frames]
        pos += c
        if last:
            break
    reps = rx.modeac() if modeac else None
    st = rx.modeac_stats() if modeac else None
    rx.close()
    return reps, frames, st


@pytest.mark.parametrize("rate,n,nr", [(4e6, 40_000, 12), (5e6, 40_000, 10), (10e6, 60_000, 8), (20e6, 90_000, 6)])
def test_replies_equal_the_oracle(port, rate, n, nr):
    sc = scene(rate, n, nr, 40 + int(rate / 1e6))
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    assert len(want) >= nr - 1
    got, frames, st = run(sc.iq, rate)
    assert mo.same(got, want)
    assert st.replies == len(want)
    bb, avg = port.frontend(sc.iq, rate, True)
    g = am.query_geometry(rate, 7.0, True)
    assert dict(candidates=st.candidates, replies=st.replies, overlap_drops=st.overlap_drops,
                with_altitude=st.with_altitude) == mo.stats(bb, avg, g.rate_int, g.threshold)
    _, frames_off, _ = run(sc.iq, rate, modeac=False)
    assert frames == frames_off


def test_every_cut_and_random_cuts(port):
    rate = 4e6
    sc = scene(rate, 12_000, 3, 7, n_bursts=1)
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    assert len(want) >= 2
    n = sc.n
    for cut in range(512, n, 1499):
        got, _, _ = run(sc.iq, rate, chunks=[cut])
        assert mo.same(got, want), cut
    rng = np.random.default_rng(5)
    cuts = [int(x) for x in rng.integers(1, 3000, 6)]
    got, _, _ = run(sc.iq, rate, chunks=cuts)
    assert mo.same(got, want)


def test_dc_blocker_and_int16(port):
    rate = 4e6
    sc = scene(rate, 30_000, 6, 11)
    want = mo.run_iq(port, sc.iq, rate, 7.0, use_dcblock=True)
    got, _, _ = run(sc.iq, rate, dcblock=True, chunks=[7_000])
    assert len(want) >= 4 and mo.same(got, want)
    q = (np.clip(np.rint(sc.iq * 32768.0), -32768, 32767) / 32768.0).astype(np.float32)
    want16 = mo.run_iq(port, q, rate, 7.0)
    got16, _, _ = run(sc.iq, rate, sc16=True)
    assert len(want16) >= 4 and mo.same(got16, want16)


def test_launch_counts(launches):
    rate = 4e6
    iq = scene(rate, 24_000, 4, 3).iq
    for modeac, extra in ((False, 0), (True, 2)):
        rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, modeac=modeac)
        s0, c0 = rx.stats().kernel_launches, launches()
        rx.process(iq[:2 * 12_000])
        rx.process(iq[2 * 12_000:], flush=True)
        got, want = rx.stats().kernel_launches - s0, launches() - c0
        assert got == want
        if modeac:
            assert got - base == 2 * extra          # two calls, two launches each
        else:
            base = got
        rx.close()


def test_errors():
    rate = 4e6
    iq = scene(rate, 8_000, 1, 2, n_bursts=0).iq
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    rx.process(iq[:4000])
    with pytest.raises(RuntimeError):
        rx.set_modeac(True)                         # a stream has started
    rx.reset()
    rx.set_modeac(True)
    with pytest.raises(RuntimeError):
        rx.defer_resolve(True)
    with pytest.raises(RuntimeError):
        rx.seek(0, 1000)
    assert rx._ctx.call("amb_set_option", b"modeac", 1) == 0
    assert rx._ctx._lib.amb_set_option(rx._ctx._h, b"modeac", 2) == _lib.ERR_INVALID
    rx.process(iq, flush=True)
    assert rx._ctx._lib.amb_drain_modeac_device(rx._ctx._h, None, -1) == _lib.ERR_INVALID
    assert rx._ctx._lib.amb_poll_modeac(rx._ctx._h, None, 3) == _lib.ERR_INVALID
    rx.close()
    nopmf = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=False, modeac=True)
    with pytest.raises(RuntimeError):
        nopmf.process(iq, flush=True)
    nopmf.close()
    slow = am.rx_path(2e6, 7.0, am.msg_queue(), use_pmf=True, modeac=True)
    with pytest.raises(RuntimeError):
        slow.process(iq, flush=True)
    slow.close()
    split = am.preamble(rate, 7.0)
    split._ctx.call("amb_set_option", b"modeac", 1)
    with pytest.raises(RuntimeError):
        split.process(np.zeros(4000, np.float32), np.zeros(4000, np.float32))


def pulses(n, rate, t_us, amp=0.1, start=3000.37, noise=0.002, seed=1):
    """A stream of n samples: noise plus 0.45 us pulses at the times t_us (microseconds after `start`; a (time, amplitude)
    pair gives that pulse its own amplitude)."""
    rng = np.random.default_rng(seed)
    c = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) * np.float32(noise)
    spu = rate / 1e6
    for t in t_us:
        t, a = t if isinstance(t, tuple) else (t, amp)
        s = start + t * spu
        lo = np.arange(int(s) - 1, int(s + 0.45 * spu) + 2, dtype=np.float64)
        cover = np.clip(np.minimum(lo + 1, s + 0.45 * spu) - np.maximum(lo, s), 0.0, None)
        c[lo.astype(np.int64)] += (a * cover).astype(np.complex64)
    return c.view(np.float32).copy()


def frame_us(code, spi):
    return [0.0] + [1.45 * k for k in range(1, 14) if k != 7 and (code >> (13 - k)) & 1] + [20.3] + ([24.65] if spi else [])


@pytest.mark.parametrize("extra", [1.45 * g + 0.725 for g in range(14)] + [10.15])
def test_an_extra_pulse_in_a_gap_or_at_x(port, extra):
    """A pulse in any one of the 14 gaps, or at X, is what rules 4-5 look for; kernel and oracle agree on each."""
    rate = 4e6
    code = 0o1234 & ~0x40
    iq = pulses(8000, rate, frame_us(code, False) + [extra])
    want = mo.run_iq(port, iq, rate, 7.0)
    got, _, _ = run(iq, rate)
    assert mo.same(got, want)
    h = am.query_geometry(rate, 7.0, True).history - 1
    assert not [r for r in want if abs(r["sample_index"] - h - 3000) <= 4]          # the reply is gone


@pytest.mark.parametrize("ratio", [0.3, 0.6, 0.7, 1.5, 2.5])
def test_framing_pulses_of_unequal_power(port, ratio):
    """F2 at `ratio` times F1's amplitude: the weaker framing pulse must stay above the space threshold (rule 4)."""
    rate = 4e6
    code = 0o4321 & ~0x40
    t = [x for x in frame_us(code, False) if x != 20.3] + [(20.3, 0.1 * ratio)]
    iq = pulses(8000, rate, t)
    want = mo.run_iq(port, iq, rate, 7.0)
    got, _, _ = run(iq, rate)
    assert mo.same(got, want)
    h = am.query_geometry(rate, 7.0, True).history - 1
    found = [r for r in want if abs(r["sample_index"] - h - 3000) <= 4]
    assert bool(found) == (0.7 <= ratio <= 1.5), [r["sample_index"] - h for r in want]


def test_rule7_across_a_cut(port):
    """C2 and SPI lie 20.3 us apart: with B2 = 0 the C2 pulse starts a second run of rules 1-5 that only rule 7 drops.
    Every cut that puts the call boundary between the reply and that start needs the carried state."""
    rate = 4e6
    code = (1 << 10)                                 # C2 alone
    iq = pulses(9000, rate, frame_us(code, True))
    want = mo.run_iq(port, iq, rate, 7.0)
    bb, avg = port.frontend(iq, rate, True)
    g = am.query_geometry(rate, 7.0, True)
    st = mo.stats(bb, avg, g.rate_int, g.threshold)
    assert len(want) == 1 and want[0]["code"] == code and want[0]["spi"] == 1 and st["overlap_drops"] >= 1
    i = want[0]["sample_index"] - (g.history - 1)
    guard = g.shard_fwd + g.history - 1
    for cut in range(i + guard - 2, i + guard + mo.geometry(g.rate_int)["slot"][3] + 3):
        got, _, s = run(iq, rate, chunks=[cut])
        assert mo.same(got, want) and s.overlap_drops == st["overlap_drops"], cut
