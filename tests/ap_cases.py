"""Shared scenarios of the "ap_filter" tests (address/parity check): tests/test_ap_simt.py runs them against the
emulated library, tests/test_ap_gpu.py on the device. Expected results always come from the oracle plus the checkers
of tests/ec_oracle.py, tests/ec_any_oracle.py and tests/ap_oracle.py."""
import os
import sys

import numpy as np

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ap_oracle as apo  # noqa: E402


def fleet_scene(rate, n, n_aircraft, nb, seed, **kw):
    """A fleet scene (synth.make_fleet_scene) on the 14-bit grid: interleaved float32 IQ and the bursts sent."""
    kw.setdefault("quantize_bits", 14)
    sc = synth.make_fleet_scene(rate, n, n_aircraft, nb, seed, **kw)
    return sc.iq, sc.bursts


def place_scene(rate, n, placed, seed, noise_sigma=0.003):
    """Quiet IQ with one burst per (start, frame) in `placed` at high SNR, on the 14-bit grid."""
    rng = np.random.default_rng(seed)
    spc = rate / 2e6
    iq = (rng.standard_normal((n, 2)) * noise_sigma).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    for s, frame in placed:
        n0, w = synth.burst_waveform(synth.Burst(float(s), frame, 0.3, float(rng.uniform(0, 2 * np.pi))), spc)
        c[n0:n0 + w.size] += w
    q = float(1 << 13)
    np.clip(np.rint(iq * q), -q, q - 1, out=iq)
    iq /= np.float32(q)
    return iq.reshape(2 * n)


def one_frame(df, addr, rng, code=0):
    """One frame of `df` from aircraft `addr` (II/SI `code` for DF11)."""
    fr, nb = synth.make_fleet_frames(np.array([df]), np.array([addr], np.uint32), np.array([code], np.uint32), rng)
    return fr[0, :nb[0]].tobytes()


def run_chain(iq, rate, s, k=0, m=0, chunks=None, resolver=0, set_zero_first=False, rx=None, q=None, close=True):
    q = q if q is not None else am.msg_queue()
    rx = rx or am.rx_path(rate, 7.0, q, use_pmf=True, ec=k, ec_any=m, ap_filter=s)
    if set_zero_first:
        rx.set_ap_filter(60)
        rx.set_ap_filter(0)
    rx.set_option("resolver", resolver)
    frames, pos, n = [], 0, iq.size // 2
    for c in (chunks or []) + [n]:
        c = int(min(c, n - pos))
        last = pos + c >= n
        rx.process(iq[2 * pos: 2 * (pos + c)], flush=last)
        frames += rx.frames
        pos += c
        if last:
            break
    st = rx.stats()
    if close:
        rx.close()
    return q.strings(), frames, st


def check_frames(frames, want_frames, k, m, s, rate_int, table=None):
    """Every amb_frame against the oracle's frame after the checkers; returns [(ec, ec_any, ap) statuses, kinds]."""
    res = apo.apply(want_frames, k, m, s, rate_int, table)
    assert len(frames) == len(res)
    out = []
    for got, (ec_st, any_st, ap, g) in zip(frames, res):
        assert got.sample_index == g.index
        assert bytes(got.data) == bytes(g.data), (bytes(got.data).hex(), bytes(g.data).hex())
        assert (got.crc, got.passed, got.nbits, got.df, got.numlowconf) == (g.crc, g.passed, g.nbits, g.df, g.numlowconf)
        assert bytes(got.lowconfbits) == bytes(g.lowconfbits)
        assert got.ref_level == g.ref_level or (np.isnan(got.ref_level) and np.isnan(g.ref_level))
        bits = tuple(any_st[1]) + (0,) * (2 - len(any_st[1]))
        assert bytes(got.pad_) == bytes((ec_st[0], len(ec_st[1]), any_st[0]) + bits + (ap,)), (bytes(got.pad_), ec_st, any_st, ap)
        kind = apo.classify(g, ec_st[0], any_st[0])[0] if ap == apo.AP_NOT_CHECKED else None
        out.append((ec_st[0], any_st[0], ap, kind))
    return out


def check_chain(port, iq, rate, frames, msgs, s, k=0, m=0, table=None):
    want = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL)
    assert [f.sample_index for f in frames] == [int(x) for x in want.index]
    statuses = check_frames(frames, want.frames, k, m, s, int(rate), table)
    assert msgs == apo.merged_messages(port, want.frames, k, m, s, int(rate), table=table)
    return want, statuses


def count(statuses, ap):
    return sum(x[2] == ap for x in statuses)
