"""Shared scenarios of the "ec_any" tests (DF17 correction by at most M bits anywhere): tests/test_ec_any_simt.py runs
them against the emulated library, tests/test_ec_any_gpu.py on the device. Expected results always come from the
oracle plus the brute-force checkers of tests/ec_oracle.py and tests/ec_any_oracle.py."""
import os
import sys

import numpy as np

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_any_oracle as ea  # noqa: E402
import ec_cases as ecc  # noqa: E402
import ec_oracle as eo  # noqa: E402

M = 2


def slicer_packets():
    """chips[n, 240] of DF17 packets whose bits are wrong with full confidence at chosen positions (the first and last
    position of the search set, both sides of the message/parity boundary), plus what must not be touched."""
    rng = np.random.default_rng(41)
    out = []

    def add(df, sure_wrong=(), low=(), wrong=()):
        fr = synth.make_frame(df, rng)
        out.append(ecc.packet_chips(fr, low=set(low) - set(wrong), wrong=wrong, sure_wrong=sure_wrong))

    for e in [(5,), (87,), (88,), (111,), (40,), (5, 6), (5, 111), (87, 88), (86, 87), (88, 89), (110, 111), (30, 64)]:
        add(17, sure_wrong=e)
    add(17, sure_wrong=(5, 87, 88))                         # three bits: no solution
    add(17, sure_wrong=(20, 60, 100))
    add(11, sure_wrong=(20,))                               # DF11: never tried
    add(17, sure_wrong=(4,))                                # DF field flipped (DF16): not a candidate
    add(17, sure_wrong=(2, 40))
    add(17, low=[30, 60, 100], wrong=[60])                  # "ec" fixes it (when on): not tried again
    add(17, low=list(range(20, 30)), wrong=[25], sure_wrong=(70,))   # too many for "ec", then two bits
    add(17, low=list(range(20, 44)), sure_wrong=(50,))      # saturated count of 24: still a candidate
    add(17, low=[12, 20, 33], wrong=[20], sure_wrong=(99,))  # "ec" finds no solution, then two bits
    add(17)                                                 # passes as it is
    add(20, sure_wrong=(40,))                               # DF20: no CRC rule
    return np.stack(out)


def check_frame(got, st, any_st):
    """An amb_frame against the checkers' verdicts: st = (ec status, ec flips, frame after both passes), any_st =
    (ec_any status, ec_any bits)."""
    g = st[2]
    assert bytes(got.data) == bytes(g.data), (bytes(got.data).hex(), bytes(g.data).hex())
    assert (got.crc, got.passed, got.nbits, got.df, got.numlowconf) == (g.crc, g.passed, g.nbits, g.df, g.numlowconf)
    assert bytes(got.lowconfbits) == bytes(g.lowconfbits)
    assert got.ref_level == g.ref_level or (np.isnan(got.ref_level) and np.isnan(g.ref_level))
    assert (got.ec, got.ec_flips) == (st[0], len(st[1])), (got.ec, got.ec_flips, st[0], st[1])
    bits = tuple(any_st[1]) + (0,) * (2 - len(any_st[1]))
    assert (got.ec_any, got.ec_any_bits) == (any_st[0], bits), (got.ec_any, got.ec_any_bits, any_st)
    assert bytes(got.pad_)[5:] == b"\0"


def check_frames(frames, want_frames, k, m, table=None):
    """Every amb_frame against the oracle's frame after both checkers; returns [(ec status, ec_any status)]."""
    statuses = []
    for f, w in zip(frames, want_frames):
        (st, flips), any_st, g = ea.correct_both(w, k, m, table)
        check_frame(f, (st, flips, g), any_st)
        statuses.append((st, any_st[0]))
    return statuses


def run_slicer_packets(port, k, m):
    chips = slicer_packets()
    n = chips.shape[0]
    q = am.msg_queue()
    sl = am.slicer(q, ec=k, ec_any=m)
    frames = sl.process(chips, [(0, 0.0)] * n)
    want = port.run_slicer(chips, np.zeros(n, np.uint64), np.zeros(n))
    assert len(frames) == n
    statuses = check_frames(frames, want.frames, k, m)
    assert q.strings() == ea.merged_messages(port, want.frames, k, m)
    return statuses


PATTERNS = [(5,), (87,), (88,), (111,), (5, 111), (87, 88), (20, 60, 100), (), (33, 34), (70,)]


def chosen(k, df, rng):
    """Full-confidence wrong bits of burst k: a fix at burst 0, so the stream's first message is a corrected one."""
    if df != 17:
        return (20,) if k % 3 == 0 else ()
    return (40,) if k == 0 else PATTERNS[k % len(PATTERNS)]


def any_scene(rate, n, nb, seed, wrong_max=0, noise_sigma=0.003, quantize_bits=14):
    """The waveform of ec_cases.ec_scene: bursts spaced apart, DF17 or DF11. The bits `chosen` picks are sent wrong with
    full confidence; with wrong_max > 0, all but every fifth burst also carry 1..wrong_max low-confidence wrong bits
    (both chips in llslicer's band, the wrong one slightly stronger). Returns (interleaved float32 IQ, sent frames)."""
    rng = np.random.default_rng(seed)
    spc = rate / 2e6
    iq = (rng.standard_normal((n, 2)) * noise_sigma).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    span = 240 * spc + 8
    gap = (n - 3 * span) / nb
    sent = []
    for k in range(nb):
        df = 17 if rng.random() < 0.6 else 11
        frame = synth.make_frame(df, rng)
        nbits = 8 * len(frame)
        bits = np.array(ecc.bits_of(frame))
        bits[list(chosen(k, df, rng))] ^= 1
        chips = np.zeros(240)
        chips[[0, 2, 7, 9]] = 1.0
        chips[16:16 + 2 * nbits:2] = bits
        chips[17:17 + 2 * nbits:2] = 1 - bits
        if wrong_max and k % 5:
            for j in rng.choice(np.arange(5, nbits), int(rng.integers(1, wrong_max + 1)), replace=False):
                a = 16 + 2 * int(j) + (0 if bits[j] else 1)   # the chip that is on
                chips[a], chips[a ^ 1] = 0.93, 1.0            # its partner (the wrong decision) slightly stronger
        start = span + k * gap + rng.uniform(0, gap - span)
        knots = np.arange(241) * spc
        cum = np.concatenate([[0.0], np.cumsum(chips) * spc])
        n0, n1 = int(np.floor(start)), int(np.ceil(start + 240 * spc)) + 1
        integ = np.interp(np.arange(n0, n1 + 1) - start, knots, cum)
        ph = rng.uniform(0, 2 * np.pi)
        c[n0:n1] += (0.3 * np.diff(integ) * np.exp(1j * ph)).astype(np.complex64)
        sent.append(frame)
    q = float(1 << (quantize_bits - 1))
    np.clip(np.rint(iq * q), -q, q - 1, out=iq)
    iq /= np.float32(q)
    return iq.reshape(2 * n), sent


def run_chain(iq, rate, k, m, chunks=None, resolver=0, set_zero_first=False):
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True, ec=k, ec_any=m)
    if set_zero_first:
        rx.set_ec_any(2)
        rx.set_ec_any(0)
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
    rx.close()
    return q.strings(), frames, st


def check_chain(port, iq, rate, frames, msgs, k, m, table=None):
    want = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL)
    assert [f.sample_index for f in frames] == [int(x) for x in want.index]
    statuses = check_frames(frames, want.frames, k, m, table)
    assert msgs == ea.merged_messages(port, want.frames, k, m, table=table)
    return want, statuses


def n_fixed(statuses):
    return sum(eo.EC_FIXED in s for s in statuses)
