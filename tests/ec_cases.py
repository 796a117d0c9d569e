"""Shared scenarios of the error-correction tests (option "ec"): tests/test_ec_simt.py runs them against the emulated
library, tests/test_ec_gpu.py on the device. Expected results always come from the oracle plus the brute-force checker
of tests/ec_oracle.py."""
import os
import sys

import numpy as np

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_oracle as eo  # noqa: E402

K = 9
PRE = (2.0, 0.0, 2.0, 0.0)                 # reference level 1.0: llslicer's band is (0.707, 1.414)


def bits_of(frame: bytes):
    return [(frame[j // 8] >> (7 - j % 8)) & 1 for j in range(8 * len(frame))]


def packet_chips(frame: bytes, low=(), wrong=(), sure_wrong=()):
    """240 chips of `frame`: bits in `low` are right but low-confidence (both chips in band), bits in `wrong` are
    low-confidence and wrong, bits in `sure_wrong` wrong with full confidence; all others right and sure."""
    c = np.zeros(240, np.float32)
    c[[0, 2, 7, 9]] = PRE
    for j, b in enumerate(bits_of(frame)):
        if j in wrong:
            pair = (1.0, 1.2) if b else (1.2, 1.0)
        elif j in low:
            pair = (1.2, 1.0) if b else (1.0, 1.2)
        elif j in sure_wrong:
            pair = (0.0, 1.0) if b else (1.0, 0.0)
        else:
            pair = (1.0, 0.0) if b else (0.0, 1.0)
        c[16 + 2 * j], c[17 + 2 * j] = pair
    return c


def slicer_packets(codewords):
    """(chips[n, 240], healed chips[n, 240]) covering every outcome at K = 9. `healed` has the wrong bits right (still
    low-confidence): what a fixed frame must equal."""
    rng = np.random.default_rng(31)
    out = []

    def add(df, L, wrong=(), sure_wrong=()):
        fr = synth.make_frame(df, rng)
        out.append((packet_chips(fr, low=set(L) - set(wrong), wrong=wrong, sure_wrong=sure_wrong),
                    packet_chips(fr, low=L, sure_wrong=sure_wrong)))

    for t in range(6):                                      # fixed: DF17 / DF11, message and parity bits, 1-4 flips
        nb = 112 if t % 2 == 0 else 56
        L = sorted(int(p) for p in rng.choice(np.arange(5, nb), 7 if nb == 112 else 6, replace=False))
        add(17 if nb == 112 else 11, L, wrong=L[-1 - t % 4:])
    add(17, [2, 30, 60, 100], wrong=[60])                   # a DF bit in L (right, low confidence): never flipped
    add(17, list(range(20, 30)), wrong=[25])                # too many: 10 > K
    add(17, list(range(20, 44)), wrong=[25])                # 24 low-confidence bits: saturated
    add(11, [12, 20, 33], wrong=[20], sure_wrong=[40])      # an error outside L: no solution
    for nb, cw in codewords.items():                        # L holds a codeword: two solutions
        add(17 if nb == 112 else 11, sorted(cw + [min(set(range(5, nb)) - set(cw))]), wrong=cw[:2])
    add(17, [50, 51])                                       # passes as it is
    add(11, list(range(10, 20)), wrong=[15])                # DF11 with 10 low-confidence bits: dropped by :171, crc 0
    add(20, [], sure_wrong=[40])                            # DF20: no CRC rule, never a candidate
    chips, healed = zip(*out)
    return np.stack(chips), np.stack(healed)


def check_frame(got, st):
    """An amb_frame against the checker's verdict st = (status, flips, corrected oracle frame)."""
    g = st[2]
    assert bytes(got.data) == bytes(g.data), (bytes(got.data).hex(), bytes(g.data).hex())
    assert (got.crc, got.passed, got.nbits, got.df, got.numlowconf) == (g.crc, g.passed, g.nbits, g.df, g.numlowconf)
    assert bytes(got.lowconfbits) == bytes(g.lowconfbits)
    assert got.ref_level == g.ref_level or (np.isnan(got.ref_level) and np.isnan(g.ref_level))
    assert (got.ec, got.ec_flips) == (st[0], len(st[1])), (got.ec, got.ec_flips, st[0], st[1])
    assert bytes(got.pad_)[2:] == b"\0" * 4


def run_slicer_packets(port, codewords, k=K):
    chips, healed = slicer_packets(codewords)
    n = chips.shape[0]
    q = am.msg_queue()
    sl = am.slicer(q, ec=k)
    tags = [(0, 0.0)] * n
    frames = sl.process(chips, tags)
    want = port.run_slicer(chips, np.zeros(n, np.uint64), np.zeros(n))
    statuses = []
    for f, w, h in zip(frames, want.frames, healed):
        st = eo.correct(w, k)
        check_frame(f, st)
        statuses.append(st[0])
        if st[0] == eo.EC_FIXED:                            # the message of the healed packet, bit for bit
            hw = port.slice_packet(h)
            assert hw.passed and bytes(hw.data) == bytes(st[2].data)
            assert am.format_message(f, False) == port.format_message(hw, False)
    assert q.strings() == eo.merged_messages(port, want.frames, k)
    return statuses


# ---- the fused chain on an IQ scene whose bursts carry low-confidence wrong bits ---------------------------------
def ec_scene(rate, n, nb, seed, wrong_max=3, noise_sigma=0.003, quantize_bits=14):
    """Bursts spaced apart; in all but every fifth, 1..wrong_max data or parity bits are sent with their two chips at
    nearly equal amplitude, the wrong one slightly stronger (both inside llslicer's band: low confidence and wrong).
    The first burst always carries such bits, so the stream's first message is a corrected one. Returns
    (interleaved float32 IQ, sent frames)."""
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
        bits = np.array(bits_of(frame))
        chips = np.zeros(240)
        chips[[0, 2, 7, 9]] = 1.0
        chips[16:16 + 2 * nbits:2] = bits
        chips[17:17 + 2 * nbits:2] = 1 - bits
        if k == 0 or k % 5:
            for j in rng.choice(np.arange(5, nbits), int(rng.integers(1, wrong_max + 1)), replace=False):
                a = 16 + 2 * int(j) + (0 if bits[j] else 1)   # the chip that is on
                chips[a], chips[a ^ 1] = 0.93, 1.0            # its partner (the wrong decision) slightly stronger
        amp = 0.3
        start = span + k * gap + rng.uniform(0, gap - span)
        knots = np.arange(241) * spc
        cum = np.concatenate([[0.0], np.cumsum(chips) * spc])
        n0, n1 = int(np.floor(start)), int(np.ceil(start + 240 * spc)) + 1
        integ = np.interp(np.arange(n0, n1 + 1) - start, knots, cum)
        ph = rng.uniform(0, 2 * np.pi)
        c[n0:n1] += (amp * np.diff(integ) * np.exp(1j * ph)).astype(np.complex64)
        sent.append(frame)
    if quantize_bits:
        q = float(1 << (quantize_bits - 1))
        np.clip(np.rint(iq * q), -q, q - 1, out=iq)
        iq /= np.float32(q)
    return iq.reshape(2 * n), sent


def run_chain(iq, rate, ec, chunks=None, resolver=0, thr=7.0, pmf=True, set_zero_first=False):
    q = am.msg_queue()
    rx = am.rx_path(rate, thr, q, use_pmf=pmf, ec=ec)
    if set_zero_first:
        rx.set_ec(7)
        rx.set_ec(0)
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


def check_chain(port, iq, rate, frames, msgs, k, thr=7.0, pmf=True):
    want = port.run_iq(iq, rate, thr, pmf, co.MA_CANONICAL)
    assert [f.sample_index for f in frames] == [int(x) for x in want.index]
    statuses = []
    for f, w in zip(frames, want.frames):
        st = eo.correct(w, k)
        check_frame(f, st)
        statuses.append(st[0])
    assert msgs == eo.merged_messages(port, want.frames, k)
    return want, statuses
