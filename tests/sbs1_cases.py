"""Seeded message sets for the decoder option "sbs1" (tests/test_sbs1_*.py, tools/sbs1_cost.py): a scene with every
kind of SBS-1 line and every kind of record that takes an id without writing one, and streams that cross the
10000-id window across calls, inside one call, and in a cascade. Messages are (hex, ecc, secs, frac) in time order;
tests/track_cases.py's frames_of() turns them into frames."""
from __future__ import annotations

import numpy as np

import decode_cases as dc
import track_cases as tc
import track_ext_cases as xc

T0 = 1_700_000_000


def df11(aa, ca=5):
    """An all-call reply from address aa (interrogator 0)."""
    return dc.finish(dc.Bits(32).put(1, 5, 11).put(6, 3, ca).put(9, 24, aa).bytes())


def df0(address, alt=None, vs=0, metric=False):
    code = dc.enc_alt13(alt if alt is not None else 0) | (0x40 if metric else 0)
    return dc.finish(dc.Bits(32).put(1, 5, 0).put(6, 1, vs).put(14, 4, 2).put(20, 13, code).bytes(), address)


def df45(df, address, fs, alt=1000, squawk_code=0):
    field = dc.enc_alt13(alt) if df == 4 else squawk_code
    return dc.finish(dc.Bits(32).put(1, 5, df).put(6, 3, fs).put(20, 13, field).bytes(), address)


def velocity(aa, sub, vew, vns, dew=0, dns=0, vr=0, dvr=0):
    """BDS0,9 subtype `sub` (1..4) with the given east-west / north-south words and vertical rate."""
    me = dc.Bits(56).put(1, 5, 19).put(6, 3, sub).put(14, 1, dew).put(15, 10, vew).put(25, 1, dns).put(26, 10, vns) \
        .put(37, 1, dvr).put(38, 9, vr)
    return dc.df17(aa, me.v)


def bds61(aa):
    return dc.df17(aa, dc.Bits(56).put(1, 5, 28).put(6, 3, 1).v)


def tie_position(aa, odd, k):
    """An airborne position whose even-frame latitude 6 (8 + m / 2^17) has m = 1024 mod 2048: an exact '%.5f' tie."""
    la, lo = dc.cpr_encode(48.0 + 0.05 * k, 11.0, odd)
    if not odd:
        la = (la & ~2047) | 1024
    return dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(10000), odd, la, lo))


def mix_scene(seed=3):
    """Every SBS-1 line kind and every 'id but no line' kind, from a few aircraft below 2^15 (the emulator's pairing
    table), with DF20/21 and unqueued frames in between; some stamps with frac next to 1 or at a millisecond tie."""
    rng = np.random.default_rng(seed)
    ev = []
    t = 0.0
    addrs = [0x1234, 0x0ABC, 0x7F01, 0x0042]
    for rep in range(6):
        for j, aa in enumerate(addrs):
            lat, lon = 48.0 + 0.1 * j, 11.0 - 0.2 * j
            fr = [tc.position(aa, lat, lon, 0, False), tc.position(aa, lat, lon, 1, False),
                  tc.position(aa, lat, lon, rep % 2, True), tc.ident(aa, 1 + (rep + j) % 4, "AB%dCD E" % j)]
            fr.append(dc.df17(aa, dc.me_ident(2, 7, "BADCAT")))                    # cat 7 in row 2: IndexError
            for sub in (0, 1, 2, 3):
                fr.append(velocity(aa, sub, int(rng.integers(0, 1024)), int(rng.integers(0, 1024)),
                                   int(rng.integers(0, 2)), int(rng.integers(0, 2)), int(rng.integers(0, 512)),
                                   int(rng.integers(0, 2))))
            fr += [bds61(aa), df11(aa), df0(aa, 1000 + 25 * rep, vs=rep % 2), df0(aa, metric=True),
                   df45(4, aa, (rep + j) % 8, 2000 + 100 * j), df45(5, aa, (rep + 2 * j) % 8, squawk_code=int(rng.integers(0, 1 << 13))),
                   tc.reply(20, aa, rng), tc.reply(21, aa, rng), tie_position(aa, 1, rep), tie_position(aa, 0, rep)]
            for f, ecc in fr:
                t += float(rng.uniform(0.01, 0.3))
                ev.append((t, f, ecc))
    msgs = []
    last = -1.0
    for k, (t, f, ecc) in enumerate(ev):
        t = max(t, last + 1e-3)                         # stamps stay in time order after the moves below
        secs = int(t)
        frac = t - secs
        if k % 17 == 5:
            frac = float(np.nextafter(1.0, 0.0))        # later in the same second
        elif k % 17 == 9:
            secs, frac = (secs, 0.125) if frac <= 0.125 else (secs + 1, 0.125)
        last = secs + frac
        msgs.append((f.hex(), ecc, T0 + secs, frac))
    return msgs


def window_calls(n_first=10000, revisit=60, new_between=3, seconds_per=1e-3):
    """Calls of DF11 replies that cross the 10000-id window. Call 1: n_first new addresses. Call 2 (one call): new
    addresses and revisits of the oldest ones interleaved, so that table ids live at the start of the call expire inside
    it and each expiry hands out an id that pushes the next one out (a cascade). Call 3: the same addresses again."""
    a0 = 0x100000
    t = [0.0]

    def m(aa):
        t[0] += seconds_per
        f, ecc = df11(aa)
        secs = int(t[0])
        return (f.hex(), ecc, T0 + secs, t[0] - secs)

    first = [m(a0 + i) for i in range(n_first)]
    second = []
    for i in range(revisit):
        for j in range(new_between):
            second.append(m(a0 + n_first + i * new_between + j))
        second.append(m(a0 + i))
        second.append(m(a0 + i))
    third = [m(a0 + i) for i in range(0, n_first + revisit * new_between, 97)]
    return [first, second, third]


def big_call(n=12000, revisit=400):
    """One call with more than 10000 new addresses, then revisits of the first ones (whose ids the call itself
    expired)."""
    calls = window_calls(n_first=n, revisit=0)
    msgs = calls[0]
    secs = msgs[-1][2]
    for i in range(revisit):
        f, ecc = df11(0x100000 + (i * 7) % n)
        msgs.append((f.hex(), ecc, secs + 1, (i + 0.5) / (revisit + 1)))
    return msgs


def scenes():
    """(name, msgs) of the equality tests: the mix scene and the track extension's scenes (DF17 positions, op status,
    Comm-B and DF0/4/5/20/21 replies)."""
    yield "mix", mix_scene()
    for name, msgs, _, _ in xc.scenes():
        yield name, msgs
