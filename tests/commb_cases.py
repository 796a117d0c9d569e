"""Seeded message sets for the decoder option "commb" (tests/test_commb_*.py, tools/commb_yield.py). Frames come from
tests/decode_cases.py's encoders with AP = CRC ^ address, so that a DF20/21 record's icao is the address; MB words from
the checker's own encoder (tests/commb_oracle.py). Every generator returns messages (hex, ecc, secs, frac) in time order;
track_cases.frames_of() turns them into frames (every 97th one not queued)."""
from __future__ import annotations

import math

import numpy as np

import commb_oracle as co
import decode_cases as dc
import local_cpr_cases as lc


def reply(df, address, mb, rng):
    """A 112-bit DF20/21 reply carrying the MB word `mb`, AP = CRC ^ address."""
    return dc.long_frame(df, rng, address, mb)


def velocity(aa, speed, south=False, ew=0):
    """DF17 BDS0,9 subtype 1 with north/south speed `speed` kt and east/west `ew` kt: with ew = 0 the decoder's speed
    is exactly `speed` and its track exactly 0 (north) or 180 (south)."""
    me = dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(15, 10, ew).put(25, 1, 1 if south else 0).put(26, 10, speed) \
        .put(38, 9, 5).v
    return dc.df17(aa, me)


def _msgs(ev):
    ev.sort(key=lambda e: e[0])
    return [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc in ev]


def unique_word(reg, rng):
    """A random word of register `reg` that is a candidate for that register alone."""
    while True:
        vals = {}
        for i in range(5):
            if rng.random() < 0.7:
                lo, hi = co.raw_range(reg, i)
                vals[i] = int(rng.integers(lo, hi + 1))
        if reg == 0x40 and 2 in vals:
            vals[2] = int(rng.integers(700, 3001))
        mb = co.encode(reg, vals)
        if co.candidates(mb) == [reg]:
            return mb


def ambiguous_word(rng, gs=None, trk=None):
    """A word that is a candidate for 5,0 and 6,0, with 5,0's GS and track present (GS raw `gs`, track raw `trk` when
    given)."""
    for _ in range(100000):
        vals = {1: trk if trk is not None else int(rng.choice([0, int(rng.integers(-1024, -523))])),
                2: gs if gs is not None else int(rng.integers(0, 251))}
        if rng.random() < 0.8:
            vals[0] = int(rng.integers(-284, 285))
        if rng.random() < 0.7:
            vals[3] = int(rng.integers(-187, 188))
        if rng.random() < 0.5:
            vals[4] = int(rng.integers(max(0, vals[2] - 125), min(300, vals[2] + 125) + 1))
        mb = co.encode(0x50, vals)
        c = co.candidates(mb)
        if 0x50 in c and 0x60 in c:
            return mb
    raise ValueError("no ambiguous word for gs=%r trk=%r" % (gs, trk))


def unique_scene(seed=1):
    """Each register decoded uniquely, words with no candidate, and the untouched: parser registers (first byte
    0x00/0x10/0x20/0x30), DF20/21 with the parser's words, short replies, DF17 squitters."""
    rng = np.random.default_rng(seed)
    ev, t = [], 1.0
    for k in range(240):
        aa = 0x100 + k % 16
        kind = k % 8
        if kind < 3:
            mb = unique_word(co.REGS[kind], rng)
        elif kind == 3:
            mb = int(rng.integers(0, 1 << 56, dtype=np.uint64))                # mostly no candidate
        elif kind == 4:
            mb = (int(rng.integers(0, 4)) << 52) | int(rng.integers(0, 1 << 48))   # the parser's registers
        elif kind == 5:
            mb = co.encode(0x50, {1: -1000, 2: 200})                            # ambiguous without a reference
        elif kind == 6:
            ev.append((t, *dc.short_frame(int(rng.choice([4, 5, 20, 21])), rng, aa)))
            t += 0.05
            continue
        else:
            ev.append((t, *velocity(aa, 300)))
            t += 0.05
            continue
        ev.append((t, *reply(int(rng.choice([20, 21])), aa, mb, rng)))
        t += float(rng.choice([0.0, 0.05, 0.3]))
    return _msgs(ev)


def reference_scene(S=30, seed=2):
    """Constructed 5,0/6,0-ambiguous words, each address with its own story: a reference that agrees, disagrees in
    speed or track, is exactly S old, older than S, stamped later than the reply, none at all; GS differences of 20
    and 21 kt; track differences across +-180 deg and one LSB either side of 10 deg."""
    rng = np.random.default_rng(seed)
    ev = []
    a = [0x2000]

    def story(dt, speed, south, gs, trk):
        aa = a[0]
        a[0] += 1
        t0 = 10.0 + 0.5 * (aa - 0x2000)
        if speed is not None:
            ev.append((t0, *velocity(aa, speed, south)))
        mb = ambiguous_word(rng, gs=gs, trk=trk)
        ev.append((t0 + dt, *reply(int(rng.choice([20, 21])), aa, mb, rng)))

    for _ in range(2):
        story(1.0, 400, False, 200, 0)          # agrees: 5,0
        story(1.0, 300, False, 200, 0)          # speed disagrees: 6,0
        story(1.0, 400, False, 200, -1000)      # track disagrees: 6,0
        story(float(S), 400, False, 200, 0)     # exactly S old: applies
        story(S + 0.5, 400, False, 200, 0)      # older than S: ambiguous
        story(1.0, None, False, 200, 0)         # no reference: ambiguous
        story(1.0, 380, False, 200, 0)          # |2 gs - speed| = 20: agrees
        story(1.0, 379, False, 200, 0)          # 21: disagrees
        story(1.0, 420, False, 200, 0)          # 20 the other way
        story(1.0, 400, True, 200, -1024)       # -180 vs 180: 0 deg across the wrap, agrees
        story(1.0, 400, True, 200, -968)        # 9.84 deg across the wrap: agrees
        story(1.0, 400, True, 200, -967)        # 10.02 deg: disagrees
        story(1.0, 400, True, 200, 0)           # 180 deg: disagrees
    # stamped later: the reply comes after the velocity record in the stream but carries an earlier time
    for _ in range(3):
        aa = a[0]
        a[0] += 1
        t0 = 200.0 + aa - 0x2000
        ev.append((t0, *velocity(aa, 400)))
        ev.append((t0 + 0.001, *reply(20, aa, ambiguous_word(rng, gs=200, trk=0), rng)))
    msgs = _msgs(ev)
    # move each stamped-later pair's reply 0.5 s back in time without changing the stream order
    out = []
    for k, (h, ecc, s, f) in enumerate(msgs):
        t = s + f
        if t >= 200.0 and bytes.fromhex(h)[0] >> 3 == 20 and k > 0 and msgs[k - 1][2] + msgs[k - 1][3] >= 200.0:
            t -= 0.5
            out.append((h, ecc, int(t), float(np.float64(t - int(t)))))
        else:
            out.append((h, ecc, s, f))
    return out


def limits_scene(seed=3):
    """Every plausibility limit at the limit and one LSB past it, a status-0 field with data, a reserved 4,0 bit set."""
    rng = np.random.default_rng(seed)
    words = []
    for reg, i, at, past in ((0x40, 0, 3125, 3126), (0x40, 1, 3125, 3126), (0x40, 2, 700, 699), (0x40, 2, 3000, 3001),
                             (0x50, 0, 284, 285), (0x50, 0, -284, -285), (0x50, 2, 400, 401), (0x50, 4, 300, 301),
                             (0x60, 1, 500, 501), (0x60, 2, 250, 251), (0x60, 3, 187, 188), (0x60, 3, -187, -188),
                             (0x60, 4, 187, 188), (0x60, 4, -187, -188)):
        for v in (at, past):
            words.append(co.encode(reg, {i: v}))
            base = {j: 1 for j in range(5) if j != i}
            if reg == 0x40:
                base[2] = 1000
            base[i] = v
            words.append(co.encode(reg, base))
    for d in (125, 126):                                        # |GS - TAS|
        words.append(co.encode(0x50, {2: 300, 4: 300 - d if 300 - d >= 0 else 0}))
        words.append(co.encode(0x50, {2: 100 + d, 4: 100}))
    for reg in co.REGS:
        for i in range(5):                                      # data behind a status bit of 0
            mb = co.encode(reg, {j: 1 for j in range(5) if j != i} if reg != 0x40 else {0: 1, 1: 1, 2: 1000, 3: 1, 4: 1})
            st, sign, first, n = co.LAYOUT[reg][i]
            words.append((mb & ~(1 << (56 - st))) | (1 << (57 - first - n)))
    for j in range(10):                                         # a reserved bit of 4,0
        words.append(co.encode(0x40, {0: 100, 2: 1000}, reserved=1 << j))
    ev = [(1.0 + 0.01 * k, *reply(20 + k % 2, 0x3000 + k % 7, mb, rng)) for k, mb in enumerate(words)]
    return _msgs(ev)


def bucket_scene(n_aircraft=32, seed=9, S=30):
    """n_aircraft addresses sharing one bucket of the partition, each with velocities and replies of every kind."""
    rng = np.random.default_rng(seed)
    addrs = lc.same_bucket_addresses(n_aircraft)
    ev = []
    for k in range(3000):
        aa = int(addrs[k % n_aircraft])
        t = 0.02 * k
        r = rng.random()
        if r < 0.3:
            ev.append((t, *velocity(aa, int(rng.choice([380, 400, 420, 300])), bool(rng.random() < 0.5))))
        elif r < 0.8:
            ev.append((t, *reply(20, aa, ambiguous_word(rng, gs=200, trk=int(rng.choice([0, -1024, -968, -700]))), rng)))
        else:
            ev.append((t, *reply(21, aa, unique_word(co.REGS[int(rng.integers(0, 3))], rng), rng)))
    return _msgs(ev)


def burst_scene(seed=4):
    """One address with far more than 32 records back to back (one 32-lane step holds only it): velocities and
    ambiguous replies interleaved, so that lanes take an earlier lane's velocity, the table's, or none; a second
    address now and then."""
    rng = np.random.default_rng(seed)
    aa, bb = 0x2BCD, 0x2BCE
    ev, t = [], 10.0
    for k in range(200):
        r = rng.random()
        if r < 0.25:
            ev.append((t, *velocity(aa, int(rng.choice([400, 300])), bool(rng.random() < 0.5))))
        elif r < 0.9:
            ev.append((t, *reply(20, aa, ambiguous_word(rng, gs=200, trk=int(rng.choice([0, -1024]))), rng)))
        else:
            ev.append((t, *velocity(bb, 400)))
        if k % 60 == 59:
            t += 5.0                                            # older than S = 3
        t += float(rng.choice([0.0, 0.001, 0.01]))
    return _msgs(ev)


# ---- a synthetic fleet (tools/commb_yield.py, the GPU stress) -----------------------------------------------------------
def _q(x, lsb, lo, hi):
    return int(max(lo, min(hi, round(x / lsb))))


def fleet_scene(n_aircraft=300, seconds=200.0, seed=17, reply_rate=4.0, other_share=0.15):
    """n_aircraft aircraft over `seconds`: each sends its ADS-B velocity at about 2 Hz and DF20/21 replies (about
    `reply_rate` per second) carrying 4,0, 5,0 and 6,0 words drawn from its flight state (ground speed and TAS with a
    wind, heading = track + crab + declination), and in `other_share` of them an "other" word: a 1,7-like capability
    word, a 4,4-like met word or a random one. Returns (msgs, truth): truth[k] = 0x40 / 0x50 / 0x60 / "other" / None
    (not a reply) for message k."""
    rng = np.random.default_rng(seed)
    addrs = rng.choice(np.arange(1, 1 << 24), n_aircraft, replace=False)
    ev = []
    for aa in addrs:
        aa = int(aa)
        tas = float(rng.uniform(250, 480))
        trk = float(rng.uniform(0, 360))
        wind, wdir = float(rng.uniform(0, 80)), float(rng.uniform(0, 360))
        wn, we = -wind * math.cos(math.radians(wdir)), -wind * math.sin(math.radians(wdir))
        gn = tas * math.cos(math.radians(trk)) + wn
        ge = tas * math.sin(math.radians(trk)) + we
        gs = math.hypot(gn, ge)
        gtrk = math.degrees(math.atan2(ge, gn)) % 360
        crab = float(rng.uniform(-8, 8))
        decl = float(rng.uniform(-10, 10))
        hdg = (gtrk + crab + decl + 180) % 360 - 180
        ias = tas * float(rng.uniform(0.55, 0.75))
        mach = tas / 600.0
        alt = int(rng.integers(100, 2500))
        t0 = float(rng.uniform(0, seconds / 2))
        t = t0
        while t < seconds:                                      # ADS-B velocity about 2 Hz
            ns, ew = int(round(abs(gn))), int(round(abs(ge)))
            me = dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(14, 1, 1 if ge < 0 else 0).put(15, 10, ew) \
                .put(25, 1, 1 if gn < 0 else 0).put(26, 10, ns).put(38, 9, 1).v
            ev.append((t, *dc.df17(aa, me), None))
            t += float(rng.uniform(0.4, 0.6))
        t = t0 + float(rng.uniform(0, 1))
        while t < seconds:
            r = rng.random()
            df = int(rng.choice([20, 21]))
            if r < other_share:
                k = int(rng.integers(0, 3))
                if k == 0:
                    mb = (0x17 << 48) | int(rng.integers(0, 1 << 48))  # 1,7-like: capability bits
                elif k == 1:
                    mb = (0x4 << 52) | int(rng.integers(0, 1 << 52))   # 4,4-like: met data
                else:
                    mb = int(rng.integers(0, 1 << 56, dtype=np.uint64))
                ev.append((t, *reply(df, aa, mb, rng), "other"))
            else:
                reg = co.REGS[int(rng.integers(0, 3))]
                if reg == 0x40:
                    vals = {0: alt, 2: int(rng.integers(1000, 2400)), 3: int(rng.integers(0, 8))}
                    if rng.random() < 0.5:
                        vals[1] = alt
                elif reg == 0x50:
                    vals = {0: _q(float(rng.normal(0, 3)), 45 / 256, -511, 511),
                            1: _q((gtrk + 180) % 360 - 180, 90 / 512, -1024, 1023), 2: _q(gs, 2, 0, 1023),
                            3: _q(float(rng.normal(0, 0.3)), 8 / 256, -511, 511), 4: _q(tas, 2, 0, 1023)}
                else:
                    vals = {0: _q(hdg, 90 / 512, -1024, 1023), 1: _q(ias, 1, 0, 1023), 2: _q(mach, 2.048 / 512, 0, 1023),
                            3: _q(float(rng.normal(0, 500)), 32, -511, 511), 4: _q(float(rng.normal(0, 500)), 32, -511, 511)}
                ev.append((t, *reply(df, aa, co.encode(reg, vals), rng), reg))
            t += float(rng.exponential(1.0 / reply_rate))
    ev.sort(key=lambda e: e[0])
    msgs = [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc, _ in ev]
    return msgs, [e[3] for e in ev]


def scenes():
    """(name, msgs, S) for the equality tests."""
    yield "unique", unique_scene(), 30
    yield "reference", reference_scene(S=30), 30
    yield "limits", limits_scene(), 30
    yield "bucket", bucket_scene(), 30
    yield "burst", burst_scene(), 3
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    yield "case14", msgs, 10
