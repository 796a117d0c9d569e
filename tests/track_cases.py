"""Seeded message sets for the decoder option "track" (tests/test_track_*.py, tools/track_cost.py). Frames come from
tests/decode_cases.py's encoders and tests/local_cpr_cases.py's scenes; every generator returns messages
(hex, ecc, secs, frac) in time order, and frames_of() turns them into frames with varied reference levels."""
from __future__ import annotations

import numpy as np

import decode_cases as dc
import local_cpr_cases as lc


def frames_of(msgs, seed=0, unqueued_every=97):
    """FRAME_DTYPE array of msgs with reference levels drawn from 1e-9 .. 1 (some below the 1e-8 floor of the rssi);
    every `unqueued_every`-th frame is marked as not queued by the slicer (passed = 0)."""
    from gr_air_modes_b200 import decode
    arr, n = decode.frames_from_messages(msgs)
    fr = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE)[:n].copy()
    rng = np.random.default_rng(seed)
    fr["ref_level"] = (10.0 ** rng.uniform(-9, 0, n)).astype(np.float32)
    if unqueued_every:
        fr["passed"][unqueued_every - 1::unqueued_every] = 0
    return fr


def _mb(bds1, rng):
    """A Comm-B word the parser handles: register bds1 (0..3), bds2 = 0."""
    return dc.Bits(56).put(1, 4, bds1).put(9, 48, int(rng.integers(0, 1 << 48))).v


def reply(df, address, rng, alt=None):
    """DF0/4/5/20/21 reply whose AP field carries `address` (so the record's icao is that address); DF0/4/20 with a
    25 ft altitude (`alt`), else random contents."""
    if df in (20, 21):
        fr, ecc = dc.long_frame(df, rng, address, _mb(int(rng.integers(0, 4)), rng))
        if alt is None:
            return fr, ecc
        b = dc.Bits(88).put(1, 5, df).put(6, 14, int(rng.integers(0, 1 << 14))).put(20, 13, dc.enc_alt13(alt)) \
            .put(33, 56, _mb(0, rng))
        return dc.finish(b.bytes(), address)
    if alt is None:
        return dc.short_frame(df, rng, address)
    b = dc.Bits(32).put(1, 5, df).put(6, 14, int(rng.integers(0, 1 << 14))).put(20, 13, dc.enc_alt13(alt))
    return dc.finish(b.bytes(), address)


def position(aa, lat, lon, odd, surface, alt=10000, gillham=False, rng=None):
    la, lo_ = dc.cpr_encode(lat, lon, odd, surface)
    if surface:
        return dc.df17(aa, dc.me_surface(7, 12, 1, int(rng.integers(0, 128)) if rng is not None else 33, odd, la, lo_))
    return dc.df17(aa, dc.me_airborne(11, (dc.enc_alt12(alt) & ~0x10) if gillham else dc.enc_alt12(alt), odd, la, lo_))


def velocity(aa, sub, rng):
    return dc.df17(aa, dc.Bits(56).put(1, 5, 19).put(6, 3, sub).put(9, 48, int(rng.integers(0, 1 << 48))).v)


def ident(aa, ftc, text):
    return dc.df17(aa, dc.me_ident(ftc, 3, text))


def eps(aa, v):
    return dc.df17(aa, dc.Bits(56).put(1, 5, 28).put(9, 3, v).v)


def _msgs(ev):
    ev.sort(key=lambda e: e[0])
    return [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc in ev]


def life_scene(seed=1, S=20):
    """A handful of aircraft living through the rules: silences longer than S after which a DF0/4/5/20/21 reply or a
    DF11 comes first (and must not revive the row) before a DF17 does; a silence of exactly S (still alive); replies to
    known and to unknown addresses; surface <-> airborne transitions, a BDS0,5 without a usable altitude, idents of
    every FTC 1-4, velocities of every subtype, eps."""
    rng = np.random.default_rng(seed)
    ev = []
    craft = [0x1000 + 17 * k for k in range(6)]                 # small addresses: emulated tables may be small
    unknown = [0x6000 + k for k in range(8)]
    for j, aa in enumerate(craft):
        t, surface = float(rng.uniform(0, 1)), j % 2 == 1
        lat, lon = 51.0 + 0.3 * j, -0.5 + 0.2 * j
        while t < 150.0:
            kind = int(rng.integers(0, 10))
            if kind < 3:
                if rng.random() < 0.1:
                    surface = not surface                   # takes off / lands
                ev.append((t, *position(aa, lat, lon, int(rng.integers(0, 2)), surface, alt=int(rng.integers(0, 1600)) * 25,
                                        gillham=rng.random() < 0.1, rng=rng)))
            elif kind == 3:
                ev.append((t, *velocity(aa, int(rng.integers(0, 8)), rng)))
            elif kind == 4:
                ev.append((t, *ident(aa, int(rng.integers(1, 5)), "TRK%03dX" % int(rng.integers(0, 1000)))))
            elif kind == 5:
                ev.append((t, *eps(aa, int(rng.integers(0, 8)))))
            elif kind == 6:
                ev.append((t, *reply(int(rng.choice([0, 4, 20])), aa, rng, alt=int(rng.integers(0, 1600)) * 25)))
            elif kind == 7:
                ev.append((t, *reply(int(rng.choice([5, 21])), aa, rng)))
            elif kind == 8:
                ev.append((t, *reply(int(rng.choice([0, 4, 5, 20, 21])), int(rng.choice(unknown)), rng)))
            else:
                b = dc.Bits(32).put(1, 5, 11).put(6, 3, 5).put(9, 24, aa)
                ev.append((t, *dc.finish(b.bytes(), 0)))
            lat += 1e-3
            t += float(rng.choice([0.0, 0.2, 0.7, 1.5]))
            if j % 3 == 0 and rng.random() < 0.02:          # a silence longer than S: a reply or a DF11 comes back first
                t += S + float(rng.uniform(0.5, 10))
                ev.append((t, *reply(int(rng.choice([0, 4, 5, 20, 21])), aa, rng, alt=5000 if rng.random() < 0.5 else None)))
                b = dc.Bits(32).put(1, 5, 11).put(6, 3, 5).put(9, 24, aa)
                ev.append((t + 0.1, *dc.finish(b.bytes(), 0)))
                t += 0.5
            elif j == 1 and rng.random() < 0.02:            # a silence of exactly S: the row is still alive
                t += S
    return _msgs(ev)


def bucket_scene(n_aircraft=32, seed=9):
    """n_aircraft addresses sharing one bucket of the partition (local_cpr_cases.same_bucket_addresses), their position
    squitters from local_cpr_cases.bucket_scene (with its 40 s silence), plus idents, velocities and replies."""
    rng = np.random.default_rng(seed)
    base = lc.bucket_scene(n_aircraft=n_aircraft, n=3000, seed=seed)
    addrs = lc.same_bucket_addresses(n_aircraft)
    ev = [(float(s) + float(f), bytes.fromhex(h), ecc) for h, ecc, s, f in base]
    t_end = ev[-1][0]
    for _ in range(800):
        t = float(rng.uniform(0, t_end))
        aa = int(rng.choice(addrs))
        k = int(rng.integers(0, 4))
        if k == 0:
            ev.append((t, *ident(aa, int(rng.integers(1, 5)), "B%05d" % aa)))
        elif k == 1:
            ev.append((t, *velocity(aa, int(rng.integers(0, 4)), rng)))
        else:
            ev.append((t, *reply(int(rng.choice([0, 4, 5, 20, 21])), aa, rng, alt=12000 if k == 2 else None)))
    return _msgs(ev)


def burst_scene(seed=4, S=3):
    """One address with far more than 32 records back to back (so one 32-lane step holds only it), its row expiring and
    being recreated inside a step, non-DF17 replies landing in the gaps; a second address now and then."""
    rng = np.random.default_rng(seed)
    aa, bb = 0x2BCD, 0x2BCE
    ev, t = [], 10.0
    for k in range(150):
        r = rng.random()
        if k % 37 == 20:
            t += S + 1.0                                    # silence: the next records find the row expired
            ev.append((t, *reply(int(rng.choice([4, 5, 21])), aa, rng, alt=3000 if rng.random() < 0.5 else None)))
            t += 0.01
        if r < 0.3:
            ev.append((t, *position(aa, 40.0 + 1e-4 * k, 3.0, k % 2, k % 11 < 3, rng=rng)))
        elif r < 0.45:
            ev.append((t, *velocity(aa, int(rng.integers(0, 4)), rng)))
        elif r < 0.55:
            ev.append((t, *ident(aa, int(rng.integers(1, 5)), "BURST%02d" % (k % 100))))
        elif r < 0.8:
            ev.append((t, *reply(int(rng.choice([0, 4, 5, 20, 21])), aa, rng, alt=int(rng.integers(0, 400)) * 25)))
        else:
            ev.append((t, *eps(aa, int(rng.integers(0, 8)))))
        if k % 50 == 49:
            ev.append((t, *ident(bb, 4, "OTHER")))
        t += float(rng.choice([0.0, 0.001, 0.01]))
    return _msgs(ev)


def fleet_scene(n_aircraft=2000, seconds=600.0, seed=17, rate=0.5):
    """n_aircraft aircraft over `seconds`, each heard `rate` times per second on average (positions, velocities, idents,
    replies), arriving and leaving at random times."""
    rng = np.random.default_rng(seed)
    addrs = rng.choice(np.arange(1, 1 << 24), n_aircraft, replace=False)
    ev = []
    for aa in addrs:
        aa = int(aa)
        t0 = float(rng.uniform(0, seconds))
        t1 = min(seconds, t0 + float(rng.uniform(30, 400)))
        m = int(rng.poisson(rate * (t1 - t0)))
        lat, lon = float(rng.uniform(-60, 60)), float(rng.uniform(-170, 170))
        for t in np.sort(rng.uniform(t0, t1, m)):
            k = int(rng.integers(0, 8))
            if k < 3:
                ev.append((float(t), *position(aa, lat, lon, k % 2, False, alt=20000)))
            elif k == 3:
                ev.append((float(t), *velocity(aa, 1, rng)))
            elif k == 4:
                ev.append((float(t), *ident(aa, 4, "F%06X" % aa)))
            else:
                ev.append((float(t), *reply(int(rng.choice([0, 4, 5, 20, 21])), aa, rng, alt=20000 if k == 5 else None)))
    return _msgs(ev)


def scenes():
    """(name, location or None, msgs, S) for the equality tests."""
    for kw, S in zip(dc.CASES, (10, 30, 600, 5)):
        loc, msgs = dc.make_case(**kw)
        yield "case%d" % kw["seed"], loc, msgs, S
    yield "life", [51.5, -0.2], life_scene(), 20
    yield "life_noloc", None, life_scene(seed=2), 20
    yield "bucket", [10.0, 20.0], bucket_scene(), 30
    yield "burst", None, burst_scene(), 3
    traj, _ = lc.trajectory_scene(3, n_aircraft=40, seconds=120.0, drop=0.8, surface_share=0.3)
    yield "traj", [48.0, 11.0], traj, 15
