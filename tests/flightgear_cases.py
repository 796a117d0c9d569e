"""Seeded message sets for the decoder option "flightgear" (tests/test_flightgear_*.py, tests/golden/
make_flightgear_golden.py): every BDS0,8 category row with every cat (the out-of-range one included), velocity
subtypes 0, 1 and 3, airborne and surface positions, callsigns and velocities that arrive after positions, and a
fleet of more aircraft than one call holds. Messages are (hex, ecc, secs, frac) in time order; addresses stay below
2^15 (the emulator's pairing table); tests/track_cases.py's frames_of() turns them into frames."""
from __future__ import annotations

import numpy as np

import decode_cases as dc
import sbs1_cases as sc
import track_cases as tc

T0 = 1_700_000_000
LOCATION = [47.9, 11.1]


def _velocity(aa, sub, rng):
    """BDS0,9 with ME subtype `sub` (1..4) and random words (the reference's subtypes 0 and 1, and 3 for sub 4)."""
    return sc.velocity(aa, sub, int(rng.integers(1, 1024)), int(rng.integers(1, 1024)), int(rng.integers(0, 2)),
                       int(rng.integers(0, 2)), int(rng.integers(0, 512)), int(rng.integers(0, 2)))


def _pos(aa, lat, lon, k, surface=False):
    return [tc.position(aa, lat, lon, 0, surface, alt=1000 + 25 * k), tc.position(aa, lat, lon, 1, surface, alt=1000 + 25 * k)]


def _msgs(ev):
    msgs, last = [], -1.0
    for t, (f, ecc) in sorted(ev, key=lambda e: e[0]):
        t = max(t, last + 1e-4)
        last = t
        secs = int(t)
        msgs.append((f.hex(), ecc, T0 + secs, t - secs))
    return msgs


def category_scene(seed=5):
    """One aircraft per (ftc, cat), 1..4 x 0..7: callsign, a velocity of each subtype, then positions; cat 7 of ftc 2
    (IndexError) never gets a callsign, so its positions write nothing."""
    rng = np.random.default_rng(seed)
    ev, t = [], 0.0
    for ftc in range(1, 5):
        for cat in range(8):
            aa = 0x100 + 8 * ftc + cat
            lat, lon = 47.5 + 0.05 * cat, 10.5 + 0.1 * ftc
            fr = [dc.df17(aa, dc.me_ident(ftc, cat, "C%dX%d" % (ftc, cat)))]
            for sub in (1, 2, 3, 4):
                fr.append(_velocity(aa, sub, rng))
                fr += _pos(aa, lat, lon, sub)
            for f in fr:
                t += float(rng.uniform(0.01, 0.2))
                ev.append((t, f))
    return _msgs(ev)


def late_scene(seed=6):
    """Positions before any callsign or velocity; then velocity only (subtype 3 alone, then 0 / 1); then the callsign;
    surface positions near the receiver; a second callsign and velocity that replace the first."""
    rng = np.random.default_rng(seed)
    ev, t = [], 0.0
    for j in range(12):
        aa = 0x2000 + 97 * j
        lat, lon = LOCATION[0] + 0.02 * (j - 6), LOCATION[1] + 0.03 * (j - 6)
        surface = j % 3 == 0
        steps = [_pos(aa, lat, lon, 0, surface), [_velocity(aa, 4, rng)], _pos(aa, lat, lon, 1, surface),
                 [_velocity(aa, 1 + j % 3, rng)], _pos(aa, lat, lon, 2, surface),
                 [dc.df17(aa, dc.me_ident(4, j % 8, "LATE%02d" % j))], _pos(aa, lat, lon, 3, surface),
                 [dc.df17(aa, dc.me_ident(3, (j + 3) % 8, "NEW%02d" % j)), _velocity(aa, 1 + (j + 1) % 3, rng)],
                 _pos(aa, lat + 0.01, lon, 4, surface)]
        for group in steps:
            for f in group:
                t += float(rng.uniform(0.01, 0.3))
                ev.append((t, f))
    return _msgs(ev)


def fleet_scene(n_aircraft=300, rounds=4, seed=7):
    """n_aircraft interleaved aircraft (more than a bucket's 32-record step and more than one call of the tests'
    cuts), each with a callsign, velocities and positions every round, in random order within the round."""
    rng = np.random.default_rng(seed)
    ev, t = [], 0.0
    for r in range(rounds):
        batch = []
        for j in range(n_aircraft):
            aa = 0x4000 + j * 13
            lat, lon = 46.0 + (j % 40) * 0.1, 9.0 + (j // 40) * 0.15
            batch += _pos(aa, lat + 0.001 * r, lon, r)
            if (j + r) % 3 == 0:
                batch.append(dc.df17(aa, dc.me_ident(1 + j % 4, int(rng.integers(0, 7)), "F%05d" % j)))
            if (j + r) % 2 == 0:
                batch.append(_velocity(aa, 1 + int(rng.integers(0, 4)), rng))
        for k in rng.permutation(len(batch)):
            t += 1e-3
            ev.append((t, batch[k]))
    return _msgs(ev)


def pole_scene(seed=8):
    """Aircraft far north at longitudes -90, 45 and -135 heading 270, 135 and 315 (subtype 0 words with equal or zero
    components): where the CPR fix lands on the longitude exactly, the product quaternion's w is exactly 0 for many
    latitudes, so _set_q's sign rule (q[3] > 0, not >= 0) decides the orientation's sign."""
    rng = np.random.default_rng(seed)
    ev, t = [], 0.0
    # (lon, ME subtype 1 words: vew, vns, dew, dns) for heading 270 (ns 0, ew < 0), 135 (ew > 0, ns < 0), 315
    for j, (lon, words) in enumerate(((-90.0, (101, 1, 1, 0)), (45.0, (101, 101, 0, 1)), (-135.0, (101, 101, 1, 0)))):
        for i, lat in enumerate(np.arange(77.0, 89.5, 0.31)):
            aa = 0x6000 + 64 * j + i
            fr = [dc.df17(aa, dc.me_ident(4, 5, "POLE%03d" % i)), sc.velocity(aa, 1, *words)]
            fr += _pos(aa, float(lat), lon, 0) + _pos(aa, float(lat), lon, 1)
            for f in fr:
                t += float(rng.uniform(0.01, 0.1))
                ev.append((t, f))
    return _msgs(ev)


def scenes():
    """(name, location, msgs) of the golden: the decode golden's cases and the FlightGear scenes."""
    for kw in dc.CASES:
        loc, msgs = dc.make_case(**kw)
        yield "decode_seed%d" % kw["seed"], loc, msgs
    yield "categories", LOCATION, category_scene()
    yield "late", LOCATION, late_scene()
    yield "fleet", LOCATION, fleet_scene()
    yield "pole", LOCATION, pole_scene()


# The packer grid (fg_posmsg.pack directly): (lat, lon, alt, heading). The poles and the date line, the four quadrant
# headings and the double just below 360, headings whose den ties (90, 270 and their neighbours), and the identity
# rotations the reference cannot pack (lat -90, lon 0, heading 0 / 360).
def grid():
    out = []
    lats = [-90.0, 90.0, 0.0, 45.25, -33.9]
    lons = [0.0, 180.0, -180.0, 11.1]
    hdgs = [0.0, 90.0, 180.0, 270.0, float(np.nextafter(360.0, 0.0)), 360.0, float(np.nextafter(90.0, 0.0)),
            float(np.nextafter(90.0, 180.0)), float(np.nextafter(270.0, 0.0)), float(np.nextafter(270.0, 360.0)), 1e-13]
    for lat in lats:
        for lon in lons:
            for h in hdgs:
                out.append((lat, lon, 1000, h))
    return out
