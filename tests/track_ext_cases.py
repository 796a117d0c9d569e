"""Seeded message sets for the decoder option "track_ext" (tests/test_track_ext_*.py, tools/track_ext_cost.py). Frames
come from the op-status, Comm-B and track scenes (tests/opstatus_cases.py, commb_cases.py, track_cases.py) and their
encoders; every generator returns messages (hex, ecc, secs, frac) in time order."""
from __future__ import annotations

import numpy as np

import commb_cases as cc
import decode_cases as dc
import local_cpr_cases as lc
import opstatus_cases as oc
import track_cases as tc


def _msgs(ev):
    ev.sort(key=lambda e: e[0])
    return [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc in ev]


def merge(*scenes):
    """Several message lists as one stream in time order."""
    return sorted([m for s in scenes for m in s], key=lambda m: m[2] + m[3])


def life(aa, t, rng, n=12, lat=48.0, lon=11.0, commb=True):
    """Events of one aircraft from t on: position pairs (so they get a fix), an op status, a target state and, with
    `commb`, a 4,0 / 5,0 / 6,0 reply each. Returns (events, the next free t)."""
    ev = []
    for k in range(n):
        ev.append((t, *tc.position(aa, lat + 1e-3 * k, lon, k % 2, False)))
        t += 0.1
        kind = k % 6
        if kind == 1:
            ev.append((t, *dc.df17(aa, oc.opstatus_me(0, 2, nica=1, nacp=int(rng.integers(0, 12))))))
        elif kind == 2:
            ev.append((t, *dc.df17(aa, oc.target_state_me(alt=int(rng.integers(1, 2000)), baro=int(rng.integers(1, 500)),
                                                          hdg_status=1, hdg=int(rng.integers(0, 512)), modes=0xC6))))
        elif commb and kind >= 3:
            reg = (0x40, 0x50, 0x60)[kind - 3]
            ev.append((t, *cc.reply(20 + k % 2, aa, cc.unique_word(reg, rng), rng)))
        t += 0.1
    return ev, t


def absence_scene(S=10, seed=1):
    """Rows that expire (silence longer than S) and are created again by a DF17 position, with op status, target
    state and Comm-B replies heard while the row was absent (they must not show in the new row), and more after it."""
    rng = np.random.default_rng(seed)
    ev = []
    for j, aa in enumerate((0x1100, 0x1101, 0x1102)):
        e, t = life(aa, 1.0 + j, rng)
        ev += e
        t += S + 2.0                                        # the row expires; groups written while it is absent
        ev.append((t, *dc.df17(aa, oc.opstatus_me(0, 1, nica=0, nacp=3))))
        ev.append((t + 0.1, *dc.df17(aa, oc.target_state_me(alt=7, baro=9, hdg_status=0, modes=0x02))))
        ev.append((t + 0.2, *cc.reply(20, aa, cc.unique_word(0x50, rng), rng)))
        t += 1.0
        e, _ = life(aa, t, rng, n=6 + 2 * j, commb=j != 1)  # created again; some groups written again, some not
        ev += e
    return _msgs(ev)


def age_edge(S2=30, now=100.5):
    """One aircraft whose op status lies exactly S2 before `now`, and whose target state lies 2^-40 s more than S2
    before it (so at `now` the first is shown and the second not); the row is alive at `now` with track >= 60."""
    rng = np.random.default_rng(3)
    aa = 0x1200
    ev, t = life(aa, now - S2 - 5.0, rng, n=6, commb=False)
    ev.append((now - S2, *dc.df17(aa, oc.opstatus_me(0, 2, nica=1, nacp=9))))
    ev.append((now - S2 - 2.0 ** -40, *dc.df17(aa, oc.target_state_me(alt=5, baro=5, hdg_status=1, hdg=3, modes=0x80))))
    for k in range(4):
        ev.append((now - 1.0 + 0.1 * k, *tc.position(aa, 48.1, 11.0, k % 2, False)))
    return _msgs(ev)


def burst_scene(seed=4):
    """One address with far more than 32 writers back to back (op status, target state, positions and Comm-B replies),
    so that one 32-lane step holds only it, and several writers of one group fall into one step."""
    rng = np.random.default_rng(seed)
    aa = 0x2BCD
    ev, t = [], 10.0
    for k in range(200):
        r = rng.random()
        if r < 0.3:
            ev.append((t, *tc.position(aa, 40.0 + 1e-4 * k, 3.0, k % 2, False)))
        elif r < 0.5:
            ev.append((t, *dc.df17(aa, oc.opstatus_me(int(rng.integers(0, 2)), int(rng.integers(0, 3)), nica=1,
                                                      nacp=int(rng.integers(0, 12))))))
        elif r < 0.65:
            ev.append((t, *dc.df17(aa, oc.target_state_me(alt=k + 1, baro=k + 1, hdg_status=1, hdg=k, modes=0xC0))))
        else:
            ev.append((t, *cc.reply(20 + k % 2, aa, cc.unique_word((0x40, 0x50, 0x60)[k % 3], rng), rng)))
        t += float(rng.choice([0.0, 0.001, 0.01]))
    return _msgs(ev)


def bucket_scene(seed=9):
    """32 addresses sharing one bucket of the partition (local_cpr_cases.same_bucket_addresses), each living through
    positions, op status, target state and Comm-B replies, interleaved."""
    rng = np.random.default_rng(seed)
    ev = []
    for j, aa in enumerate(lc.same_bucket_addresses(32)):
        e, _ = life(int(aa), 0.5 + 0.013 * j, rng, n=30)
        ev += e
    return _msgs(ev)


def scenes():
    """(name, msgs, S, S2) for the equality tests: the op-status, Comm-B and track scenes and the ones above."""
    yield "opstatus_table", oc.table_scene(), 60, 30
    yield "opstatus_bucket", oc.bucket_scene(), 30, 5
    yield "commb_reference", cc.reference_scene(S=30), 60, 30
    yield "commb_burst", cc.burst_scene(), 20, 3
    yield "track_life", merge(tc.life_scene(), oc.table_scene()), 20, 20
    yield "absence", absence_scene(), 10, 60
    yield "burst", burst_scene(), 20, 1
    yield "bucket", bucket_scene(), 30, 2


def fleet(n_aircraft=300, seconds=60.0):
    """The op-status fleet and the Comm-B fleet as one stream (for the stress test and the cost tool)."""
    ops, _ = oc.fleet_scene(n_aircraft=n_aircraft, seconds=seconds)
    com, _ = cc.fleet_scene(n_aircraft=n_aircraft, seconds=seconds)
    return merge(ops, com)
