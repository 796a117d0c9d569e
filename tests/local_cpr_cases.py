"""Seeded message sets for the decoder option "local_cpr" (tests/test_local_cpr_*.py, tools/cpr_yield.py). Frames come
from tests/decode_cases.py's encoders; every generator returns messages (hex, ecc, secs, frac) in time order."""
from __future__ import annotations

import math

import numpy as np

import decode_cases as dc
from gr_air_modes_b200.synth import crc24


def local_bucket(icao: int) -> int:
    """The bucket of the local stage's partition (amb_v3_bucket of the ICAO key, amb_decode_v3.cuh)."""
    return (((icao * 2654435761) & 0xFFFFFFFF) * 1024) >> 32


def same_bucket_addresses(n: int, limit: int = 1 << 15):
    """n distinct addresses below `limit` that share one bucket of the local stage."""
    by = {}
    for a in range(1, limit):
        by.setdefault(local_bucket(a), []).append(a)
        if len(by[local_bucket(a)]) == n:
            return by[local_bucket(a)]
    raise ValueError("no bucket holds %d addresses below %d" % (n, limit))


def remap_addresses(msgs, limit: int = 1 << 15):
    """The DF17 squitters' addresses mapped one to one onto small ones (for tables of fewer than 2^24 slots); the
    parity keeps its syndrome, so the message token `ecc` is unchanged."""
    table, out = {}, []
    for h, ecc, s, f in msgs:
        raw = bytes.fromhex(h)
        if len(raw) == 14 and raw[0] >> 3 == 17:
            aa = int.from_bytes(raw[1:4], "big")
            new = table.setdefault(aa, len(table) + 1)
            assert new < limit
            body = raw[:1] + new.to_bytes(3, "big") + raw[4:11]
            par = int.from_bytes(raw[11:], "big") ^ crc24(raw[:11]) ^ crc24(body)
            raw = body + par.to_bytes(3, "big")
        out.append((raw.hex(), ecc, s, f))
    return out


def trajectory_scene(seed, n_aircraft=40, seconds=120.0, drop=0.0, location=(48.0, 11.0), surface_share=0.1,
                     small_addresses=False, other=True):
    """Aircraft on straight tracks around `location`, one position squitter every 0.4-0.6 s with the format chosen at
    random, velocity squitters in between. `drop` is the share of messages lost (weak signals); every third aircraft also
    fades out for 5-25 s. Some tracks start next to an NL transition latitude. Returns (msgs, truth): truth[k] is the
    sent (lat, lon) of a position message, else None."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lat0, lon0 = location if location is not None else (48.0, 11.0)
    pool = rng.choice(np.arange(1, 1 << 15), n_aircraft, replace=False) if small_addresses else \
        rng.choice(np.arange(1, 1 << 24), n_aircraft, replace=False)
    ev = []
    for a in range(n_aircraft):
        aa = int(pool[a])
        surface = rng.random() < surface_share
        lat = lat0 + rng.uniform(-2.0, 2.0) if not (a % 7 == 3) else 10.4704713 + rng.uniform(-2e-3, 2e-3)
        lon = lon0 + rng.uniform(-2.0, 2.0)
        speed = (rng.uniform(2e-5, 1e-4) if surface else rng.uniform(1.5e-3, 3e-3))     # degrees per second
        hdg = rng.uniform(0, 2 * math.pi)
        vlat, vlon = speed * math.cos(hdg), speed * math.sin(hdg) / max(0.2, math.cos(math.radians(lat)))
        alt = int(rng.integers(40, 1600)) * 25
        t = rng.uniform(0, 2.0)
        fade_at = rng.uniform(5, seconds) if a % 3 == 0 else 1e9
        fade_len = rng.uniform(5, 25)
        while t < seconds:
            plat, plon = lat + vlat * t, lon + vlon * t
            plon = (plon + 180.0) % 360.0 - 180.0
            odd = int(rng.integers(0, 2))
            heard = rng.random() >= drop and not (fade_at < t < fade_at + fade_len)
            if heard:
                la, lo = dc.cpr_encode(plat, plon, odd, surface)
                if surface:
                    me = dc.me_surface(int(rng.integers(5, 9)), 10, 1, int(rng.integers(0, 128)), odd, la, lo)
                else:
                    me = dc.me_airborne(11, dc.enc_alt12(alt), odd, la, lo)
                ev.append((t, *dc.df17(aa, me), (plat, plon)))
            if other and rng.random() < 0.3 and rng.random() >= drop:
                me = dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(15, 10, 300).put(26, 10, 200).put(38, 9, 10).v
                ev.append((t + 0.01, *dc.df17(aa, me), None))
            t += rng.uniform(0.4, 0.6)
    ev.sort(key=lambda e: e[0])
    msgs = [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc, _ in ev]
    return msgs, [e[3] for e in ev]


def chain_scene(n_local=80, seed=5):
    """One aircraft with an airborne even/odd pair (a global fix), then n_local surface reports with no receiver
    location (the global decode never resolves them: cpr.py:86-87), so every one of them chains on the previous
    local fix; a second aircraft interleaved now and then. Small addresses."""
    rng = np.random.default_rng(seed)
    aa, bb = 0x1234, 0x0777
    lat, lon = 47.45, 8.56
    msgs, t = [], 100.0
    for odd in (0, 1):
        la, lo = dc.cpr_encode(lat, lon, odd, False)
        fr, ecc = dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(1000), odd, la, lo))
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
        t += 0.3
    for k in range(n_local):
        lat += 2e-5
        lon += 3e-5
        odd = int(rng.integers(0, 2))
        la, lo = dc.cpr_encode(lat, lon, odd, True)
        fr, ecc = dc.df17(aa, dc.me_surface(7, 10, 1, 20, odd, la, lo))
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
        if k % 9 == 4:
            la, lo = dc.cpr_encode(46.0, 7.0, odd, False)
            fr, ecc = dc.df17(bb, dc.me_airborne(11, dc.enc_alt12(30000), odd, la, lo))
            msgs.append((fr.hex(), ecc, int(t), t - int(t) + 1e-4))
        t += float(rng.choice([0.0, 0.05, 0.3]))
    return msgs


def bucket_scene(n_aircraft=32, n=3000, seed=9):
    """n_aircraft aircraft whose addresses share one bucket of the local stage, airborne and surface, position
    squitters at random, both formats, timestamps that repeat; a 40 s silence in the middle (every reference expires)."""
    rng = np.random.default_rng(seed)
    craft = [(a, float(rng.uniform(-60, 60)), float(rng.uniform(-170, 170))) for a in same_bucket_addresses(n_aircraft)]
    msgs, t = [], 0.0
    for k in range(n):
        aa, lat, lon = craft[int(rng.integers(0, n_aircraft))]
        odd = int(rng.integers(0, 2))
        surface = rng.random() < 0.3
        la, lo = dc.cpr_encode(lat + 1e-3 * rng.standard_normal(), lon + 1e-3 * rng.standard_normal(), odd, surface)
        me = dc.me_surface(6, 10, 1, 5, odd, la, lo) if surface else dc.me_airborne(11, dc.enc_alt12(20000), odd, la, lo)
        fr, ecc = dc.df17(aa, me)
        t += float(rng.choice([0.0, 1e-4, 0.05, 1.0])) + (40.0 if k == n // 2 else 0.0)
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
    return msgs


def assert_records_match(got, want, where, tol=1e-12):
    """Product records (FIELDS_DTYPE) against the checker's dicts: integers, flags, strings and the local outcome
    exact, latitude/longitude bit for bit, the libm-based values (velocity/heading, range/bearing) to `tol` relative."""
    from gr_air_modes_b200 import decode
    assert len(got) == len(want), (where, len(got), len(want))
    for k, (rec, w) in enumerate(zip(got, want)):
        g = decode.record_to_dict(rec)
        assert (g["pad_"] & 0xFF) == w["local"] and (g["pad_"] >> 8) == 0, (where, k, g, w)
        for key, wv in w.items():
            if key == "local":
                continue
            gv = g[key]
            for a, b in (zip(gv, wv) if isinstance(wv, list) else [(gv, wv)]):
                if isinstance(b, float) and math.isnan(b):
                    assert math.isnan(a), (where, k, key, g, w)
                elif key in ("val", "range", "bearing"):
                    assert abs(a - b) <= tol * max(1.0, abs(b)), (where, k, key, g, w)
                else:
                    assert a == b, (where, k, key, g, w)
