"""Multilateration cases: stations, aircraft and the frames K receivers would stamp, built directly as amb_frame records
(no IQ), with exact or sample-quantized stamps. TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from gr_air_modes_b200 import _lib, synth
from gr_air_modes_b200.mlat import SPEED_OF_LIGHT, llh2ecef

FRAME = np.dtype(_lib.Frame)
# the reference's self-test geometry (mlat.py:181-183)
SELFTEST_STATIONS = [(37.76225, -122.44254, 100.0), (37.680016, -121.772461, 100.0), (37.385844, -122.083082, 100.0),
                     (37.701207, -122.309418, 100.0)]
SELFTEST_PLANE = (37.617175, -122.400843, 8000.0)


def frame(payload: bytes, secs: int, frac: float, addr_overlay: int = 0, passed: int = 1):
    f = np.zeros((), FRAME)
    f["secs"], f["frac"], f["nbits"], f["passed"] = secs, frac, len(payload) * 8, passed
    f["df"] = payload[0] >> 3
    f["crc"] = addr_overlay
    d = np.zeros(14, np.uint8)
    d[: len(payload)] = np.frombuffer(payload, np.uint8)
    f["data"] = d
    return f


def payload(kind, addr, feet, rng):
    p = synth.mlat_frame(kind, addr, feet, rng)
    return p, (addr if kind != 17 else 0)


def random_geometry(rng, K, baseline_km):
    lat0, lon0 = rng.uniform(-60, 60), rng.uniform(-180, 180)
    st = []
    for _ in range(K):
        r, a = rng.uniform(0.1, 1.0) * baseline_km * 1e3 / 2, rng.uniform(0, 2 * math.pi)
        st.append((lat0 + r * math.cos(a) / 111e3, lon0 + r * math.sin(a) / (111e3 * math.cos(math.radians(lat0))),
                   rng.uniform(0, 500)))
    return st, (lat0, lon0)


def scene_frames(stations, plane_list, n_tx, rng, rate=None, t0=(1_700_000_000, 0.125), spacing=2e-3, kinds=(4, 20, 17),
                 drop=0.0):
    """Per station, the frames of n_tx transmissions (aircraft drawn from plane_list = [(addr, lat, lon, feet)]), in
    stream order. rate None: exact stamps; else stamps floored to the sample grid at `rate`. drop: chance that a station
    misses a frame. Returns (per-station frame arrays, truth list)."""
    S = [np.array(llh2ecef(*s)) for s in stations]
    per = [[] for _ in stations]
    truth = []
    for j in range(n_tx):
        addr, lat, lon, feet = plane_list[int(rng.integers(0, len(plane_list)))]
        kind = int(kinds[int(rng.integers(0, len(kinds)))])
        p = np.array(llh2ecef(lat, lon, feet * 0.3048))
        pl, ov = payload(kind, addr, feet, rng)
        T = 0.01 + j * spacing + rng.uniform(0, spacing / 4)
        truth.append({"payload": pl, "ecef": p, "T": T})
        for k, s in enumerate(S):
            if rng.random() < drop:
                continue
            t = T + float(np.linalg.norm(p - s)) / SPEED_OF_LIGHT
            if rate is not None:
                t = math.floor(t * rate + rng.uniform()) / rate
            frac = t0[1] + t
            per[k].append((t, frame(pl, t0[0] + int(frac), frac - int(frac), ov)))
    out = []
    for lst in per:
        lst.sort(key=lambda e: e[0])
        out.append(np.array([f for _, f in lst], FRAME) if lst else np.zeros(0, FRAME))
    return out, truth


def split(frames, t0, cuts):
    """Cut each station's frames at the times `cuts` (seconds after t0): per call, the frames with t <= cut (and
    end = the cut). Returns [(per-station arrays, end)] and the rest as a final flushed call."""
    calls, lo = [], [0] * len(frames)
    for c in list(cuts) + [None]:
        part = []
        for k, f in enumerate(frames):
            t = (f["secs"].astype(np.float64) - t0[0]) + f["frac"]
            hi = len(f) if c is None else int(np.searchsorted(t, c + t0[1], side="right"))
            part.append(f[lo[k]:hi])
            lo[k] = hi
        end = None if c is None else (t0[0] + int(t0[1] + c), (t0[1] + c) - int(t0[1] + c))
        calls.append((part, end))
    return calls
