"""Generates tests/golden/local_cpr_golden.json.gz (decoder option "local_cpr"). Run in the build container:

    python tests/golden/make_local_cpr_golden.py

Every case is pushed through the UNMODIFIED reference function python/cpr.py:cpr_resolve_local (imported where it
lies in the gr-air-modes tree, $AMB_REFERENCE_TREE, behind a stub `air_modes` package; nothing is copied). A case is
(reference lat, reference lon, encoded lat, encoded lon, format, surface) with the reference's answer (lat, lon). The
seeded cases cover both hemispheres, |lat| near 87, reference longitudes near +-180, neighbours of every NL transition
latitude, and surface and airborne encodings. Nothing in the output is hand-edited.
"""
import gzip
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from make_decode_golden import load_reference, unload_reference  # noqa: E402


def nl_transitions():
    """Latitudes where cpr.py's nl() steps down, by bisection on the decode oracle's nl (pinned to the reference's)."""
    from oracle import decode_oracle as do
    out = []
    for k in range(3, int(do.nl(0.0)) + 1):
        lo, hi = 0.0, 86.99
        while True:
            mid = lo + (hi - lo) / 2
            if not (lo < mid < hi):
                break
            if do.nl(mid) >= k:
                lo = mid
            else:
                hi = mid
        out.append(hi)
    return out


def make_cases(seed, n):
    """-> [(ref_lat, ref_lon, enclat, enclon, fmt, surface)] from a seeded mix of the regions named in the module doc."""
    import decode_cases as dc
    rng = np.random.default_rng(seed)
    trans = nl_transitions()
    cases = []
    for i in range(n):
        kind = i % 5
        surface = int(rng.random() < 0.4)
        fmt = int(rng.integers(0, 2))
        sign = 1.0 if rng.random() < 0.5 else -1.0
        if kind == 0:                                   # anywhere
            lat, lon = float(rng.uniform(-86, 86)), float(rng.uniform(-180, 180))
        elif kind == 1:                                 # near the poles' NL = 1 region
            lat, lon = sign * float(rng.uniform(86.0, 89.5)), float(rng.uniform(-180, 180))
        elif kind == 2:                                 # near the antimeridian
            lat, lon = float(rng.uniform(-80, 80)), sign * float(180.0 - rng.uniform(0, 0.3))
        else:                                           # next to an NL transition, either side
            lat = sign * (trans[int(rng.integers(0, len(trans)))] + float(rng.choice([-1, 1])) * 10.0 ** float(rng.uniform(-9, -2)))
            lon = float(rng.uniform(-180, 180))
        span = 0.05 if surface else 0.4                 # the aircraft moved this far (degrees) from its reference
        tlat = max(-89.9, min(89.9, lat + float(rng.uniform(-span, span))))
        tlon = lon + float(rng.uniform(-span, span))
        tlon = tlon - 360.0 if tlon > 180.0 else (tlon + 360.0 if tlon <= -180.0 else tlon)
        la, lo = dc.cpr_encode(tlat, tlon, fmt, bool(surface))
        cases.append((lat, lon, la, lo, fmt, surface))
    return cases


def run_reference(cases, mods=None):
    cpr = (mods or load_reference())[3]
    return [list(map(float, cpr.cpr_resolve_local([a, b], [c, d], f, s))) for a, b, c, d, f, s in cases]


def main():
    mods = load_reference()
    cases = make_cases(2024, 4000)
    got = run_reference(cases, mods)
    unload_reference()
    rows = [list(c) + g for c, g in zip(cases, got)]
    assert all(math.isfinite(x) for r in rows for x in r)
    path = os.path.join(HERE, "local_cpr_golden.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps({"seed": 2024, "cases": rows}, separators=(",", ":")).encode())
    print("wrote", path, os.path.getsize(path), "bytes,", len(rows), "cases")


if __name__ == "__main__":
    main()
