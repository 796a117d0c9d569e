"""Records tests/golden/mlat_golden.json.gz from the UNMODIFIED reference module python/mlat.py, imported where it lies
in the gr-air-modes tree ($AMB_REFERENCE_TREE; nothing is copied). Current numpy has no `numpy.float`, which mlat.py's
geoid table names, so `numpy.float = float` is set before the import; nothing else is touched.

Recorded:
  grid      llh2ecef and ecef2llh over latitudes from pole to pole, longitudes across the antimeridian and heights
            from -500 to 15 000 m: (lat, lon, h) -> llh2ecef, and ecef2llh of that point
  geoid     wgs84_height at the self-test stations (mlat.py:181), so that the tests can place them on the ellipsoid
  selftest  the reference's mlat() on its own self-test geometry with physical stamps (t_i = T + |p - s_i| / c for
            every station, the first included): whether it raised, and its message

    python tests/golden/make_mlat_golden.py
"""
import gzip
import importlib.util
import json
import os

import numpy

REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mlat_golden.json.gz")
STATIONS = [[37.76225, -122.44254, 100], [37.680016, -121.772461, 100], [37.385844, -122.083082, 100],
            [37.701207, -122.309418, 100]]
PLANE = [37.617175, -122.400843, 8000]


def load_reference():
    if not hasattr(numpy, "float"):
        numpy.float = float
    spec = importlib.util.spec_from_file_location("ref_mlat", os.path.join(REF, "mlat.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def grid_points():
    pts = []
    for lat in (-90.0, -89.999, -60.5, -37.25, -1e-9, 0.0, 12.75, 45.0, 52.3, 89.999, 90.0):
        for lon in (-180.0, -179.999, -122.4, -0.5, 0.0, 4.25, 90.0, 179.999, 180.0):
            for h in (-500.0, 0.0, 100.0, 3000.0, 15000.0):
                pts.append([lat, lon, h])
    return pts


def main():
    m = load_reference()
    grid = []
    for p in grid_points():
        e = [float(v) for v in m.llh2ecef(list(p))]
        grid.append({"llh": p, "ecef": e, "llh_back": [float(v) for v in m.ecef2llh(e)]})
    geoid = [float(m.wgs84_height(s[0], s[1])) for s in STATIONS]
    # physical stamps: every station's stamp is T + range / c, the first one's too
    plane = numpy.array(m.llh2ecef(list(PLANE)))
    stamps = [10.0 + float(numpy.linalg.norm(plane - numpy.array(m.llh2geoid(list(s))))) / m.c for s in STATIONS]
    replies = [(list(s), t) for s, t in zip(STATIONS, stamps)]
    try:
        ans = m.mlat(replies, PLANE[2])
        selftest = {"raised": False, "answer": [float(v) for v in ans]}
    except Exception as exc:                          # the reference raises a bare Exception
        selftest = {"raised": True, "message": str(exc)}
    rec = {"grid": grid, "geoid": geoid, "stations": STATIONS, "plane": PLANE, "stamps": stamps,
           "selftest": selftest}
    with gzip.open(OUT, "wt") as f:
        json.dump(rec, f)
    print("wrote %s: %d grid points, selftest %s" % (OUT, len(grid), selftest))


if __name__ == "__main__":
    main()
