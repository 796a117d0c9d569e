"""Multilateration on the CPU: the host and checker geodesy against the unmodified reference (tests/golden/
mlat_golden.json.gz, and live where the reference tree is present), the reference's self-test geometry with physical
stamps - where the reference's mlat() fails and the checker's solve lands within 1 mm - exact stamps on random
geometries, and the CLI's stamp arithmetic."""
import gzip
import json
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import mlat_oracle as mo  # noqa: E402
from gr_air_modes_b200 import mlat as ml  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "mlat_golden.json.gz")
REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python", "mlat.py")


@pytest.fixture(scope="module")
def golden():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def _dlon(a, b):
    d = abs(a - b) % 360.0
    return min(d, 360.0 - d)


def test_geodesy_equals_the_reference(golden):
    for g in golden["grid"]:
        e = ml.llh2ecef(*g["llh"])
        s = mo.station(*g["llh"])["s"]
        assert max(abs(a - b) for a, b in zip(e, g["ecef"])) <= 1e-6, g
        assert max(abs(a - b) for a, b in zip(s, g["ecef"])) <= 1e-6, g
        lat, lon, h = ml.ecef2llh(g["ecef"])
        la, lo, hh = mo.ecef2llh_rad(g["ecef"])
        want = g["llh_back"]
        for got in ((lat, lon, h), (la * (180.0 / math.pi), lo * (180.0 / math.pi), hh)):
            assert abs(got[0] - want[0]) <= 1e-10, (g, got)
            if abs(want[0]) < 89.99:              # longitude at a pole, and height through cos(lat) ~ 0, are not defined
                assert _dlon(got[1], want[1]) <= 1e-10, (g, got)
                assert abs(got[2] - want[2]) <= 1e-6, (g, got)


@pytest.mark.skipif(not os.path.exists(REF), reason="the reference tree is not present")
def test_geodesy_live_against_the_reference():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_mlat_golden
    m = make_mlat_golden.load_reference()
    rng = np.random.default_rng(4)
    for _ in range(2000):
        p = [rng.uniform(-89.9, 89.9), rng.uniform(-180, 180), rng.uniform(-500, 15000)]
        e = m.llh2ecef(list(p))
        assert max(abs(a - b) for a, b in zip(ml.llh2ecef(*p), e)) <= 1e-6
        back = ml.ecef2llh(e)
        want = m.ecef2llh(e)
        assert abs(back[0] - want[0]) <= 1e-10 and _dlon(back[1], want[1]) <= 1e-10 and abs(back[2] - want[2]) <= 1e-6


@pytest.mark.parametrize("k", [4, 3])
def test_selftest_geometry_with_physical_stamps(golden, k):
    """The reference's mlat() raises on this case (recorded in the golden); the stage's formulation solves it."""
    assert golden["selftest"]["raised"] and "converge" in golden["selftest"]["message"]
    st = [(s[0], s[1], s[2] + g) for s, g in zip(golden["stations"], golden["geoid"])][:k]    # on the ellipsoid
    sta = [mo.station(*s) for s in st]
    t = golden["stamps"][:k]
    r = min(range(k), key=lambda i: (t[i], i))
    dt = [ti - t[r] for ti in t] + [0.0] * (32 - k)
    s = mo.solve(sta, (1 << k) - 1, r, dt, golden["plane"][2])
    truth = ml.llh2ecef(*golden["plane"])
    assert s["status"] == mo.SOLVED
    assert math.dist(s["x"], truth) <= 1e-3


@pytest.mark.parametrize("seed", range(12))
def test_exact_stamps_on_random_geometries(seed):
    """3..8 stations, 20..300 km baselines, 0..45 000 ft, the aircraft over the network: every SOLVED fix within 1 cm.
    With three stations the two TDOAs and the altitude can meet twice; there the fix must be one of the exact points.
    (Far outside a lopsided network Gauss-Newton can settle in a minimum whose residual is kilometres; the fix's rms
    shows it.)"""
    rng = np.random.default_rng(100 + seed)
    K = int(rng.integers(3, 9))
    base = rng.uniform(20, 300)
    lat0, lon0 = rng.uniform(-60, 60), rng.uniform(-180, 180)
    kmlat, kmlon = 111.0, 111.0 * math.cos(math.radians(lat0))
    st = []
    for k in range(K):                                # around the network, so that the aircraft is inside it
        r, a = rng.uniform(0.3, 0.5) * base, 2 * math.pi * (k + rng.uniform(-0.3, 0.3)) / K
        st.append((lat0 + r * math.cos(a) / kmlat, lon0 + r * math.sin(a) / kmlon, rng.uniform(0, 800)))
    sta = [mo.station(*s) for s in st]
    for _ in range(20):
        h = rng.uniform(0, 45000) * 0.3048
        p = ml.llh2ecef(lat0 + rng.uniform(-0.2, 0.2) * base / kmlat, lon0 + rng.uniform(-0.2, 0.2) * base / kmlon, h)
        t = [math.dist(p, s["s"]) / mo.CC for s in sta]
        r = min(range(K), key=lambda i: (t[i], i))
        dt = [ti - t[r] for ti in t] + [0.0] * (32 - K)
        s = mo.solve(sta, (1 << K) - 1, r, dt, h)
        assert s["status"] == mo.SOLVED
        if K == 3:
            assert s["rms"] < 1e-3
        else:
            assert math.dist(s["x"], p) <= 1e-2, (K, base, math.dist(s["x"], p))


def test_cli_end_stamp_is_conservative():
    import mlat_b200 as cli
    assert cli.parse_start("1700000000.000000123") == (1700000000, 0.123e-6)
    assert cli.parse_station("37.5,-122.25,30,2.5e-7=x.cfile") == ((37.5, -122.25, 30.0), 2.5e-7, "x.cfile")
    rate, look = 4e6, 300
    for fed in (0, 100, 4_000_000, 12_345_678):
        secs, frac = cli.end_stamp((1_700_000_000, 0.75), fed, look, rate, 1e-6)
        assert 0.0 <= frac < 1.0
        # the stamp of the first sample the chain may still hold, less the offset, is not before end
        held = max(fed - look, 0)
        t_held = (1_700_000_000 + held // 4_000_000, 0.75 + (held % 4_000_000) / rate - 1e-6)
        assert mo.diff(t_held, (secs, frac)) >= -1e-12
