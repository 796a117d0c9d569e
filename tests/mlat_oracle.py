"""CPU checker of the multilateration stage (include/airmodes_b200.h amb_mlat, DESIGN.md §8 "Multilateration"):
eligibility, grouping, completeness, carry and the solver, restated from the rules step by step in plain Python floats
(IEEE double, no contraction: the device code is compiled with -fmad=false). Only the libm functions (sin, cos, atan2)
may differ from the device's in the last bit, so positions agree within a tolerance while groups and statuses are the
same. TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from gr_air_modes_b200 import _lib
from gr_air_modes_b200.mlat import SPEED_OF_LIGHT as CC, WGS84_A as A, WGS84_B as B, WGS84_E2 as E2

SOLVED, NO_CONVERGENCE, DEGENERATE = _lib.MLAT_SOLVED, _lib.MLAT_NO_CONVERGENCE, _lib.MLAT_DEGENERATE
MAX_STEPS, STOP, RCOND = 25, 1e-3, 1e-9
FRAME_DTYPE = np.dtype(_lib.Frame)


# ---- eligibility (amb_mlat_eligible) ----------------------------------------------------------------------------
def gray2bin(g):
    i = g >> 1
    while i:
        g ^= i
        i >>= 1
    return g


def decode_alt(alt, bit13):
    """altitude.py decode_alt: feet, or None for a metric altitude."""
    if (alt & 0x40) and bit13:
        return None
    if alt & 0x10:
        t = (((alt & 0x3F80) >> 2) | ((alt & 0x20) >> 1)) if bit13 else ((alt & 0x1FE0) >> 1)
        return ((alt & 0x0F) | t) * 25 - 1000
    if not bit13:
        alt = (alt & 0x3F) | (alt & (0x0FC0 << 1))
    big = (((alt & 0x0002) >> 1) + ((alt & 0x0008) >> 2) + ((alt & 0x0020) >> 3) + ((alt & 0x0080) >> 4) +
           ((alt & 0x0200) >> 5) + ((alt & 0x0800) >> 6) + ((alt & 0x0001) << 6) + ((alt & 0x0004) << 5))
    d = gray2bin(big)
    c = gray2bin(((alt & 0x0100) >> 8) + ((alt & 0x0400) >> 9) + ((alt & 0x1000) >> 10))
    if c == 7:
        c = 5
    if d % 2:
        c = 6 - c
    return d * 500 + c * 100 - 1300


def eligible(f):
    """(df, addr, feet) of an eligible frame (a row of np.dtype(Frame)), else None."""
    if not f["passed"]:
        return None
    nbits = int(f["nbits"])
    data = bytes(f["data"][: nbits // 8])
    v = int.from_bytes(data, "big")

    def bits(s, n):                                  # message bits s .. s+n-1, 1-based
        if s + n - 1 > nbits:
            return 0
        return (v >> (nbits - (s + n - 1))) & ((1 << n) - 1)
    df = bits(1, 5)
    if df in (0, 4, 16, 20):
        code, bit13, addr = bits(20, 13), 1, int(f["crc"])
    elif df == 17:
        tc = bits(33, 5)
        if not 9 <= tc <= 18:
            return None
        code, bit13, addr = bits(41, 12), 0, bits(9, 24)
    else:
        return None
    if code == 0:
        return None
    feet = decode_alt(code, bit13)
    return None if feet is None else (df, addr, feet)


# ---- geodesy ------------------------------------------------------------------------------------------------------
def station(lat_deg, lon_deg, h):
    """(ECEF, n, cl, sl, co, so) as amb_mlat_create computes it on the host."""
    la, lo = lat_deg * (math.pi / 180.0), lon_deg * (math.pi / 180.0)
    sl, cl, so, co = math.sin(la), math.cos(la), math.sin(lo), math.cos(lo)
    n = A / math.sqrt(1 - E2 * (sl * sl))
    s = ((n + h) * cl * co, (n + h) * cl * so, (n * (1 - E2) + h) * sl)
    return {"s": s, "n": n, "cl": cl, "sl": sl, "co": co, "so": so}


def norm3(a, b, c):
    return math.sqrt(a * a + b * b + c * c)


def ecef2llh_rad(x):
    ep = math.sqrt((A * A - B * B) / (B * B))
    p = math.sqrt(x[0] * x[0] + x[1] * x[1])
    th = math.atan2(A * x[2], B * p)
    lon = math.atan2(x[1], x[0])
    st, ct = math.sin(th), math.cos(th)
    lat = math.atan2(x[2] + ep * ep * B * (st * st * st), p - E2 * A * (ct * ct * ct))
    sl = math.sin(lat)
    n = A / math.sqrt(1 - E2 * (sl * sl))
    return lat, lon, p / math.cos(lat) - n


def default_window(stations):
    S = [station(*s)["s"] for s in stations]
    dmax = 0.0
    for i in range(len(S)):
        for j in range(i + 1, len(S)):
            d = norm3(S[i][0] - S[j][0], S[i][1] - S[j][1], S[i][2] - S[j][2])
            dmax = d if d > dmax else dmax
    return dmax / CC + 2e-6


# ---- solver (amb_mlat_rows / amb_mlat_qr / amb_mlat_solve_group) ----------------------------------------------------
def rows(x, sta, mask, r, dt, h):
    J, f = [], []
    sr = sta[r]["s"]
    er = (x[0] - sr[0], x[1] - sr[1], x[2] - sr[2])
    dr = norm3(*er)
    for k in range(32):
        if not (mask >> k) & 1 or k == r:
            continue
        si = sta[k]["s"]
        e = (x[0] - si[0], x[1] - si[1], x[2] - si[2])
        di = norm3(*e)
        f.append((di - dr) - CC * dt[k])
        J.append([e[0] / di - er[0] / dr, e[1] / di - er[1] / dr, e[2] / di - er[2] / dr])
    lat, _, _ = ecef2llh_rad(x)
    sl, cl = math.sin(lat), math.cos(lat)
    nn = A / math.sqrt(1 - E2 * (sl * sl))
    q, z = (nn + h) * cl, (nn * (1 - E2) + h) * sl
    rho = math.sqrt(q * q + z * z)
    nx = norm3(*x)
    f.append(nx - rho)
    J.append([x[0] / nx, x[1] / nx, x[2] / nx])
    return J, f


def qr(Am, b):
    """Householder QR in place, as amb_mlat_qr; returns True when R is degenerate."""
    n = len(Am)
    for j in range(3):
        s = 0.0
        for i in range(j, n):
            s += Am[i][j] * Am[i][j]
        nrm = math.sqrt(s)
        alpha = -nrm if Am[j][j] > 0.0 else nrm
        vj = Am[j][j] - alpha
        vtv = vj * vj
        for i in range(j + 1, n):
            vtv += Am[i][j] * Am[i][j]
        if vtv > 0.0:
            for k in range(j + 1, 4):
                col = (lambda i: Am[i][k]) if k < 3 else (lambda i: b[i])
                dot = vj * col(j)
                for i in range(j + 1, n):
                    dot += Am[i][j] * col(i)
                tau = (dot + dot) / vtv
                if k < 3:
                    Am[j][k] -= tau * vj
                    for i in range(j + 1, n):
                        Am[i][k] -= tau * Am[i][j]
                else:
                    b[j] -= tau * vj
                    for i in range(j + 1, n):
                        b[i] -= tau * Am[i][j]
        Am[j][j] = alpha
    r = [abs(Am[0][0]), abs(Am[1][1]), abs(Am[2][2])]
    mx = r[0] if r[0] > r[1] else r[1]
    mx = mx if mx > r[2] else r[2]
    if not mx > 0.0:
        return True
    lim = RCOND * mx
    return any(not (v >= lim) for v in r)


def solve(sta, mask, r, dt, h, trace=None):
    """Returns dict(status, steps, x, rms, dop); trace (a list) gets |dx| of every step."""
    o = sta[r]
    x = [(o["n"] + h) * o["cl"] * o["co"], (o["n"] + h) * o["cl"] * o["so"], (o["n"] * (1 - E2) + h) * o["sl"]]
    status, steps = NO_CONVERGENCE, MAX_STEPS
    for it in range(1, MAX_STEPS + 1):
        J, f = rows(x, sta, mask, r, dt, h)
        f = [-v for v in f]
        if qr(J, f):
            status, steps = DEGENERATE, it - 1
            break
        d2 = f[2] / J[2][2]
        d1 = (f[1] - J[1][2] * d2) / J[1][1]
        d0 = (f[0] - J[0][1] * d1 - J[0][2] * d2) / J[0][0]
        x = [x[0] + d0, x[1] + d1, x[2] + d2]
        nd = norm3(d0, d1, d2)
        if trace is not None:
            trace.append(nd)
        if nd <= STOP:
            status, steps = SOLVED, it
            break
    J, f = rows(x, sta, mask, r, dt, h)
    ss = 0.0
    for v in f:
        ss += v * v
    rms = math.sqrt(ss / len(f))
    if qr(J, f):
        dop = float("nan")
    else:
        u00, u11, u22 = 1.0 / J[0][0], 1.0 / J[1][1], 1.0 / J[2][2]
        u01 = -(J[0][1] * u11) / J[0][0]
        u12 = -(J[1][2] * u22) / J[1][1]
        u02 = -(J[0][1] * u12 + J[0][2] * u22) / J[0][0]
        dop = math.sqrt(u00 * u00 + u01 * u01 + u02 * u02 + u11 * u11 + u12 * u12 + u22 * u22)
    return {"status": status, "steps": steps, "x": x, "rms": rms, "dop": dop}


# ---- grouping (the stateful checker) --------------------------------------------------------------------------------
def diff(a, b):
    """d(a, b) for (secs, frac) pairs."""
    ds = (int(a[0]) - int(b[0]) + (1 << 63)) % (1 << 64) - (1 << 63)     # (int64)(uint64 difference)
    return float(ds) + (a[1] - b[1])


class Checker:
    """The stage's rules over calls: process(frames_per_station, end, flush) -> list of fix dicts (the fields of
    amb_mlat_fix plus "margin": the smallest | |dx| - 1e-3 | over the steps, for the step-count tolerance)."""

    def __init__(self, stations, window_us=None, offsets=None):
        self.K = len(stations)
        self.sta = [station(*s) for s in stations]
        self.W = default_window(stations) if window_us is None else window_us / 1e6
        self.off = list(offsets or [0.0] * self.K)
        self.carry = []
        self.counts = dict(eligible=0, carried=0, solved=0, no_convergence=0, degenerate=0, too_few=0, duplicate=0,
                           span=0)

    def items(self, frames_per_station):
        out = []
        for k, frames in enumerate(frames_per_station):
            arr = np.frombuffer(bytes(frames), FRAME_DTYPE) if not isinstance(frames, np.ndarray) else frames
            for f in arr:
                e = eligible(f)
                if e is None:
                    continue
                nbits = int(f["nbits"])
                payload = bytes(f["data"][: nbits // 8]) + bytes(14 - nbits // 8)
                out.append({"t": (int(f["secs"]), float(f["frac"]) - self.off[k]), "station": k, "nbits": nbits,
                            "data": payload, "df": e[0], "addr": e[1], "alt": e[2]})
        return out

    @staticmethod
    def _tkey(it):
        return it["t"], it["station"]

    def process(self, frames_per_station, end=(0, 0.0), flush=False):
        new = self.items(frames_per_station)
        self.counts["eligible"] += len(new)
        allit = self.carry + new
        # time order (t by the sign of d, ties by station; carried before new at equal (t, station))
        import functools

        def cmp(a, b):
            d = diff(a[1]["t"], b[1]["t"])
            if d != 0.0:
                return -1 if d < 0 else 1
            if a[1]["station"] != b[1]["station"]:
                return a[1]["station"] - b[1]["station"]
            return a[0] - b[0]
        order = sorted(enumerate(allit), key=functools.cmp_to_key(cmp))
        by_payload = {}
        for rank, (_, it) in enumerate(order):
            it["rank"] = rank
            by_payload.setdefault((it["nbits"], it["data"]), []).append(it)
        groups, carry = [], []
        for seq in by_payload.values():
            runs, cur = [], [seq[0]]
            for it in seq[1:]:
                if diff(it["t"], cur[-1]["t"]) <= self.W:
                    cur.append(it)
                else:
                    runs.append(cur)
                    cur = [it]
            runs.append(cur)
            for run in runs:
                first, last = run[0], run[-1]
                if not flush and not diff(end, last["t"]) >= self.W:
                    carry += run
                    continue
                st = [it["station"] for it in run]
                if len(set(st)) != len(st):
                    self.counts["duplicate"] += 1
                elif len(run) < 3:
                    self.counts["too_few"] += 1
                elif diff(last["t"], first["t"]) > self.W:
                    self.counts["span"] += 1
                else:
                    groups.append(run)
        groups.sort(key=lambda run: run[0]["rank"])
        carry.sort(key=lambda it: it["rank"])
        self.carry = [{k: v for k, v in it.items() if k != "rank"} for it in carry]
        self.counts["carried"] = len(self.carry)
        fixes = [self.fix(run) for run in groups]
        for fx in fixes:
            self.counts[{SOLVED: "solved", NO_CONVERGENCE: "no_convergence", DEGENERATE: "degenerate"}[fx["status"]]] += 1
        return fixes

    def fix(self, run):
        ref = run[0]
        r = ref["station"]
        dt, mask = [0.0] * 32, 0
        for it in run:
            dt[it["station"]] = diff(it["t"], ref["t"])
            mask |= 1 << it["station"]
        h = ref["alt"] * 0.3048
        trace = []
        s = solve(self.sta, mask, r, dt, h, trace)
        x = s["x"]
        sr = self.sta[r]["s"]
        secs, frac = ref["t"][0], ref["t"][1] - norm3(x[0] - sr[0], x[1] - sr[1], x[2] - sr[2]) / CC
        if math.isfinite(frac):
            while frac < 0.0:
                frac += 1.0
                secs -= 1
            while frac >= 1.0:
                frac -= 1.0
                secs += 1
        lat, lon, hh = ecef2llh_rad(x)
        return {"data": ref["data"], "nbits": ref["nbits"], "df": ref["df"], "addr": ref["addr"], "status": s["status"],
                "n": len(run), "steps": s["steps"], "ref": r, "stations": mask, "altitude": ref["alt"], "secs": secs,
                "frac": frac, "lat": lat * (180.0 / math.pi), "lon": lon * (180.0 / math.pi), "height": hh,
                "x": x[0], "y": x[1], "z": x[2], "rms": s["rms"], "dop": s["dop"],
                "margin": min((abs(v - STOP) for v in trace), default=float("inf"))}


def compare(got, want, tol=1e-6):
    """Device fixes (structured array) against the checker's: the same groups exactly and the same statuses; positions
    within tol m when the step counts agree; a count may differ by one only where the checker's |dx| came within 1e-9 m
    of the stopping limit. Returns a list of problems (empty when they agree)."""
    bad = []
    if len(got) != len(want):
        return ["%d fixes, checker %d" % (len(got), len(want))]
    for i, (g, w) in enumerate(zip(got, want)):
        same = (bytes(g["data"]) == w["data"] and int(g["nbits"]) == w["nbits"] and int(g["df"]) == w["df"] and
                int(g["addr"]) == w["addr"] and int(g["stations"]) == w["stations"] and int(g["ref"]) == w["ref"] and
                int(g["n"]) == w["n"] and int(g["altitude"]) == w["altitude"])
        if not same:
            bad.append("fix %d: a different group" % i)
            continue
        if int(g["status"]) != w["status"] and w["margin"] > 1e-9:
            bad.append("fix %d: status %d, checker %d" % (i, g["status"], w["status"]))
            continue
        if int(g["steps"]) == w["steps"]:
            d = norm3(g["x"] - w["x"], g["y"] - w["y"], g["z"] - w["z"])
            if w["status"] == SOLVED:
                if not d <= tol:
                    bad.append("fix %d: %.3g m from the checker" % (i, d))
                # the derived fields: degrees of 1e-9 are ~0.1 mm; a time of 1e-12 s is 0.3 mm of range
                close = {"lat": abs(g["lat"] - w["lat"]) <= 1e-9, "lon": abs(g["lon"] - w["lon"]) <= 1e-9,
                         "height": abs(g["height"] - w["height"]) <= 1e-5,
                         "emission": abs(diff((int(g["secs"]), float(g["frac"])), (w["secs"], w["frac"]))) <= 1e-12,
                         "rms": abs(g["rms"] - w["rms"]) <= 1e-6,
                         "dop": abs(g["dop"] - w["dop"]) <= 1e-6 * abs(w["dop"])}
                bad += ["fix %d: %s differs from the checker" % (i, k) for k, ok in close.items() if not ok]
        elif abs(int(g["steps"]) - w["steps"]) > 1 or w["margin"] > 1e-9:
            bad.append("fix %d: %d steps, checker %d (margin %.3g)" % (i, g["steps"], w["steps"], w["margin"]))
    return bad
