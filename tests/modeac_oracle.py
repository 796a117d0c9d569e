"""Checker of the Mode A/C reply rules (include/airmodes_b200.h, option "modeac"), written from the rules on the canonical
front end that the plain-C oracle port computes (oracle.cpu_oracle.Port.frontend). numpy, float32 exactly where the rules
are float; the whole stream at once, so it knows nothing of calls. Records are dicts with the amb_modeac fields (no stamp).
"""
import math

import numpy as np

NO_ALTITUDE = -(1 << 31)


def off(t_us: float, rate_int: int) -> int:
    return int(math.floor(t_us * rate_int / 1e6 + 0.5))


def geometry(rate_int: int) -> dict:
    return {"slot": [off(1.45 * k, rate_int) for k in range(15)],
            "gap": [off(1.45 * g + 0.725, rate_int) for g in range(14)],
            "spi": off(24.65, rate_int), "back": off(25.1, rate_int)}


def decode_id(v: int) -> int:                        # parse.py:233-254
    a = ((v & 0x0800) >> 11) + ((v & 0x0200) >> 8) + ((v & 0x0080) >> 5)
    b = ((v & 0x0020) >> 5) + ((v & 0x0008) >> 2) + ((v & 0x0002) << 1)
    c = ((v & 0x1000) >> 12) + ((v & 0x0400) >> 9) + ((v & 0x0100) >> 6)
    d = ((v & 0x0010) >> 2) + ((v & 0x0004) >> 1) + ((v & 0x0001) << 2)
    return a * 1000 + b * 100 + c * 10 + d


def _gray2bin(g: int) -> int:
    i = g >> 1
    while i:
        g ^= i
        i >>= 1
    return g


def gillham_feet(code: int) -> int:
    """altitude.py decode_alt(code, True) on its Gillham path (bit M = X = 0, bit Q = D1 = 0)."""
    alt = code
    big = (((alt & 0x0002) >> 1) + ((alt & 0x0008) >> 2) + ((alt & 0x0020) >> 3) + ((alt & 0x0080) >> 4) +
           ((alt & 0x0200) >> 5) + ((alt & 0x0800) >> 6) + ((alt & 0x0001) << 6) + ((alt & 0x0004) << 5))
    d = _gray2bin(big)
    c = _gray2bin(((alt & 0x0100) >> 8) + ((alt & 0x0400) >> 9) + ((alt & 0x1000) >> 10))
    if c == 7:
        c = 5
    if d % 2:
        c = 6 - c
    return d * 500 + c * 100 - 1300


def c_group(code: int) -> int:
    """C1 C2 C4 as a 3-bit number."""
    return ((code >> 10) & 4) | ((code >> 9) & 2) | ((code >> 8) & 1)


def altitude(code: int) -> int:
    if code & 0x10 or c_group(code) not in (1, 3, 2, 6, 4):
        return NO_ALTITUDE
    return gillham_feet(code)


def evaluate(bb, avg, rate_int: int, thr, lo: int = 0, hi: int | None = None) -> dict:
    """Per start i in [lo, hi): the masks of rules 1-2, 1-5, and the replies (1-7), plus code / spi / peak / floor arrays
    (index i - lo). Rule 7 only sees starts >= lo: exact for i >= lo + o(25.1), or everywhere when lo = 0."""
    G = geometry(rate_int)
    thr = np.float32(thr)
    hi = bb.size if hi is None else hi
    n = hi - lo
    pad = G["spi"] + 2
    avg = np.asarray(avg[lo:hi], np.float32)
    x = np.zeros(n + 1 + pad, np.float32)                                             # x[1 + s - lo] = in[s]
    a, b = max(lo - 1, 0), min(hi + pad, bb.size)
    x[a - lo + 1: b - lo + 1] = bb[a:b]

    def at(o):
        return x[1 + o: 1 + o + n]

    cur = at(0)
    lvl = avg * thr
    r1 = (cur > lvl) & (at(-1) < cur) & ~(at(1) > cur)
    f2 = at(G["slot"][14])
    r12 = r1 & ~(f2 < lvl)
    with np.errstate(all="ignore"):
        avgpeak = (cur + f2) / np.float32(2.0)
        space = avg + (avgpeak - avg) / thr
        clear = lvl * thr
    r15 = r12 & (cur > space) & (f2 > space) & (cur > clear) & (f2 > clear) & ~(at(G["slot"][7]) > space)   # rule 4
    for g in G["gap"]:
        r15 &= ~(at(g) > space)
    c = np.concatenate([[0], np.cumsum(r15.astype(np.int64))])
    idx = np.arange(n)
    earlier = c[idx] - c[np.maximum(idx - G["back"], 0)]                              # starts in [i - back, i) passing 1-5
    reply = r15 & (earlier == 0)
    code = np.zeros(n, np.int64)
    for k in range(1, 14):
        code |= (at(G["slot"][k]) > space).astype(np.int64) << (13 - k)
    spi = at(G["spi"]) > space
    return {"r12": r12, "r15": r15, "reply": reply, "drop": r15 & (earlier != 0), "code": code, "spi": spi,
            "peak": avgpeak, "floor": avg}


def replies(bb, avg, rate_int: int, thr, history: int, chunk: int = 1 << 22) -> list:
    """The records, in ascending sample_index (= sample + history - 1, the reported index frames use). Long streams are
    evaluated `chunk` starts at a time, each with the o(25.1) starts in front of it."""
    back = geometry(rate_int)["back"]
    out = []
    for a in range(0, bb.size, chunk):
        lo, hi = max(0, a - back), min(bb.size, a + chunk)
        ev = evaluate(bb, avg, rate_int, thr, lo, hi)
        for k in np.flatnonzero(ev["reply"][a - lo:]) + (a - lo):
            code = int(ev["code"][k])
            out.append({"sample_index": int(k) + lo + history - 1, "code": code, "spi": int(ev["spi"][k]),
                        "peak": np.float32(ev["peak"][k]), "floor": np.float32(ev["floor"][k]),
                        "squawk": decode_id(code), "altitude": altitude(code)})
    return out


def stats(bb, avg, rate_int: int, thr) -> dict:
    ev = evaluate(bb, avg, rate_int, thr)
    reps = np.flatnonzero(ev["reply"])
    return {"candidates": int(ev["r12"].sum()), "replies": int(reps.size), "overlap_drops": int(ev["drop"].sum()),
            "with_altitude": int(sum(altitude(int(ev["code"][s])) != NO_ALTITUDE for s in reps))}


def run_iq(port, iq, rate, thr_db, use_pmf=True, use_dcblock=False) -> list:
    """The replies of an interleaved float32 IQ stream through the canonical front end (and the DC blocker when on)."""
    from gr_air_modes_b200 import blocks
    g = blocks.query_geometry(rate, thr_db, use_pmf)
    iq = np.ascontiguousarray(iq, np.float32)
    if use_dcblock:
        iq = port.dc_blocker(iq, 100 * int(rate / 2e6))
    bb, avg = port.frontend(iq, rate, use_pmf)
    return replies(bb, avg, g.rate_int, g.threshold, g.history)


def same(got, want) -> bool:
    """Record for record, peak and floor bit for bit (got: a MODEAC_DTYPE array)."""
    if len(got) != len(want):
        return False
    for g, w in zip(got, want):
        if (int(g["sample_index"]), int(g["code"]), int(g["spi"]), int(g["squawk"]), int(g["altitude"])) != \
                (w["sample_index"], w["code"], w["spi"], w["squawk"], w["altitude"]):
            return False
        if np.float32(g["peak"]).tobytes() != w["peak"].tobytes() or np.float32(g["floor"]).tobytes() != w["floor"].tobytes():
            return False
    return True
