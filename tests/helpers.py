import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def load_golden():
    with open(os.path.join(HERE, "golden", "golden.json")) as f:
        meta = json.load(f)
    z = np.load(os.path.join(HERE, "golden", "scenes.npz"))
    scenes = []
    for s in meta["scenes"]:
        iq = z[s["name"]].astype(np.float32) / np.float32(2048.0)
        scenes.append((s, iq))
    return meta, scenes


def parse_msg(m):
    """'<hex> <crc> <ref> <secs> <frac>' (slicer_impl.cc:186-192, parse.py:425)."""
    data, crc, ref, secs, frac = m.split()
    return data, int(crc, 16), float(ref), int(secs), float(frac)


def first_four(bb, avg, rate, threshold_db, port):
    """Indices (reported coordinates) passing preamble_impl.cc:173-179, vectorised in float32."""
    p = port.params(rate, threshold_db)
    H = p.history - 1
    n = bb.size
    pad = 16 * int(np.ceil(p.spc)) + 8
    a = np.concatenate([np.zeros(H, np.float32), bb, np.zeros(pad, np.float32)])
    v = np.concatenate([np.zeros(H, np.float32), avg, np.zeros(pad, np.float32)])
    m = n + H
    thr = (v[:m] * np.float32(p.threshold)).astype(np.float32)
    ok = a[:m] > thr
    ok &= ~(a[1:m + 1] > a[:m])
    for k in (1, 2, 3):
        ok &= ~(a[p.po[k]:m + p.po[k]] < thr)
    return np.nonzero(ok)[0]


# ---- decision boundaries (tests/test_decision_edges_gpu.py, and the oracle pinned at the same points) -------------
# One rate per class of samples per chip: every integer spc 1..10 and a fractional one beside each (2.4 and 3 Msps
# both have spc_i 1). Together with PMF on and off they reach every instantiation of the scan, exact and slice kernels.
EDGE_RATES = (2e6, 2.4e6, 3e6, 4e6, 5e6, 6e6, 7e6, 8e6, 9e6, 10e6, 11e6, 12e6, 12.5e6, 14e6, 15e6, 16e6, 17e6, 18e6,
              19e6, 20e6)
EDGE_MATRIX = [(rate, pmf) for rate in EDGE_RATES for pmf in (True, False)]
EDGE_GRID = tuple(3.0 + 0.5 * k for k in range(21))      # coarse threshold grid (dB)
EDGE_CAP = 8                                               # knife edges kept per scene


def edge_scene(rate, pmf):
    """A small scene (15 k samples per Msps, <= 300 k) whose wide SNR spread puts bursts near every threshold."""
    from gr_air_modes_b200 import synth
    seed = 5000 + 2 * EDGE_RATES.index(rate) + int(pmf)
    return synth.make_scene(rate, int(15_000 * rate / 1e6), 10, seed, snr_db=(3.0, 14.0))


def _f32_bits(x):
    return int(np.array(x, np.float32).view(np.int32))


def _bits_f32(i):
    return float(np.array(i, np.int32).view(np.float32))


def knife_edges(port, bb, avg, rate, grid=EDGE_GRID, cap=EDGE_CAP):
    """Thresholds where the oracle's output (detection indices + messages) changes, each as two ADJACENT float32
    threshold_db values (lo, hi) with the change between them, found by bisecting the float32 bit pattern (monotone
    for positive floats) between neighbouring grid points that disagree. Kind "pulse": the reference's first four
    tests (preamble_impl.cc:173-179) differ between lo and hi; "quiet": they do not, so the quiet zone (:198-209) or
    the late gate decided. Returns (edges kept - at most `cap`, alternating kinds - and the number found)."""
    def out(t):
        r = port.run_streams(bb, avg, rate, t)
        return tuple(int(x) for x in r.index), tuple(r.msgs)

    outs = [out(t) for t in grid]
    found = []
    for k in range(len(grid) - 1):
        if outs[k] == outs[k + 1]:
            continue
        lo, hi = _f32_bits(grid[k]), _f32_bits(grid[k + 1])
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if out(_bits_f32(mid)) == outs[k]:
                lo = mid
            else:
                hi = mid
        tl, th = _bits_f32(lo), _bits_f32(hi)
        pulse = not np.array_equal(first_four(bb, avg, rate, tl, port), first_four(bb, avg, rate, th, port))
        found.append((tl, th, "pulse" if pulse else "quiet"))
    pulses = [e for e in found if e[2] == "pulse"]
    quiet = [e for e in found if e[2] == "quiet"]
    kept = []
    while len(kept) < cap and (pulses or quiet):
        for lst in (pulses, quiet):
            if lst and len(kept) < cap:
                kept.append(lst.pop(0))
    return sorted(kept), len(found)


def preamble_decisions(port, bb, avg, rate, threshold_db, index):
    """Replays preamble_impl.cc:172-209 in numpy for each detection in `index` (reported coordinates) and returns, per
    detection, what decided it: the candidate where the walk started, whether the peak test tied (in[i+1] == in[i]),
    how late the correlation walk went and whether it stopped on a tie (late_corr == now_corr), and the quiet zone's
    largest sample against space_threshold."""
    p = port.params(rate, threshold_db)
    H, spc, sps, thr = p.history - 1, float(p.spc), np.float32(p.sps), np.float32(p.threshold)
    k = int(spc)
    pad = 32 * (k + 1) + 64
    a = np.concatenate([np.zeros(H, np.float32), bb, np.zeros(pad, np.float32)])
    v = np.concatenate([np.zeros(H, np.float32), avg, np.zeros(pad, np.float32)])
    maxlate = 1
    while maxlate < spc:
        maxlate += 1
    qa = list(range(int(1.5 * float(sps)), int(np.floor(np.float32(3) * sps)) + 1))
    qb = list(range(int(np.float32(5) * sps), int(np.floor(7.5 * float(sps))) + 1))

    def corr(i):                                                  # correlate_preamble (:91-98), in double
        return sum(float(a[i + c * k + j]) for c in (0, 2, 7, 9) for j in range(k))

    ff = set(int(x) for x in first_four(bb, avg, rate, threshold_db, port))
    out = []
    for idx in (int(x) for x in index):
        start = None
        for s in range(idx - maxlate, idx + 1):
            if s not in ff:
                continue
            i, late = s, 0
            while True:
                now, nxt = corr(i), corr(i + 1)
                if nxt > now:
                    i += 1; late += 1
                if not (nxt > now and late < spc):
                    break
            if i == idx:
                start = (s, late, nxt == now)
                break
        assert start is not None, idx
        s, late, late_tie = start
        with np.errstate(all="ignore"):
            avgpeak = np.float32(np.float64(np.float32(np.float32(np.float32(a[idx] + a[idx + p.po[1]]) + a[idx + p.po[2]])
                                                       + a[idx + p.po[3]])) / 4.0)
            st = np.float32(v[idx] + np.float32(np.float32(avgpeak - v[idx]) / thr))
        quiet = max(a[idx + j] for j in qa + qb)
        out.append(dict(index=idx, start=s, peak_tie=bool(a[s + 1] == a[s]), late=late, maxlate=maxlate,
                        late_tie=bool(late_tie and late < spc), quiet_max=quiet, space_threshold=st))
    return out


def quiet_zone_tie(port, bb, avg, rate, idx, lo=3.0, hi=13.0):
    """The float32 threshold_db at which space_threshold (:203) of the detection at `idx` equals its quiet zone's largest
    sample exactly, or None: bisects on the bit pattern for the largest threshold that still accepts the preamble."""
    def state(t):                                                 # (space_threshold, quiet zone maximum) at idx
        p = port.params(rate, t)
        H, sps, thr = p.history - 1, np.float32(p.sps), np.float32(p.threshold)
        a = lambda j: np.float32(bb[idx + j - H])                 # noqa: E731 - reported coordinates -> bb
        qa = range(int(1.5 * float(sps)), int(np.floor(np.float32(3) * sps)) + 1)
        qb = range(int(np.float32(5) * sps), int(np.floor(7.5 * float(sps))) + 1)
        avgpeak = np.float32(np.float64(np.float32(np.float32(np.float32(a(0) + a(p.po[1])) + a(p.po[2])) + a(p.po[3])))
                             / 4.0)
        v = np.float32(avg[idx - H])
        return np.float32(v + np.float32(np.float32(avgpeak - v) / thr)), max(a(j) for j in list(qa) + list(qb))

    a, b = _f32_bits(lo), _f32_bits(hi)
    st, q = state(_bits_f32(a))
    if not st >= q:
        return None
    while b - a > 1:
        m = (a + b) // 2
        st, q = state(_bits_f32(m))
        if st >= q:
            a = m
        else:
            b = m
    st, q = state(_bits_f32(a))
    return _bits_f32(a) if st == q else None


class TieCase:
    def __init__(self, name, iq, rate, pmf, threshold_db):
        self.name, self.iq, self.rate, self.pmf, self.threshold_db = name, iq, rate, pmf, threshold_db


def flat_pulse_scene(rate, starts, seed):
    """Bursts of rectangular pulses on a 2^-11 grid (int16 IQ as tests/golden stores it) without noise: every plateau
    sample has the same |x|^2, so peak tests, correlations and PMF sums tie exactly."""
    from gr_air_modes_b200 import synth
    n = int(max(starts) + 300 * rate / 2e6) + 2000
    return synth.make_scene(rate, n, 0, seed, noise_sigma=0.0, starts=list(starts), amplitude=0.25,
                            quantize_bits=12).iq


def constructed_tie_cases(port):
    """Scenes where preamble_impl.cc's comparisons tie, each with the tie asserted on the oracle's own bb and avg:
    the peak test in[i+1] == in[i] (:175) and late_corr == now_corr (:188) at flat pulses, and a quiet-zone sample
    equal to space_threshold (:206, :208) at a threshold found by bisection, in int16-grid noise. PMF off (bb = |x|^2)
    and on (ascending sums of equal floats are exact). Returns (cases, {tie kind: PMF settings it was reached with})."""
    from gr_air_modes_b200 import synth
    cases = []
    seen = {"peak": set(), "late_tie": set(), "quiet": set()}
    for rate, starts in ((4e6, (3000.0, 9000.25, 15000.5)), (5e6, (3000.0, 9000.4, 15000.8)),
                         (9e6, (3000.0, 9000.5, 15000.25)), (12.5e6, (4000.0, 12000.6, 20000.3))):
        for pmf in (False, True):
            iq = flat_pulse_scene(rate, starts, int(rate // 1000) + pmf)
            bb, avg = port.frontend(iq, rate, pmf, 0)
            t = 7.0
            det = port.run_streams(bb, avg, rate, t).index
            assert len(det) > 0, (rate, pmf)
            for d in preamble_decisions(port, bb, avg, rate, t, det):
                if d["peak_tie"]:
                    seen["peak"].add(pmf)
                if d["late_tie"]:
                    seen["late_tie"].add(pmf)
            cases.append(TieCase("flat %g Msps pmf=%d" % (rate / 1e6, pmf), iq, rate, pmf, t))
    for rate in (5e6, 9e6, 12.5e6, 17e6, 19e6, 4e6):
        for pmf in (False, True):
            iq = synth.make_scene(rate, int(15_000 * rate / 1e6), 10, 77 + int(pmf), snr_db=(6.0, 20.0), quantize_bits=12).iq
            bb, avg = port.frontend(iq, rate, pmf, 0)
            det = port.run_streams(bb, avg, rate, 7.0).index
            name = "int16 noise %g Msps pmf=%d" % (rate / 1e6, pmf)
            for idx in (int(x) for x in det):
                tq = quiet_zone_tie(port, bb, avg, rate, idx)
                if tq is None or idx not in [int(x) for x in port.run_streams(bb, avg, rate, tq).index]:
                    continue
                d = preamble_decisions(port, bb, avg, rate, tq, [idx])[0]
                assert d["quiet_max"] == d["space_threshold"], (name, idx, tq)  # equal is still quiet: accepted
                seen["quiet"].add(pmf)
                cases.append(TieCase("%s quiet-zone tie at %d" % (name, idx), iq, rate, pmf, tq))
                break
    return cases, seen


# ---- llslicer limits (slicer_impl.cc:67-100) ---------------------------------------------------------------------
def slicer_ref_level(c0, c2, c7, c9):
    """reference_level of slicer_impl.cc:128-131: float adds left to right, the division by 4.0 in double."""
    f = np.float32
    with np.errstate(all="ignore"):
        return f(np.float64(f(f(f(c0) + f(c2)) + f(c7)) + f(c9)) / 4.0)


def slicer_limits(ref):
    """(highlimit, lowlimit, lowlimit*0.5) of llslicer: float = float * double rounds a double product (:71-72), and
    lowlimit * 0.5 is compared in double (:91, :94)."""
    with np.errstate(all="ignore"):
        hl = np.float32(np.float64(ref) * 1.414)
        ll = np.float32(np.float64(ref) * 0.707)
    return hl, ll, np.float64(ll) * 0.5


def _around(x):
    x = np.float32(x)
    return [np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))]


def single_constant_ref(const):
    """The first reference level from 1.0 upwards whose limit with the single-precision constant differs from the
    reference's double product, however the float constant is applied (float or double multiply)."""
    r = np.float32(1.0)
    c32 = np.float32(const)
    while True:
        want = np.float32(np.float64(r) * const)
        if want != np.float32(r * c32) and want != np.float32(np.float64(r) * np.float64(c32)):
            return r
        r = np.nextafter(r, np.float32(2.0))


def _encode(pre, pairs):
    c = np.zeros(240, np.float32)
    c[[0, 2, 7, 9]] = pre
    for j, (a, b) in enumerate(pairs):
        c[16 + 2 * j], c[17 + 2 * j] = a, b
    return c


def _frame_bits(frame):
    return [(frame[j // 8] >> (7 - j % 8)) & 1 for j in range(8 * len(frame))]


def slicer_edge_packets():
    """240-chip packets whose chips sit exactly on llslicer's limits and on the packet rules' boundaries. Returns
    (chips[n, 240] float32, facts) where facts records what the construction relies on, for the tests to assert."""
    from gr_air_modes_b200 import synth
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    one, zero = (np.float32(1.0), np.float32(0.0))
    hi_bit, lo_bit = (inf, -inf), (-inf, -inf)          # decision 1 / 0 with full confidence at every finite ref
    header16 = [hi_bit, lo_bit, lo_bit, lo_bit, lo_bit]  # DF16: long, no CRC or confidence rule applies (:140, :170-182)
    packets, facts = [], {}
    # reference levels: ordinary, negative, zero, denormal, huge, overflowing to inf, NaN, summation order, and the
    # two levels where a single-precision 1.414 / 0.707 gives another limit than the reference's double product
    r1414, r0707 = single_constant_ref(1.414), single_constant_ref(0.707)
    facts["ref_1414"], facts["ref_0707"] = float(r1414), float(r0707)
    pres = []
    for r in (1.0, 0.3, 1e-3, -0.5, 0.0, 2 ** -148, 1e-40, 1e30, r1414, r0707):
        r = np.float32(r)
        pres.append((r + r, zero, r + r, zero))                                   # ((2r + 0) + 2r) + 0 = 4r exactly
    pres.append((np.float32(-0.0),) * 4)
    pres.append((np.float32(3e38),) * 4)                                          # the sum overflows: ref = inf
    pres.append((nan, one, one, one))
    order = (np.float32(1e8), one, np.float32(-1e8), one)                         # ((1e8 + 1) - 1e8) + 1 = 1, not 2
    pres.append(order)
    facts["order_ref"] = float(slicer_ref_level(*order))
    for pre in pres:
        ref = slicer_ref_level(*pre)
        hl, ll, lh = slicer_limits(ref)
        vals = {}
        for v in _around(hl) + _around(ll) + _around(lh) + [zero, np.float32(-0.0), nan, inf, -inf, ref]:
            vals.setdefault(int(np.array(v, np.float32).view(np.uint32)), np.float32(v))
        vals = list(vals.values())
        pairs = [(a, b) for a in vals for b in vals]                             # every probe against every other
        for k in range(0, len(pairs), 20):                                       # <= 20 low-confidence bits: all recorded
            body = pairs[k:k + 20]
            packets.append(_encode(pre, header16 + body + [lo_bit] * (107 - len(body))))
    # packet rules: DF11 with 9 / 10 low-confidence bits (:171), short DF4 with 0 / 1 (:170); the deciding bit is a
    # '1' whose second chip sits on the three floats around lowlimit*0.5 (neither chip in the reference band)
    rng = np.random.default_rng(11)
    pre1 = (np.float32(2.0), zero, np.float32(2.0), zero)                        # ref = 1.0
    hl, ll, lh = slicer_limits(slicer_ref_level(*pre1))
    big = np.float32(3.0)                                                        # above highlimit
    for df, nlow in ((11, 9), (4, 0)):
        frame = synth.make_frame(df, rng)
        bits = _frame_bits(frame)
        ones = [j for j in range(5, 56) if bits[j]]
        lows = [j for j in range(5, 56) if j not in ones[-1:]][:nlow]
        for v in _around(lh):
            pairs = []
            for j, b in enumerate(bits):
                if j == ones[-1]:
                    pairs.append((big, v))                                       # low confidence unless v < lowlimit*0.5
                elif j in lows:
                    pairs.append((np.float32(1.2), one) if b else (one, np.float32(1.2)))   # both in band: low
                else:
                    pairs.append((one, zero) if b else (zero, one))
            packets.append(_encode(pre1, pairs + [lo_bit] * (112 - len(pairs))))
    # DF11 / DF17 / DF20 headers whose first '1' is decided at highlimit: (x, 1.0) is a '1' (both chips in band) for
    # x just below highlimit and a '0' at highlimit (first chip out of band), which turns the packet into DF3 / DF1 / DF4
    for df in (11, 17, 20):
        frame = synth.make_frame(df, rng)
        bits = _frame_bits(frame)
        first = bits.index(1)
        for x in _around(hl):
            pairs = [(x, one) if j == first else ((one, zero) if b else (zero, one)) for j, b in enumerate(bits)]
            packets.append(_encode(pre1, pairs + [lo_bit] * (112 - len(pairs))))
    return np.stack(packets).astype(np.float32), facts


# ---- field-decode parity (SURVEY.md 8 row f4) -----------------------------------------------------
def load_decode_golden():
    import gzip
    with gzip.open(os.path.join(HERE, "golden", "decode_golden.json.gz"), "rt") as f:
        return json.load(f)["cases"]


def compare_decode(rec, ref, tol=0.0, where="", tol_libm=None):
    """rec: one decoded record (dict with the members of struct amb_fields); ref: what the unmodified reference
    computed for the same message (tests/golden/make_decode_golden.py). Integers and strings must be equal.
    Latitude/longitude/ground track (+, -, *, /, floor, fmod only) are compared with relative tolerance `tol`
    (0 = bit-exact); velocity, heading, range and bearing go through hypot/atan2/sin/cos/pow, where CPython's own
    hypot and each libm differ in the last place: `tol_libm` (default = tol)."""
    import math
    NO_HANDLER, METRIC, NOPOS, STRADDLE, HASPOS, HASRNG = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20

    if tol_libm is None:
        tol_libm = tol

    def close(a, b, t=None):
        t = tol if t is None else t
        if b is None:
            return a is None or math.isnan(a)
        if t == 0.0:
            return a == b
        return abs(a - b) <= t * max(1.0, abs(b))

    st = rec["status"]
    if "dropped" in ref:
        assert st & NO_HANDLER, (where, rec, ref)
        return
    assert not (st & NO_HANDLER), (where, rec, ref)
    assert rec["df"] == ref["df"], (where, rec, ref)
    for k in ("vs", "ri", "sl", "fs", "ca", "icao", "squawk", "ftc", "cat", "eps", "tti", "ast", "subtype"):
        if k in ref:
            assert rec[k] == ref[k], (where, k, rec, ref)
    if "bds" in ref:
        assert rec["bds"] == ref["bds"], (where, rec, ref)
    if "metric_alt" in ref:
        assert st & METRIC, (where, rec, ref)
    elif "altitude" in ref:
        assert not (st & METRIC) and rec["altitude"] == ref["altitude"], (where, rec, ref)
    if "ident" in ref:
        assert rec["ident"] == ref["ident"], (where, rec, ref)
    if "aux" in ref:
        assert list(rec["aux"]) == ref["aux"], (where, rec, ref)
    if "ara" in ref:
        assert rec["aux"][0] == ref["ara"] and rec["aux"][1] == ref["rac"], (where, rec, ref)
        assert rec["aux"][2] == (ref["rat"] | (ref["mte"] << 1)), (where, rec, ref)
    if "tid" in ref:
        assert rec["aux"][3] == ref["tid"], (where, rec, ref)
    if "tidr" in ref:
        assert rec["aux"][3] == (ref["tidr"] | (ref["tidb"] << 8)) and rec["threat_alt"] == ref["threat_alt"], (where, rec, ref)
        assert not (st & 0x40), (where, rec, ref)
    if "threat_metric_alt" in ref:
        assert st & 0x40, (where, rec, ref)          # AMB_FS_METRIC_THREAT
    if "cpr" in ref:
        assert [rec["cpr_format"], rec["cpr_lat"], rec["cpr_lon"]] == ref["cpr"], (where, rec, ref)
    if "ground_track" in ref:
        assert close(rec["val"][0], ref["ground_track"]), (where, rec, ref)
    if "val" in ref:
        for a, b in zip(rec["val"], ref["val"]):
            assert close(a, b, tol_libm), (where, rec, ref)
    if ref.get("cpr_error") == "straddle":
        assert (st & STRADDLE) and (st & NOPOS) and not (st & HASPOS), (where, rec, ref)
    elif ref.get("cpr_error") == "nopos":
        assert (st & NOPOS) and not (st & (STRADDLE | HASPOS)), (where, rec, ref)
    elif "pos" in ref:
        lat, lon, rng, brg = ref["pos"]
        assert (st & HASPOS) and not (st & NOPOS), (where, rec, ref)
        assert close(rec["lat"], lat) and close(rec["lon"], lon), (where, rec, ref)
        if rng is None:
            assert not (st & HASRNG), (where, rec, ref)
        else:
            assert st & HASRNG, (where, rec, ref)
            assert close(rec["range"], rng, tol_libm) and close(rec["bearing"], brg, tol_libm), (where, rec, ref)
