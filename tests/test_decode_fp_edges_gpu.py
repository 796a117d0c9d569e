"""The batch decoder's libm-derived fields over their whole input domain, and the decisions built on them at their ties.
Need an H100.

A. Velocity (parseBDS09_0 / _1, amb_decode_core.h amb_decode_fields): every 11-bit ns x 11-bit ew x both signs of
   subtype 0 (2^24 words) and every 10-bit ns x ew x signs of subtypes 1 and 2 (2 x 2^22 words), built as DF17 frames
   and decoded in batches of 2^20. The reference uses no device libm: the speed is the IEEE square root of the exact
   integer ns^2 + ew^2 (correctly rounded; the sum is below 2^26), the heading atan2 / atan in long double rounded once to
   double, followed by the decoder's own double operations. The speed must be bit-exact, so a perfect square gives
   exactly its integer root: the ties of the Comm-B speed rule. The heading must stay within HEADING_ULP of the correctly
   rounded value, and in [0, 360). Vertical rate and turn rate / geometric difference are bit-exact. Where the device
   differs from CPython's math.hypot / math.atan2 (oracle/decode_oracle.py, the reference's parser), the printed report
   line must be the same.
B. Range and bearing (amb_range_bearing) at their geometric edges, positions from real CPR pairs, global and local: the
   reference is the function restated operation by operation, each +, -, *, / in double as the device does it and each
   libm call in long double rounded once to double. The device must stay within RANGE_ULP / BEARING_ULP of it; bearing in
   [0, 360]; range exactly 0 at the receiver's own position; bearing bit-equal to CPython's where the receiver is due
   N/S/E/W (atan2 returns 0, +-pi/2 or +-pi in both libms); the report text equal to the text from CPython's values.
C. Comm-B decisions (amb_commb_agree): the checker tests/commb_oracle.py fed with CPython's velocities, not the
   decoder's own; Pythagorean ties of the +-20 kt speed rule decided RESOLVED at 2 GS - speed = +-20 and not at +-22;
   and the 10 deg track rule at every heading of A with the 5,0 tracks nearest 10 deg either side.
"""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import commb_cases as cc  # noqa: E402
import commb_oracle as co  # noqa: E402
import decode_cases as dc  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu

BATCH = 1 << 20
SPEED_ULP = 0            # bit-exact
HEADING_ULP = 2
RANGE_ULP = 2
BEARING_ULP = 1
CPYTHON_SHARE = 1 / 64   # of the records that differ from the correctly rounded values, decoded again in CPython
L = np.longdouble


def _ulps(got, want):
    """Distance in units in the last place of two arrays of finite doubles of the same sign."""
    return np.abs(np.asarray(got, np.float64).view(np.int64) - np.asarray(want, np.float64).view(np.int64))


def _hist(u, top=8):
    return _hist_of_counts(np.bincount(np.minimum(u, top), minlength=top + 1))


def _hist_of_counts(h):
    """{ulps: count} of a histogram whose last bin holds everything from there up."""
    top = len(h) - 1
    return {("%d" % k if k < top else ">=%d" % top): int(v) for k, v in enumerate(h) if v}


def _near_tie(x_ld, x):
    """Long-double values within 2^-8 ulp of the midpoint between two doubles: their rounding is not certain."""
    ulp = np.spacing(np.abs(x)).astype(L)
    r = np.abs((x_ld - x.astype(L)) / np.where(ulp > 0, ulp, 1))
    return (np.abs(r - 0.5) < 2.0 ** -8) & (x != 0)


# ---- DF17 frames built with numpy ----------------------------------------------------------------------------------
_CRC = None


def _crc_table():
    """Parity of an 11-byte DF17 body is the XOR of one entry per byte (the Mode S CRC is linear)."""
    global _CRC
    if _CRC is None:
        from gr_air_modes_b200.synth import crc24
        _CRC = np.zeros((11, 256), dtype=np.uint32)
        for i in range(11):
            for v in range(256):
                b = bytearray(11)
                b[i] = v
                _CRC[i, v] = crc24(bytes(b))
    return _CRC


def _df17_frames(me, icao):
    """Queued, CRC-clean DF17 frames (FRAME_DTYPE) carrying the 56-bit ME words `me` from addresses `icao`."""
    from gr_air_modes_b200 import decode
    n = len(me)
    body = np.zeros((n, 11), dtype=np.uint8)
    body[:, 0] = (17 << 3) | 5
    for i in range(3):
        body[:, 1 + i] = (icao >> (8 * (2 - i))) & 0xFF
    for i in range(7):
        body[:, 4 + i] = (me >> np.uint64(8 * (6 - i))) & np.uint64(0xFF)
    tab = _crc_table()
    par = np.zeros(n, dtype=np.uint32)
    for i in range(11):
        par ^= tab[i, body[:, i]]
    fr = np.zeros(n, dtype=decode.FRAME_DTYPE)
    fr["data"][:, :11] = body
    for i in range(3):
        fr["data"][:, 11 + i] = (par >> (8 * (2 - i))) & 0xFF
    k = np.arange(n)
    fr["secs"], fr["frac"] = k // 1000, (k % 1000) * 1e-3
    fr["nbits"], fr["df"], fr["passed"], fr["ref_level"] = 112, 17, 1, 0.5
    return fr


def _put(v, first, width):
    """Field at ME bits first..first+width-1 (1-based from the MSB)."""
    return np.asarray(v, dtype=np.uint64) << np.uint64(57 - first - width)


def test_df17_frames_match_the_bitwise_encoder():
    me = np.array([0x99_1234_5678_9ABC, 0x58_C382_D690_C8AC], dtype=np.uint64)
    fr = _df17_frames(me, np.array([0x4840D6, 0xABCDEF]))
    for k, (m, a) in enumerate(((0x99_1234_5678_9ABC, 0x4840D6), (0x58_C382_D690_C8AC, 0xABCDEF))):
        assert bytes(fr["data"][k]) == dc.df17(a, m)[0]


# ---- A: velocity ---------------------------------------------------------------------------------------------------
def _velocity_batch(sub, idx, rng):
    """ME words of subtype `sub` for the (ns, ew, signs) indices `idx`, the other fields random, and the reference
    record values: speed, heading (correctly rounded libm), vs, tr / geo, plus the near-tie flags of the long-double
    libm values."""
    n = len(idx)
    r = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    rb = lambda sh, w: (r >> np.uint64(sh)) & np.uint64((1 << w) - 1)          # noqa: E731
    me = _put(19, 1, 5) | _put(sub, 6, 3)
    if sub == 0:
        ew_f, ns_f, se, sn = idx & 0x7FF, (idx >> 11) & 0x7FF, (idx >> 22) & 1, (idx >> 23) & 1
        tr_s, tr_f, vs_s, vs_f = rb(0, 1), rb(1, 6), rb(7, 1), rb(8, 9)
        me |= _put(rb(17, 1), 9, 1) | _put(se, 10, 1) | _put(ew_f, 11, 11) | _put(sn, 22, 1) | _put(ns_f, 23, 11)
        me |= _put(tr_s, 34, 1) | _put(tr_f, 35, 6) | _put(vs_s, 41, 1) | _put(vs_f, 42, 9) | _put(rb(18, 6), 51, 6)
        ns, ew = ns_f.astype(np.int64) - 1, ew_f.astype(np.int64) - 1
        speed = np.sqrt((ns * ns + ew * ew).astype(np.float64))
        ews, nss = np.where(se == 1, -ew, ew), np.where(sn == 1, -ns, ns)
        a_ld = np.arctan2(ews.astype(L), nss.astype(L))
        a = a_ld.astype(np.float64)
        hdg = a * (180.0 / math.pi)
        hdg = np.where(hdg < 0, hdg + 360, hdg)
        vs = (vs_f.astype(np.int64) * 32) * np.where(vs_s == 1, -1, 1)
        tr = (tr_f.astype(np.int64) * 15).astype(np.float64) / 62
        tr = np.where(tr_s == 1, 0 - tr, tr)
        v2, v3 = vs.astype(np.float64), tr
    else:
        ew_f, ns_f, se, sn = idx & 0x3FF, (idx >> 10) & 0x3FF, (idx >> 20) & 1, (idx >> 21) & 1
        vs_s, vs_f, geo_s, geo_f = rb(0, 1), rb(1, 9), rb(10, 1), rb(11, 6)
        me |= _put(rb(17, 5), 9, 5) | _put(se, 14, 1) | _put(ew_f, 15, 10) | _put(sn, 25, 1) | _put(ns_f, 26, 10)
        me |= _put(rb(22, 1), 36, 1) | _put(vs_s, 37, 1) | _put(vs_f, 38, 9) | _put(rb(23, 2), 47, 2)
        me |= _put(geo_s, 49, 1) | _put(geo_f, 50, 6) | _put(rb(25, 1), 56, 1)
        ns, ew = ns_f.astype(np.float64), ew_f.astype(np.float64)
        if sub == 2:
            ns, ew = ns * 4, ew * 4
        speed = np.sqrt(ns * ns + ew * ew)
        ews = np.where(se == 1, 0 - ew, ew)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = ews / ns
        a_ld = np.arctan(np.where(ns == 0, 0.0, q).astype(L))
        a = a_ld.astype(np.float64)
        hdg = np.where(ns == 0, 0.0, a * (180.0 / math.pi))
        hdg = np.where(sn == 1, 180 - hdg, hdg)
        hdg = np.where(hdg < 0, hdg + 360, hdg)
        vs = (vs_f.astype(np.float64) - 1) * 64
        v2 = np.where(vs_s == 1, 0 - vs, vs)
        geo = geo_f.astype(np.int64) * 25
        v3 = np.where(geo_s == 1, -geo, geo).astype(np.float64)
    return me, speed, hdg, v2, v3, _near_tie(a_ld, a)


def _trk_side_agree(track, target_side):
    """For every track, the 5,0 track raw values whose difference d lies nearest 10 deg on the given side (+10 / -10):
    amb_commb_agree's track decision (d <= 10) for each, and whether d == 10 exactly. Shapes (n, 4)."""
    t0 = np.floor((track + target_side) * 512.0 / 90.0).astype(np.int64)
    t = (t0[:, None] + np.arange(-1, 3)[None, :] + 1024) % 2048 - 1024
    return t


def _agree_track(t, track):
    trk = t * 90.0 / 512.0
    d = np.fmod(np.abs(trk - track[:, None]), 360.0)
    d = np.where(d < 360.0 - d, d, 360.0 - d)
    return d <= 10.0, d == 10.0


@pytest.fixture(scope="module")
def velocity_domain():
    """Decode every velocity word; per subtype: the ulp histograms, the counts, and the records where the device and
    the correctly rounded values differ (for the CPython comparison)."""
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    rng = np.random.default_rng(12)
    out = {}
    for sub, bits in ((0, 24), (1, 22), (2, 22)):
        s = {"n": 0, "squares": 0, "su_hist": np.zeros(65, np.int64), "hu_hist": np.zeros(65, np.int64),
             "near_tie": 0, "near_tie_max": 0, "hdg_range_bad": 0, "exact_bad": 0, "vs_bad": 0, "meta_bad": 0, "trk_mismatch": 0,
             "trk_ties": 0, "trk_checked": 0, "diff": []}
        for start in range(0, 1 << bits, BATCH):
            idx = np.arange(start, min(start + BATCH, 1 << bits), dtype=np.int64)
            me, speed, hdg, v2, v3, near = _velocity_batch(sub, idx, rng)
            icao = 0xA00000 | (idx & 0xFFFF)
            fr = _df17_frames(me, icao)
            rec = d.decode(fr)
            val = rec["val"]
            s["meta_bad"] += int(np.sum((rec["status"] != 0) | (rec["bds"] != 9) | (rec["subtype"] != min(sub, 1))
                                        | (rec["icao"] != icao)))
            su, hu = _ulps(val[:, 0], speed), _ulps(val[:, 1], hdg)
            s["su_hist"] += np.bincount(np.minimum(su, 64), minlength=65)
            s["hu_hist"] += np.bincount(np.minimum(hu[~near], 64), minlength=65)
            s["near_tie"] += int(np.sum(near))
            s["near_tie_max"] = max(s["near_tie_max"], int(hu[near].max(initial=0)))
            sq = speed == np.floor(speed)
            s["squares"] += int(np.sum(sq))
            s["exact_bad"] += int(np.sum(val[sq, 0].view(np.int64) != speed[sq].view(np.int64)))
            if sub == 0:
                s["hdg_range_bad"] += int(np.sum(~((val[:, 1] >= 0) & (val[:, 1] < 360))))
            s["vs_bad"] += int(np.sum((val[:, 2].view(np.int64) != v2.view(np.int64))
                                      | (val[:, 3].view(np.int64) != v3.view(np.int64))))
            # the Comm-B track rule at the 5,0 tracks nearest 10 deg either side: device heading vs correctly rounded
            for side in (10.0, -10.0):
                t = _trk_side_agree(hdg, side)
                ag_dev, tie_dev = _agree_track(t, val[:, 1])
                ag_ref, tie_ref = _agree_track(t, hdg)
                s["trk_mismatch"] += int(np.sum(ag_dev != ag_ref))
                s["trk_ties"] += int(np.sum(tie_dev | tie_ref))
                s["trk_checked"] += t.size
            bad = np.flatnonzero((su != 0) | (hu != 0))
            if len(bad):
                s["diff"].append((fr[bad], rec[bad], speed[bad], hdg[bad]))
            s["n"] += len(idx)
        out[sub] = s
    d.close()
    return out


def test_velocity_speed_is_the_correctly_rounded_root_over_the_whole_domain(velocity_domain):
    for sub, s in velocity_domain.items():
        print("subtype %d: %d words, %d perfect squares, speed ulp histogram %s" % (
            sub, s["n"], s["squares"], _hist_of_counts(s["su_hist"])))
        assert s["n"] == (1 << 24 if sub == 0 else 1 << 22)
        assert s["meta_bad"] == 0
        assert s["exact_bad"] == 0, (sub, s["exact_bad"])
        assert np.all(s["su_hist"][SPEED_ULP + 1:] == 0), (sub, s["su_hist"][:8])


def test_velocity_heading_within_its_ulp_bound(velocity_domain):
    for sub, s in velocity_domain.items():
        print("subtype %d: heading ulp histogram %s; %d long-double values within 2^-8 ulp of a rounding boundary, "
              "at most %d ulp apart there" % (sub, _hist_of_counts(s["hu_hist"]), s["near_tie"], s["near_tie_max"]))
        assert np.all(s["hu_hist"][HEADING_ULP + 1:] == 0), (sub, s["hu_hist"][:8])
        assert s["near_tie_max"] <= HEADING_ULP + 1
        assert s["hdg_range_bad"] == 0
        assert s["vs_bad"] == 0


def test_velocity_report_text_equals_cpythons_where_the_doubles_differ(velocity_domain):
    """The records where the device and the correctly rounded value differ (a seeded CPYTHON_SHARE of them, every
    perfect square among them), decoded by oracle/decode_oracle.py (CPython math.hypot / math.atan2, as the reference's
    parser): count where the device differs from CPython, and the printed line (%.0f of speed and heading) must be the
    same there."""
    from gr_air_modes_b200 import decode, report
    from oracle import decode_oracle as do
    for sub, s in velocity_domain.items():
        n = n_speed = n_hdg = n_cr = 0
        rng = np.random.default_rng(sub)
        for fr, rec, speed, hdg in s["diff"]:
            keep = np.flatnonzero((speed == np.floor(speed)) | (rng.random(len(fr)) < CPYTHON_SHARE))
            for k in keep:
                hx = bytes(fr["data"][k]).hex()
                want = do.decode_one(hx, 0, float(fr["secs"][k]) + float(fr["frac"][k]), do.CprState())
                got = rec[k]
                dv, wv = [float(x) for x in got["val"][:2]], want["val"][:2]
                n += 1
                n_speed += dv[0] != wv[0]
                n_hdg += dv[1] != wv[1]
                n_cr += (wv[0] != speed[k]) or (wv[1] != hdg[k])
                if dv != wv:
                    msg = "%s 000000 0.5 %d %r" % (hx, int(fr["secs"][k]), float(fr["frac"][k]))
                    mine = decode.record_to_dict(got)
                    mine["val"] = wv + mine["val"][2:]
                    assert report.format_report(msg, got) == report.format_report(msg, mine), (sub, hx, dv, wv)
        print("subtype %d: %d records differ from the correctly rounded values; CPython differs from the device in "
              "%d speeds and %d headings, and from the correctly rounded values in %d records" % (sub, n, n_speed, n_hdg, n_cr))


def test_commb_track_rule_at_every_heading(velocity_domain):
    """No exact tie at 10 deg is reachable: the 5,0 track trk_raw * 90 / 512 is a dyadic rational with denominator 2^9
    and trk +- 10 one with denominator 2^8, whereas the heading of integer speeds is an angle whose tangent is rational,
    which (Niven) is a rational number of degrees only at multiples of 45 deg, none of which is trk +- 10; so a tie
    would need the double rounding of a heading to land exactly on such a dyadic. Counted here over every heading the
    decoder produces, with the track raw values nearest 10 deg on both sides: none does, and the device's decision
    equals the one from the correctly rounded heading for every one of them."""
    for sub, s in velocity_domain.items():
        print("subtype %d: %d (heading, 5,0 track) pairs near the 10 deg rule, %d exact ties, %d decisions differ" % (
            sub, s["trk_checked"], s["trk_ties"], s["trk_mismatch"]))
        assert s["trk_ties"] == 0 and s["trk_mismatch"] == 0


# ---- B: range and bearing ------------------------------------------------------------------------------------------
def range_bearing_ref(a_lat, a_lon, b_lat, b_lon):
    """amb_range_bearing (cpr.py:158-181) with every +, -, *, / in double as written, and each libm call (sin, pow,
    cos, atan2, hypot) in long double, rounded once to double."""
    f = float
    es = (1 / 298.257223563) * (2 - (1 / 298.257223563))
    r_mi = 3963.19059 * (math.pi / 180)
    dlat, dlon = b_lat - a_lat, b_lon - a_lon
    avg = ((a_lat + b_lat) / 2.0) * math.pi / 180
    s = f(np.sin(L(avg)))
    s2 = s * s                                       # pow(s, 2.0) correctly rounded
    r1 = r_mi * (1.0 - es) / f(np.power(L(1.0 - es * s2), L(1.5)))
    r2 = r_mi / math.sqrt(1.0 - es * s2)
    north = r1 * dlat
    east = r2 * f(np.cos(L(avg))) * dlon
    b = f(np.arctan2(L(east), L(north))) * (180.0 / math.pi)
    if b < 0.0:
        b += 360.0
    return f(np.hypot(L(east), L(north))), b, east, north


RECEIVERS = [(lat, lon) for lat in (0.0, 45.0, -45.0, 86.9, -86.9) for lon in (10.0, 179.95, -179.95)]
OFFSETS = [(0.4, 0.0), (-0.4, 0.0), (0.0, 0.6), (0.0, -0.6), (0.3, 0.45), (-0.2, -0.35), (0.0, 0.0)]


def _pos_msgs(targets, local):
    """One aircraft per target: an even/odd pair (global fix); with `local`, 20 s later one even report of a point
    0.01 deg further north (the pair has expired: a local fix from the global one). Returns (msgs, index of the record
    that carries each target's position)."""
    ev, which = [], []
    for i, (lat, lon) in enumerate(targets):
        aa = 0x500000 + i
        t = 1.0 + 0.01 * i
        for odd in (0, 1):
            la, lo_ = dc.cpr_encode(lat, lon, odd)
            ev.append((t + 0.1 * odd, *dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(30000), odd, la, lo_))))
        if local:
            la, lo_ = dc.cpr_encode(min(lat + 0.01, 89.9), lon, 0)
            ev.append((t + 20.0, *dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(30000), 0, la, lo_))))
    msgs = tc._msgs(ev)
    return msgs


def _decode_positions(decode, loc, msgs, local):
    d = decode.batch_decoder(loc, local_cpr=30 if local else 0)
    recs = d.decode(tc.frames_of(msgs, unqueued_every=0))
    d.close()
    return recs


def _wrap(lon):
    return (lon + 180.0) % 360.0 - 180.0


def test_range_and_bearing_at_their_geometric_edges():
    from gr_air_modes_b200 import decode, report
    from oracle import decode_oracle as do
    rows = []                                        # (receiver, record, message string)
    for local in (False, True):
        for rx in RECEIVERS:
            targets = [(max(-89.0, min(89.0, rx[0] + a)), _wrap(rx[1] + b)) for a, b in OFFSETS]
            targets.append((rx[0] + 0.1, _wrap(rx[1] + 0.2 if rx[1] > 0 else rx[1] - 0.2)))   # across +-180 near 179.95
            msgs = _pos_msgs(targets, local)
            recs = _decode_positions(decode, list(rx), msgs, local)
            fixes = [k for k in range(len(recs)) if recs["status"][k] & decode.FS_HAS_RANGE]
            # the same fixes seen from receivers due N/S, due E/W and at the fix itself
            for k in fixes:
                lat, lon = float(recs["lat"][k]), float(recs["lon"][k])
                for loc in ([rx[0], lon], [lat, rx[1]], [lat, lon]):
                    r2 = _decode_positions(decode, loc, msgs, local)
                    assert r2["lat"][k] == lat and r2["lon"][k] == lon
                    rows.append((tuple(loc), r2[k], msgs, k))
                rows.append((rx, recs[k], msgs, k))
    n_local = sum(1 for _, r, _, _ in rows if decode.local_outcome(r) == decode.LOCAL_DECODED)
    ru, bu, n_axis, n_zero = [], [], 0, 0
    texts = dc.message_strings
    for loc, r, msgs, k in rows:
        lat, lon, rng_d, brg_d = float(r["lat"]), float(r["lon"]), float(r["range"]), float(r["bearing"])
        rng_r, brg_r, east, north = range_bearing_ref(loc[0], loc[1], lat, lon)
        ru.append(int(_ulps([rng_d], [rng_r])[0]))
        bu.append(int(_ulps([brg_d], [brg_r])[0]))
        rng_c, brg_c = do.range_bearing(list(loc), [lat, lon])
        assert 0.0 <= brg_d <= 360.0, (loc, lat, lon, brg_d)
        if lat == loc[0] and lon == loc[1]:
            n_zero += 1
            assert rng_d == 0.0 and brg_d == brg_c, (loc, rng_d, brg_d)
        if east == 0.0 or north == 0.0:
            n_axis += 1
            assert brg_d == brg_c, (loc, lat, lon, brg_d, brg_c)
        assert "%.2f" % rng_d == "%.2f" % rng_c and "%.0f" % brg_d == "%.0f" % brg_c, (loc, lat, lon, rng_d, rng_c)
        msg = texts([msgs[k]])[0]
        mine = decode.record_to_dict(r)
        mine["range"], mine["bearing"] = rng_c, brg_c
        assert report.format_report(msg, r) == report.format_report(msg, mine)
    ru, bu = np.array(ru), np.array(bu)
    print("range/bearing: %d fixes (%d local), %d due N/S/E/W, %d at the receiver; range ulp histogram %s, bearing ulp "
          "histogram %s" % (len(rows), n_local, n_axis, n_zero, _hist(ru), _hist(bu)))
    assert n_local > 50 and n_axis > 100 and n_zero > 50
    assert ru.max() <= RANGE_ULP and bu.max() <= BEARING_ULP


# ---- C: Comm-B decisions -------------------------------------------------------------------------------------------
def cpython_velocities(msgs, off):
    """`off` with the speed and track of every velocity reference record replaced by what oracle/decode_oracle.py
    (CPython math) computes for the same message."""
    from oracle import decode_oracle as do
    recs = off.copy()
    want = do.decode_batch(msgs)
    n = 0
    for k in range(len(recs)):
        if co.is_reference(recs[k]):
            v = want[k]["val"]
            n += (float(recs["val"][k][0]) != v[0]) or (float(recs["val"][k][1]) != v[1])
            recs["val"][k, 0], recs["val"][k, 1] = v[0], v[1]
    return recs, n


def with_val_of(recs, off):
    """The checker's records with the decoder's own `val` back (only aux and pad_ are the option's)."""
    recs["val"] = off["val"]
    return recs


def test_commb_scenes_equal_the_checker_fed_with_cpython_velocities():
    from gr_air_modes_b200 import decode
    for name, msgs, S in cc.scenes():
        frames = tc.frames_of(msgs)
        plain = decode.batch_decoder(None)
        off = plain.decode(frames)
        plain.close()
        d = decode.batch_decoder(None, commb=S)
        on = d.decode(frames)
        d.close()
        co.assert_records_equal(on, co.replay(frames, off, S), (name, "own velocities"))
        py, n = cpython_velocities(msgs, off)
        co.assert_records_equal(on, with_val_of(co.replay(frames, py, S), off), (name, "CPython velocities"))
        print("%s: %d velocity references differ from CPython's" % (name, n))


def tie_outcomes(on, cases):
    """(counts, failures) of the tie scene's replies: RESOLVED as 5,0 exactly where |2 GS - c| = 20 (speed cases)."""
    o, reg = co.outcome_of(on), (np.asarray(on["pad_"], dtype=np.uint64) >> np.uint64(16)) & np.uint64(0xFF)
    counts, bad = {}, []
    for k, case in enumerate(cases):
        if case is None:
            continue
        as50 = o[k] == co.RESOLVED and reg[k] == 0x50
        kind, delta = case
        key = (kind, delta) if kind == "speed" else (kind, "<=10" if delta <= 10.0 else ">10")
        counts[key] = counts.get(key, 0) + 1
        want = abs(delta) == 20 if kind == "speed" else delta <= 10.0
        if as50 != want:
            bad.append((k, case, int(o[k]), int(reg[k])))
    return counts, bad


def test_commb_speed_ties_and_track_edges():
    from gr_air_modes_b200 import decode
    msgs, cases = cc.tie_scene()
    frames = tc.frames_of(msgs, unqueued_every=0)
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    d = decode.batch_decoder(None, commb=30)
    on = d.decode(frames)
    d.close()
    py, n = cpython_velocities(msgs, off)
    co.assert_records_equal(on, with_val_of(co.replay(frames, py, 30), off), "ties, CPython velocities")
    co.assert_records_equal(on, co.replay(frames, off, 30), "ties, own velocities")
    counts, bad = tie_outcomes(on, cases)
    print("Comm-B ties: %d velocities (%d differ from CPython), replies per case %s" % (
        sum(c is None for c in cases), n, dict(sorted(counts.items(), key=str))))
    assert not bad, bad[:10]
    assert all(counts.get(("speed", x), 0) > 500 for x in (-22, -20, 20, 22))
    assert counts.get(("track", "<=10"), 0) > 500 and counts.get(("track", ">10"), 0) > 500
