"""Brute-force checker of the batch decoder's option "local_cpr" (include/airmodes_b200.h AMB_FIELDS_LOCAL). Test-only.

It starts from the records of the reference's decoder (oracle/decode_oracle.py, option off) and walks the position
messages in stream order. For each one without a global fix it finds the aircraft's reference position by scanning
EVERY earlier message of the same ICAO in its own output for the latest one with a position - no table, no buckets,
O(n^2) - and decodes relative to it. The local decode is cpr_resolve_local (cpr.py:61-82) restated here in plain
Python; tests/golden/local_cpr_golden.json.gz pins it bit for bit against the unmodified reference function.
"""
from __future__ import annotations

import math

from oracle import decode_oracle as do

LOCAL_NOT_TRIED, LOCAL_DECODED, LOCAL_NO_REF, LOCAL_STALE, LOCAL_REJECTED = 0, 1, 2, 3, 4


def zone_lat(fmt: int, surface: int) -> float:
    """Latitude zone size: 90 or 360 degrees over 60 (even) or 59 (odd) zones."""
    return (90.0 if surface else 360.0) / (60 - fmt)


def resolve_local(ref_lat: float, ref_lon: float, enclat: int, enclon: int, fmt: int, surface: int):
    """The position (lat, lon) nearest to the reference whose CPR encoding is (enclat, enclon); Python's float % is
    the floor modulo."""
    zl = zone_lat(fmt, surface)
    yl = enclat / 131072.0
    lat = zl * (math.floor(ref_lat / zl) + math.floor(0.5 + (ref_lat % zl) / zl - yl) + yl)
    zo = (90.0 if surface else 360.0) / max(do.nl(lat) - fmt, 1)
    xl = enclon / 131072.0
    lon = zo * (math.floor(ref_lon / zo) + math.floor(0.5 + (ref_lon % zo) / zo - xl) + xl)
    return lat, lon


def is_position(r) -> bool:
    return r["df"] == 17 and r["bds"] in (0x05, 0x06) and not (r["status"] & (do.FS_NO_HANDLER | do.FS_NOT_QUEUED))


def apply_local(recs, times, location, S):
    """recs: decode_oracle records of one stream (option off), times: secs + frac per record. Returns new records with
    the local decode applied and the outcome under "local"."""
    out = []
    for k, r0 in enumerate(recs):
        r = dict(r0)
        r["local"] = LOCAL_NOT_TRIED
        out.append(r)
        if S <= 0 or not is_position(r) or (r["status"] & do.FS_HAS_POS):
            continue
        ref = None
        for j in range(k - 1, -1, -1):                      # the latest earlier position of this aircraft
            q = out[j]
            if is_position(q) and q["icao"] == r["icao"] and (q["status"] & do.FS_HAS_POS):
                ref = (q["lat"], q["lon"], times[j])
                break
        if ref is None:
            r["local"] = LOCAL_NO_REF
            continue
        age = times[k] - ref[2]
        if not (age >= 0.0) or age > S:
            r["local"] = LOCAL_STALE
            continue
        lat, lon = resolve_local(ref[0], ref[1], r["cpr_lat"], r["cpr_lon"], r["cpr_format"], r["surface"])
        if lon > 180.0:
            lon -= 360.0
        elif lon <= -180.0:
            lon += 360.0
        if abs(lat) > 90.0 or abs(lat - ref[0]) > zone_lat(r["cpr_format"], r["surface"]) / 2:
            r["local"] = LOCAL_REJECTED
            continue
        r["lat"], r["lon"], r["status"] = lat, lon, r["status"] | do.FS_HAS_POS
        if location is not None:
            r["range"], r["bearing"] = do.range_bearing(location, [lat, lon])
            r["status"] |= do.FS_HAS_RANGE
        r["local"] = LOCAL_DECODED
    return out


def decode_local(msgs, location, S):
    """msgs: (payload_hex, ecc, secs, frac) in stream order -> records with the option local_cpr = S."""
    recs = do.decode_batch(msgs, location)
    return apply_local(recs, [float(s) + float(f) for _, _, s, f in msgs], location, S)
