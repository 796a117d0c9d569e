"""Sequential checker of the batch decoder's option "track" (include/airmodes_b200.h amb_aircraft). Test-only.

It replays the rules one record at a time, in stream order, over the decoder's own records and the frames they came
from, into a plain dict of rows per address - no buckets, no warps, no bitmap. So it checks the aircraft table alone;
the records are checked elsewhere. Rules (DESIGN.md §8 "Aircraft table"):

  a record counts when its status has neither FS_NOT_QUEUED nor FS_NO_HANDLER (and its icao fits 24 bits);
  a = its icao, t = float(secs) + frac of its frame;
  expiry:    a row with t - seen > S counts as absent (its data stays until a DF17 record replaces it);
  creation:  without a live row a DF17 record creates one (all columns blank, first_seen = t, messages = 0); any other
             record is ignored;
  apply:     messages += 1, seen = t, ref_level = the frame's; altitude from DF0/4/16/20 and BDS0,5 when set; BDS0,5
             clears ON_GROUND, BDS0,6 sets altitude 0 and ON_GROUND; squawk from DF5/21; ident/ftc/cat from BDS0,8;
             lat/lon/pos_t = t from FS_HAS_POS, range/bearing with FS_HAS_RANGE (else NaN); speed/heading/vertical =
             val[0..2] of BDS0,9 subtypes 0 and 1; heading = val[0] of BDS0,6; eps from BDS6,1;
  snapshot:  rows with seen <= now and now - seen <= S, ascending address; now = None: the t of the latest queued
             record since reset.
"""
from __future__ import annotations

import math

import numpy as np

FS_NO_HANDLER, FS_HAS_POS, FS_HAS_RANGE, FS_NOT_QUEUED = 0x01, 0x10, 0x20, 0x80
NO_ALTITUDE = -(1 << 31)
AC_HAS_ALT, AC_HAS_SQUAWK, AC_HAS_IDENT, AC_HAS_POS, AC_HAS_RANGE = 0x001, 0x002, 0x004, 0x008, 0x010
AC_HAS_VELOCITY, AC_HAS_HEADING, AC_HAS_EPS, AC_ON_GROUND = 0x020, 0x040, 0x080, 0x100
NAN = float("nan")


def _blank(a, t):
    return {"icao": a, "messages": 0, "first_seen": t, "seen": t, "ref_level": np.float32(0), "flags": 0,
            "ftc": -1, "cat": -1, "ident": b"\0" * 8, "altitude": NO_ALTITUDE, "squawk": -1, "lat": NAN, "lon": NAN,
            "range": NAN, "bearing": NAN, "pos_t": NAN, "speed": NAN, "heading": NAN, "vertical": NAN, "eps": -1}


def _set(row, flag, on):
    row["flags"] = (row["flags"] | flag) if on else (row["flags"] & ~flag)


def apply(row, r, t, ref_level):
    """One counting record r (a FIELDS_DTYPE record) applied to a live row."""
    row["messages"] += 1
    row["seen"] = t
    row["ref_level"] = np.float32(ref_level)
    df, bds, st = int(r["df"]), int(r["bds"]), int(r["status"])
    b05, b06 = df == 17 and bds == 0x05, df == 17 and bds == 0x06
    alt = int(r["altitude"])
    if (df in (0, 4, 16, 20) or b05) and alt != NO_ALTITUDE:
        row["altitude"] = alt
        _set(row, AC_HAS_ALT, True)
    if b05:
        _set(row, AC_ON_GROUND, False)
    if b06:
        row["altitude"] = 0
        _set(row, AC_HAS_ALT, True)
        _set(row, AC_ON_GROUND, True)
    if df in (5, 21):
        row["squawk"] = int(r["squawk"])
        _set(row, AC_HAS_SQUAWK, True)
    if df == 17 and bds == 0x08:
        row["ident"] = bytes(np.asarray(r["ident"]).tobytes()).ljust(8, b"\0")
        row["ftc"], row["cat"] = int(r["ftc"]), int(r["cat"])
        _set(row, AC_HAS_IDENT, True)
    if st & FS_HAS_POS:
        row["lat"], row["lon"], row["pos_t"] = float(r["lat"]), float(r["lon"]), t
        rb = bool(st & FS_HAS_RANGE)
        row["range"], row["bearing"] = (float(r["range"]), float(r["bearing"])) if rb else (NAN, NAN)
        _set(row, AC_HAS_POS, True)
        _set(row, AC_HAS_RANGE, rb)
    if df == 17 and bds == 0x09 and int(r["subtype"]) in (0, 1):
        row["speed"], row["heading"], row["vertical"] = float(r["val"][0]), float(r["val"][1]), float(r["val"][2])
        _set(row, AC_HAS_VELOCITY, True)
        _set(row, AC_HAS_HEADING, True)
    if b06:
        row["heading"] = float(r["val"][0])
        _set(row, AC_HAS_HEADING, True)
    if df == 17 and bds == 0x61:
        row["eps"] = int(r["eps"])
        _set(row, AC_HAS_EPS, True)


class Tracker:
    """The table of one decoder with track = S, fed batch after batch like the decoder."""

    def __init__(self, S: int):
        self.S = S
        self.rows = {}
        self.last_t = NAN

    def reset(self):
        self.rows, self.last_t = {}, NAN

    def feed(self, frames, records):
        """frames: FRAME_DTYPE array (secs, frac, ref_level), records: the decoder's FIELDS_DTYPE records of them."""
        secs, frac, ref = frames["secs"], frames["frac"], frames["ref_level"]
        for k in range(len(records)):
            r = records[k]
            st = int(r["status"])
            if st & FS_NOT_QUEUED:
                continue
            t = float(secs[k]) + float(frac[k])
            self.last_t = t
            a = int(r["icao"])
            if st & FS_NO_HANDLER or a > 0xFFFFFF:
                continue
            row = self.rows.get(a)
            if row is None or t - row["seen"] > self.S:
                if int(r["df"]) != 17:
                    continue
                row = _blank(a, t)
                self.rows[a] = row
            apply(row, r, t, ref[k])

    def snapshot(self, now=None):
        """Rows shown at `now` (None: the latest queued record's t), ascending address, as dicts."""
        now = self.last_t if now is None else float(now)
        return [self.rows[a] for a in sorted(self.rows)
                if self.rows[a]["seen"] <= now and now - self.rows[a]["seen"] <= self.S]

    def snapshot_array(self, now=None):
        return pack(self.snapshot(now))


def pack(rows):
    """Checker rows -> AIRCRAFT_DTYPE array (pad zero)."""
    from gr_air_modes_b200 import decode
    out = np.zeros(len(rows), dtype=decode.AIRCRAFT_DTYPE)
    for k, row in enumerate(rows):
        for name, v in row.items():
            out[k][name] = np.frombuffer(v, dtype="S1") if name == "ident" else v
    return out


def assert_rows_equal(got, want, where=""):
    """Two AIRCRAFT_DTYPE arrays equal bit for bit, every NaN matching a NaN (whatever its payload)."""
    assert got.dtype == want.dtype and len(got) == len(want), (where, len(got), len(want))
    if len(got) == 0:
        return
    for name in got.dtype.names:
        g, w = got[name], want[name]
        if g.dtype.kind == "f":
            gn, wn = np.isnan(g), np.isnan(w)
            bad = np.nonzero((gn != wn) | (~gn & (g.view("u%d" % g.dtype.itemsize) != w.view("u%d" % w.dtype.itemsize))))[0]
        else:
            bad = np.nonzero(np.asarray(g != w).reshape(len(g), -1).any(axis=1))[0]
        assert bad.size == 0, (where, name, int(got["icao"][bad[0]]), got[bad[0]], want[bad[0]])


def replay(frames, records, S, now=None):
    """The snapshot after the whole stream, in one call."""
    tr = Tracker(S)
    tr.feed(frames, records)
    return tr.snapshot_array(now)


def t_of(frames):
    return [float(s) + float(f) for s, f in zip(frames["secs"], frames["frac"])]


def rssi(ref_level) -> float:
    return 10.0 * math.log10(max(1e-8, float(ref_level)))
