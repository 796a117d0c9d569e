"""Sequential checker of the batch decoder's option "track_ext" (include/airmodes_b200.h amb_aircraft_ext). Test-only.

It replays the decoder's own frames and records one at a time, in stream order, into a plain dict of groups per
address - no buckets, no warps, no bitmap - and takes the base rows from tests/track_oracle.py. So it checks the
extension alone; the records are checked by the op-status and Comm-B checkers. Rules (DESIGN.md §8 "Aircraft table
extension"):

  a queued record (status without FS_NOT_QUEUED) writes at most one group of address a = its icao, t = secs + frac:
    OPS    ES outcome (pad_ byte 5) == OPSTATUS                          aux, ES version (byte 6)
    TS     ES outcome == TARGET_STATE                                     aux
    INTEG  ES outcome in (NIC, NUC) and FS_HAS_POS                        aux[0..1], ES outcome, version, NIC (5..7)
    B40 / B50 / B60  Comm-B outcome (byte 1) in (DECODED, RESOLVED) and register (byte 2) 0x40 / 0x50 / 0x60:
                                                                          raw fields 0..4 (aux as int16), mask (3), outcome
  a later writer of a group replaces it; reset forgets every group;
  snapshot at now: the base rows of the track checker's snapshot; a group is shown when first_seen <= t <= now and
  now - t <= S2; a hidden group has t = NaN and every field byte 0.
"""
from __future__ import annotations

import math

import numpy as np

import track_oracle as to

FS_HAS_POS, FS_NOT_QUEUED = 0x10, 0x80
ES_OPSTATUS, ES_TARGET_STATE, ES_NIC, ES_NUC = 1, 2, 3, 4
COMMB_DECODED, COMMB_RESOLVED = 1, 2
OPS, TS, INTEG, B40, B50, B60 = range(6)


def group_of(r):
    """The group record r (a FIELDS_DTYPE record) writes, or None."""
    st = int(r["status"])
    if st & FS_NOT_QUEUED:
        return None
    pad = int(r["pad_"])
    es, cb, reg = (pad >> 40) & 0xFF, (pad >> 8) & 0xFF, (pad >> 16) & 0xFF
    if es == ES_OPSTATUS:
        return OPS
    if es == ES_TARGET_STATE:
        return TS
    if es in (ES_NIC, ES_NUC) and st & FS_HAS_POS:
        return INTEG
    if cb in (COMMB_DECODED, COMMB_RESOLVED) and reg in (0x40, 0x50, 0x60):
        return {0x40: B40, 0x50: B50, 0x60: B60}[reg]
    return None


def _put(x, g, r, t):
    """Group g of the packed extension row x := what record r carries, at time t."""
    pad = int(r["pad_"])
    aux = np.asarray(r["aux"], dtype="<u4")
    x["t"][g] = t
    if g == OPS:
        x["ops"] = aux
        x["ops_version"] = (pad >> 48) & 0xFF
    elif g == TS:
        x["ts"] = aux
    elif g == INTEG:
        x["integ"] = aux[:2]
        x["integ_es"], x["integ_version"], x["integ_nic"] = (pad >> 40) & 0xFF, (pad >> 48) & 0xFF, (pad >> 56) & 0xFF
    else:
        c = g - B40
        x["commb"][c] = aux.view("<i2")[:5]
        x["commb_mask"][c], x["commb_outcome"][c] = (pad >> 24) & 0xFF, (pad >> 8) & 0xFF


class ExtTracker:
    """The aircraft table (track = S) and its extension (track_ext = S2) of one decoder, fed batch after batch."""

    def __init__(self, S: int, S2: int):
        self.base = to.Tracker(S)
        self.S2 = S2
        self.groups = {}                    # address -> {group: (t, record)}

    def reset(self):
        self.base.reset()
        self.groups = {}

    def feed(self, frames, records):
        """frames: FRAME_DTYPE array, records: the decoder's FIELDS_DTYPE records of them (all its options on)."""
        self.base.feed(frames, records)
        secs, frac = frames["secs"], frames["frac"]
        for k in range(len(records)):
            r = records[k]
            g = group_of(r)
            a = int(r["icao"])
            if g is None or a > 0xFFFFFF:
                continue
            self.groups.setdefault(a, {})[g] = (float(secs[k]) + float(frac[k]), r.copy())

    def snapshot_arrays(self, now=None):
        """(AIRCRAFT_DTYPE rows, AIRCRAFT_EXT_DTYPE extensions) at `now` (None: the latest queued record's t)."""
        from gr_air_modes_b200 import decode
        rows = self.base.snapshot(now)
        now = self.base.last_t if now is None else float(now)
        ext = np.zeros(len(rows), dtype=decode.AIRCRAFT_EXT_DTYPE)
        for i, row in enumerate(rows):
            a = row["icao"]
            x = ext[i]
            x["icao"] = a
            x["t"] = math.nan
            shown = 0
            for g, (t, r) in sorted(self.groups.get(a, {}).items()):
                if row["first_seen"] <= t <= now and now - t <= self.S2:
                    _put(x, g, r, t)
                    shown |= 1 << g
            x["shown"] = shown
        return to.pack(rows), ext


def assert_snapshots_equal(got, want, where=""):
    """(rows, ext) pairs equal bit for bit, every NaN matching a NaN."""
    to.assert_rows_equal(got[0], want[0], (where, "rows"))
    to.assert_rows_equal(got[1], want[1], (where, "ext"))


def replay(frames, records, S, S2, now=None):
    """The snapshot after the whole stream, in one call."""
    tr = ExtTracker(S, S2)
    tr.feed(frames, records)
    return tr.snapshot_arrays(now)
