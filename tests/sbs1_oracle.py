"""Sequential checker of the decoder option "sbs1" (include/airmodes_b200.h, DESIGN.md §8 "SBS-1 feed"), written from
the rules and not from the kernels: it replays a decoder's records and frames in stream order, keeps the aircraft ids
in a dict with the window of sbs1.py:83-88 as Python 2 runs it, and formats every line with Python's own % and
datetime, in the formats of sbs1.py:153-222."""
from __future__ import annotations

import datetime
import math

FS_NO_HANDLER, FS_METRIC_ALT, FS_HAS_POS, FS_NOT_QUEUED = 0x01, 0x02, 0x10, 0x80
WINDOW = 10000
LAST_SEC = 253402300799
EPOCH = datetime.datetime(1970, 1, 1)
CATEGORY_ROWS = (8, 7, 8, 8)                           # len(categories[ftc - 1]), parse.py:270-273


def decode_fs(fs):                                      # sbs1.py:117-131
    return {0: "0,0,0,0", 1: "0,0,0,1", 2: "1,0,0,0", 3: "1,0,0,1", 4: "1,0,1,", 5: "0,0,1,"}.get(fs, ",,,")


def stamp(secs, frac, tz=0):
    """Rule 5: [date, time] strings of a frame's stamp, or ["", ""] outside 1970 .. 9999 or for a frac that is not
    finite. A negative frac (never in a frame) counts as 0 milliseconds."""
    secs, frac = int(secs), float(frac)
    if not math.isfinite(frac):
        return ["", ""]
    secs += int(frac)                                   # modes_types.stamp (modes_types.py:29-33)
    frac -= int(frac)
    ms = max(0, min(999, math.floor(frac * 1000.0)))
    s = secs + 60 * tz
    if not 0 <= s <= LAST_SEC:
        return ["", ""]
    dt = EPOCH + datetime.timedelta(seconds=s)
    return [dt.strftime("%Y/%m/%d"), dt.strftime("%H:%M:%S") + ".%03d" % ms]


def published(r) -> bool:
    """Rule 1."""
    st = int(r["status"])
    return not st & (FS_NOT_QUEUED | FS_NO_HANDLER) and int(r["df"]) in (0, 4, 5, 11, 17) and int(r["icao"]) < (1 << 24)


def line(r, aircraft_id, date, tod):
    """Rule 3: the line of published record r, or None."""
    df, st, icao = int(r["df"]), int(r["status"]), int(r["icao"])
    head = (aircraft_id, icao, aircraft_id + 100, date, tod, date, tod)
    if df == 0:
        if st & FS_METRIC_ALT:
            return None
        return "MSG,7,0,%i,%06X,%i,%s,%s,%s,%s,,%s,,,,,,,,,," % (head + (int(r["altitude"]),)) + \
            ("1\r\n" if int(r["vs"]) else "0\r\n")
    if df == 4:
        if st & FS_METRIC_ALT:
            return None
        return "MSG,5,0,%i,%06X,%i,%s,%s,%s,%s,,%s,,,,,,," % (head + (int(r["altitude"]),)) + decode_fs(int(r["fs"])) + "\r\n"
    if df == 5:
        return "MSG,6,0,%i,%06X,%i,%s,%s,%s,%s,,,,,,,,%04i," % (head + (int(r["squawk"]),)) + decode_fs(int(r["fs"])) + "\r\n"
    if df == 11:
        return "MSG,8,0,%i,%06X,%i,%s,%s,%s,%s,,,,,,,,,,,,\r\n" % head
    bds = int(r["bds"])
    if bds == 0x08:
        ftc, cat = int(r["ftc"]), int(r["cat"])
        if not 1 <= ftc <= 4 or cat >= CATEGORY_ROWS[ftc - 1]:
            return None                                 # IndexError in parseBDS08 (parse.py:275)
        ident = bytes(r["ident"]).decode("ascii")
        return "MSG,1,0,%i,%06X,%i,%s,%s,%s,%s,%s,,,,,,,,,,,\r\n" % (head + (ident,))
    if bds in (0x05, 0x06):
        if not st & FS_HAS_POS:
            return None
        alt = 0 if bds == 0x06 else int(r["altitude"])
        return "MSG,%i,0,%i,%06X,%i,%s,%s,%s,%s,,%i,,,%.5f,%.5f,,,,0,0,0\r\n" % (
            (2 if bds == 0x06 else 3,) + head + (alt, float(r["lat"]), float(r["lon"])))
    if bds == 0x09 and int(r["subtype"]) == 1:
        v = r["val"]
        return "MSG,4,0,%i,%06X,%i,%s,%s,%s,%s,,,%.1f,%.1f,,,%i,,,,,\r\n" % (head + (float(v[0]), float(v[1]), float(v[2])))
    return None                                         # BDS0,9 subtypes 0 and 3, BDS6,1


class Sbs1Checker:
    """One decoder's SBS-1 stage: feed(frames, records) per decode call returns that call's text (bytes)."""

    def __init__(self, tz: int = 0):
        self.tz = tz
        self.reset()

    def reset(self):
        self.ids = {}                                   # address -> id
        self.n = 0                                      # ids handed out since the reset

    def aircraft_id(self, icao):
        """Rule 2: the id is live when it is in the map and id > n - 10000."""
        i = self.ids.get(icao)
        if i is not None and i > self.n - WINDOW:
            return i
        self.n += 1
        self.ids[icao] = self.n
        return self.n

    def feed(self, frames, recs, ids_out=None) -> bytes:
        out = []
        for f, r in zip(frames, recs):
            if not published(r):
                continue
            i = self.aircraft_id(int(r["icao"]))
            if ids_out is not None:
                ids_out.append(i)
            date, tod = stamp(int(f["secs"]), float(f["frac"]), self.tz)
            s = line(r, i, date, tod)
            if s is not None:
                out.append(s)
        return "".join(out).encode("ascii")
