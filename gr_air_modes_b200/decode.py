"""Batch field decode on the GPU (SURVEY.md 8 row f4): the host-side mirror of what the reference does per message
in Python after the slicer.

  parse.modes_reply(...) field tables, decode_id            python/parse.py:27-254
  altitude.decode_alt                                       python/altitude.py:28-108
  parse.parseBDS05/06/08/09_0/09_1/09_3/62, parseMB_*       python/parse.py:256-420
  cpr.cpr_decoder(my_location).decode(...)                  python/cpr.py:183-240

`batch_decoder` plays the role of one `cpr_decoder` plus the parser: feed it the frames (or the message strings) of a
stretch of the stream in order, get one record per message (struct amb_fields, include/airmodes_b200.h). All
arithmetic runs in libairmodes_b200.so on the GPU; there is no CPU implementation behind this module.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import Aircraft, Fields, Frame, check

FS_NO_HANDLER, FS_METRIC_ALT, FS_CPR_NO_POS, FS_CPR_STRADDLE = 0x01, 0x02, 0x04, 0x08
FS_HAS_POS, FS_HAS_RANGE, FS_METRIC_THREAT, FS_NOT_QUEUED = 0x10, 0x20, 0x40, 0x80
NO_ALTITUDE = -(1 << 31)
# local CPR outcome of a record (decoder option local_cpr; include/airmodes_b200.h AMB_LOCAL_*), read by local_outcome()
LOCAL_NOT_TRIED, LOCAL_DECODED, LOCAL_NO_REF, LOCAL_STALE, LOCAL_REJECTED = (
    _lib.LOCAL_NOT_TRIED, _lib.LOCAL_DECODED, _lib.LOCAL_NO_REF, _lib.LOCAL_STALE, _lib.LOCAL_REJECTED)
LOCAL_CPR_MAX = _lib.LOCAL_CPR_MAX
# Comm-B inference outcome of a record (decoder option commb; include/airmodes_b200.h AMB_COMMB_*), read by commb_outcome()
COMMB_NOT_TRIED, COMMB_DECODED, COMMB_RESOLVED, COMMB_AMBIGUOUS, COMMB_NONE = (
    _lib.COMMB_NOT_TRIED, _lib.COMMB_DECODED, _lib.COMMB_RESOLVED, _lib.COMMB_AMBIGUOUS, _lib.COMMB_NONE)
COMMB_MAX = _lib.COMMB_MAX
# per-aircraft table (decoder option track; include/airmodes_b200.h amb_aircraft, AMB_AC_*)
AC_HAS_ALT, AC_HAS_SQUAWK, AC_HAS_IDENT, AC_HAS_POS, AC_HAS_RANGE = (
    _lib.AC_HAS_ALT, _lib.AC_HAS_SQUAWK, _lib.AC_HAS_IDENT, _lib.AC_HAS_POS, _lib.AC_HAS_RANGE)
AC_HAS_VELOCITY, AC_HAS_HEADING, AC_HAS_EPS, AC_ON_GROUND = (
    _lib.AC_HAS_VELOCITY, _lib.AC_HAS_HEADING, _lib.AC_HAS_EPS, _lib.AC_ON_GROUND)
TRACK_MAX = _lib.TRACK_MAX

FIELDS_DTYPE = np.dtype(Fields)
FRAME_DTYPE = np.dtype(Frame)
AIRCRAFT_DTYPE = np.dtype(Aircraft)


def frames_from_messages(msgs):
    """The slicer's message strings "<hex> <crc> <ref> <secs> <frac>" (slicer_impl.cc:186-192) -> Frame array,
    i.e. what make_parser's publish() splits (parse.py:425). Every message counts as queued (passed = 1)."""
    msgs = list(msgs)
    arr = (Frame * max(len(msgs), 1))()
    for k, m in enumerate(msgs):
        if isinstance(m, str):
            data, ecc, ref, secs, frac = m.split()
            ecc, ref, secs, frac = int(ecc, 16), float(ref), int(secs), float(frac)
        else:                                   # (hex, ecc, secs, frac) tuples
            data, ecc, secs, frac = m
            ref = 0.0
        raw = bytes.fromhex(data)
        f = arr[k]
        f.nbits = 8 * len(raw)
        for i, b in enumerate(raw):
            f.data[i] = b
        f.crc, f.ref_level, f.secs, f.frac, f.passed = ecc, ref, secs, frac, 1
        f.df = raw[0] >> 3
    return arr, len(msgs)


def local_outcome(records):
    """AMB_FIELDS_LOCAL of a FIELDS_DTYPE record or array: LOCAL_* per record (the low byte of `pad_`)."""
    return np.asarray(records["pad_"], dtype=np.uint64) & np.uint64(0xFF)


# the decoder options (amb_decoder_set_option) and their maxima in seconds
OPTION_MAX = {"local_cpr": LOCAL_CPR_MAX, "track": TRACK_MAX, "commb": COMMB_MAX}


def check_option(name: str, seconds) -> int:
    """Validate a setting of decoder option `name`: an int in 0 (off) .. OPTION_MAX[name] seconds. Raises ValueError
    otherwise."""
    top = OPTION_MAX[name]
    try:
        ok = not isinstance(seconds, bool) and int(seconds) == seconds and 0 <= int(seconds) <= top
    except (TypeError, ValueError):
        ok = False
    if not ok:
        raise ValueError("%s: an integer number of seconds in 0 (off) .. %d, got %r" % (name, top, seconds))
    return int(seconds)


# check_option bound to one option, under the names the module has always exported
def check_local_cpr(seconds) -> int:
    return check_option("local_cpr", seconds)


def check_commb(seconds) -> int:
    return check_option("commb", seconds)


def check_track(seconds) -> int:
    return check_option("track", seconds)


def commb_outcome(records):
    """AMB_FIELDS_COMMB of a FIELDS_DTYPE record or array: COMMB_* per record (byte 1 of `pad_`)."""
    return (np.asarray(records["pad_"], dtype=np.uint64) >> np.uint64(8)) & np.uint64(0xFF)


# commb_values: per register, the names of fields 0..4 and their LSBs (include/airmodes_b200.h, DESIGN.md §8)
COMMB_FIELDS = {
    0x40: (("mcp_alt", 16.0), ("fms_alt", 16.0), ("baro", 0.1), ("modes", 1), ("alt_source", 1)),
    0x50: (("roll", 45.0 / 256), ("track", 90.0 / 512), ("gs", 2.0), ("track_rate", 8.0 / 256), ("tas", 2.0)),
    0x60: (("heading", 90.0 / 512), ("ias", 1.0), ("mach", 2.048 / 512), ("baro_rate", 32.0), ("inertial_rate", 32.0)),
}


def commb_values(record):
    """The register a DECODED / RESOLVED record carries, as named physical values: {"bds": 0x40 / 0x50 / 0x60, name:
    value or None for an absent field}. Degrees, knots, feet, mb (baro = 800 + 0.1 raw), Mach, ft/min and deg/s; the
    mode bits (VNAV = 4, ALT = 2, APP = 1) and the target altitude source stay integers. None for any other record.
    `record`: a FIELDS_DTYPE record or the dict from record_to_dict()."""
    pad = int(record["pad_"])
    if (pad >> 8) & 0xFF not in (COMMB_DECODED, COMMB_RESOLVED):
        return None
    reg, mask = (pad >> 16) & 0xFF, (pad >> 24) & 0xFF
    words = [int(x) for x in record["aux"]]
    raw = [((words[i // 2] >> (16 * (i % 2))) & 0xFFFF) for i in range(5)]
    raw = [x - 0x10000 if x & 0x8000 else x for x in raw]
    out = {"bds": reg}
    for i, (name, lsb) in enumerate(COMMB_FIELDS[reg]):
        if not mask & (1 << i):
            out[name] = None
        elif isinstance(lsb, int):
            out[name] = raw[i]
        else:
            out[name] = raw[i] * lsb + (800.0 if name == "baro" else 0.0)
    return out


# aircraft_to_dict: a column and the flag that says it is set
_AC_COLUMNS = (("altitude", AC_HAS_ALT), ("squawk", AC_HAS_SQUAWK), ("ident", AC_HAS_IDENT), ("ftc", AC_HAS_IDENT),
               ("cat", AC_HAS_IDENT), ("lat", AC_HAS_POS), ("lon", AC_HAS_POS), ("pos_t", AC_HAS_POS),
               ("range", AC_HAS_RANGE), ("bearing", AC_HAS_RANGE), ("speed", AC_HAS_VELOCITY),
               ("vertical", AC_HAS_VELOCITY), ("heading", AC_HAS_HEADING), ("eps", AC_HAS_EPS))


def aircraft_to_dict(row) -> dict:
    """One AIRCRAFT_DTYPE row -> plain dict for JSON: ident as str, a column whose flag is clear as None, on_ground as
    bool, and rssi = 10 log10(max(1e-8, ref_level)) as the reference computes it from the slicer's level (parse.py:430)."""
    flags = int(row["flags"])
    d = {"icao": int(row["icao"]), "messages": int(row["messages"]), "first_seen": float(row["first_seen"]),
         "seen": float(row["seen"]), "rssi": 10.0 * math.log10(max(1e-8, float(row["ref_level"]))),
         "flags": flags, "on_ground": bool(flags & AC_ON_GROUND)}
    for name, flag in _AC_COLUMNS:
        if not flags & flag:
            d[name] = None
        elif name == "ident":
            d[name] = np.asarray(row["ident"]).tobytes().rstrip(b"\0").decode("ascii", "replace")
        else:
            d[name] = row[name].item()
    return d


class batch_decoder:
    """cpr_decoder(my_location) (cpr.py:184-190) + parser, for batches. my_location = [lat, lon] or None.

    local_cpr = S > 0 also decodes every position message the global decode leaves without a fix relative to the
    aircraft's last position of at most S seconds before (DESIGN.md §8); 0, the default, is the reference's decoder.
    track = S > 0 also keeps a per-aircraft table on the device, read with aircraft() / aircraft_device(): one row per
    address heard in a DF17 squitter, dropped S seconds after its last message (DESIGN.md §8 "Aircraft table").
    commb = S > 0 also infers the register (BDS 4,0 / 5,0 / 6,0) of the DF20/21 replies the parser does not handle,
    with the address's ADS-B velocity of at most S seconds before deciding between 5,0 and the others; read with
    commb_outcome() / commb_values() (DESIGN.md §8 "Comm-B inference")."""

    def __init__(self, my_location=None, device: int = 0, local_cpr: int = 0, track: int = 0, commb: int = 0):
        settings = {"local_cpr": check_option("local_cpr", local_cpr), "track": check_option("track", track),
                    "commb": check_option("commb", commb)}
        self._lib = _lib.load()
        h = C.c_void_p()
        have, lat, lon = self._loc(my_location)
        rc = self._lib.amb_decoder_create(int(device), have, lat, lon, C.byref(h))
        if rc < 0:
            detail = self._lib.amb_decoder_last_error(None).decode()
            raise RuntimeError("libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(), (" (%s)" % detail) if detail else ""))
        self._h = h
        self._device = int(device)
        self.my_location = my_location
        self._options = dict.fromkeys(OPTION_MAX, 0)
        for name, seconds in settings.items():
            if seconds:
                self._set_option(name, seconds)

    @staticmethod
    def _loc(loc):
        return (0, 0.0, 0.0) if loc is None else (1, float(loc[0]), float(loc[1]))

    def _check(self, rc):
        if rc < 0:
            detail = self._lib.amb_decoder_last_error(self._h).decode()
            raise RuntimeError("libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(),
                                                           (" (%s)" % detail) if detail else ""))
        return rc

    def set_location(self, new_location):       # cpr.py:192-193
        self._check(self._lib.amb_decoder_set_location(self._h, *self._loc(new_location)))
        self.my_location = new_location

    def reset(self):
        """Forget every stored report, reference position, velocity and aircraft; the option settings stay."""
        self._check(self._lib.amb_decoder_reset(self._h))

    def _set_option(self, name, seconds):
        seconds = check_option(name, seconds)
        self._check(self._lib.amb_decoder_set_option(self._h, name.encode(), seconds))
        self._options[name] = seconds

    def set_local_cpr(self, seconds: int):
        """Option local_cpr = S seconds (0 = off); applies from the next decode."""
        self._set_option("local_cpr", seconds)

    def get_local_cpr(self) -> int:
        return self._options["local_cpr"]

    def set_track(self, seconds: int):
        """Option track = S seconds (0 = off); applies from the next decode."""
        self._set_option("track", seconds)

    def get_track(self) -> int:
        return self._options["track"]

    def set_commb(self, seconds: int):
        """Option commb = S seconds (0 = off); applies from the next decode."""
        self._set_option("commb", seconds)

    def get_commb(self) -> int:
        return self._options["commb"]

    @staticmethod
    def _now(now):
        return math.nan if now is None else float(now)

    def aircraft(self, now=None) -> np.ndarray:
        """The aircraft table at time `now` (None: the t of the latest queued message decoded since reset): every row
        heard within the last S seconds up to `now`, in ascending address, as a numpy AIRCRAFT_DTYPE array."""
        now = self._now(now)
        n = self._check(self._lib.amb_decoder_aircraft(self._h, now, None, 0))
        out = np.zeros(n, dtype=AIRCRAFT_DTYPE)
        if n:
            n = self._check(self._lib.amb_decoder_aircraft(self._h, now, C.c_void_p(out.ctypes.data), n))
        return out[:n]

    def aircraft_device(self, now=None, out_dev=None):
        """aircraft() into device memory: returns a CUDA uint8 tensor of 128-byte amb_aircraft rows (a view of the
        first rows of out_dev when one is given). Only the row count crosses PCIe."""
        import torch
        now = self._now(now)
        if out_dev is None:
            n = self._check(self._lib.amb_decoder_aircraft_device(self._h, now, None, 0))
            out_dev = torch.empty(n * 128, dtype=torch.uint8, device=torch.device("cuda", self._device))
        torch.cuda.current_stream(out_dev.device).synchronize()          # the decoder runs on its own stream
        n = self._check(self._lib.amb_decoder_aircraft_device(self._h, now, C.c_void_p(out_dev.data_ptr()),
                                                              int(out_dev.numel() // 128)))
        return out_dev[: n * 128]

    def decode(self, frames, n: int | None = None) -> np.ndarray:
        """frames: ctypes Frame array / list of Frame (e.g. rx_path.frames) / numpy FRAME_DTYPE array, in stream
        order. Returns a numpy structured array (FIELDS_DTYPE), one record per frame."""
        if isinstance(frames, np.ndarray):
            a = np.ascontiguousarray(frames, dtype=FRAME_DTYPE)
            n = a.size if n is None else n
            ptr, keep = C.c_void_p(a.ctypes.data), a
        else:
            if isinstance(frames, (list, tuple)):
                n = len(frames) if n is None else n
                arr = (Frame * max(n, 1))(*frames[:n])
            else:
                arr = frames
                n = len(arr) if n is None else n
            ptr, keep = C.cast(arr, C.c_void_p), arr
        out = np.zeros(n, dtype=FIELDS_DTYPE)
        if n:
            self._check(self._lib.amb_decode_frames(self._h, ptr, int(n), _lib.MEM_HOST, C.c_void_p(out.ctypes.data)))
        del keep
        return out

    def decode_device(self, frames_dev, out_dev=None):
        """frames_dev: torch CUDA uint8 tensor holding n amb_frame records (80 bytes each) in stream order; returns (or
        fills) a CUDA uint8 tensor of n amb_fields records (144 bytes each). Nothing crosses PCIe."""
        import torch
        n = frames_dev.numel() // 80
        if out_dev is None:
            out_dev = torch.empty(n * 144, dtype=torch.uint8, device=frames_dev.device)
        if n:
            torch.cuda.current_stream(frames_dev.device).synchronize()      # the decoder runs on its own stream
            self._check(self._lib.amb_decode_frames_device(self._h, C.c_void_p(frames_dev.data_ptr()), int(n),
                                                           C.c_void_p(out_dev.data_ptr())))
        return out_dev

    def decode_messages(self, msgs) -> np.ndarray:
        arr, n = frames_from_messages(msgs)
        return self.decode(arr, n)

    def stats(self):
        k, ms = C.c_uint64(), C.c_float()
        self._check(self._lib.amb_decoder_stats(self._h, C.byref(k), C.byref(ms)))
        return int(k.value), float(ms.value)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.amb_decoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class cpr_decoder:
    """Drop-in for the reference's `air_modes.cpr_decoder(my_location)` (python/cpr.py:183-240; constructed at
    apps/modes_rx:69, used by parseBDS05/06, parse.py:285,291): the same two methods, the same return list
    `[lat, lon, range, bearing]` and the same exceptions, one message per call - so the reference's unmodified
    output plugins can run on top of the GPU decoder. Reports are aged with `clock()` (default time.time, exactly
    as cpr.py:219-221 does). For throughput use batch_decoder; this class is the compatibility surface."""

    def __init__(self, my_location, device: int = 0, clock=None, _backend=None):
        import time
        self.my_location = my_location
        self._clock = clock or time.time
        self._dec = _backend if _backend is not None else batch_decoder(my_location, device)
        self._arr = (Frame * 1)()

    def set_location(self, new_location):                       # cpr.py:192-193
        self.my_location = new_location
        self._dec.set_location(new_location)

    def decode(self, icao24, encoded_lat, encoded_lon, cpr_format, surface):
        from .errors import CPRBoundaryStraddleError, CPRNoPositionError
        now = float(self._clock())
        f = self._arr[0]
        # a DF17 extended squitter carrying exactly this report: ME type 11 (airborne) / 6 (surface), parse.py:124-127
        me = ((6 if surface else 11) << 51) | ((1 if cpr_format else 0) << 34) | ((int(encoded_lat) & 0x1FFFF) << 17) \
            | (int(encoded_lon) & 0x1FFFF)
        raw = bytes([17 << 3]) + (int(icao24) & 0xFFFFFF).to_bytes(3, "big") + me.to_bytes(7, "big") + b"\0\0\0"
        for i, b in enumerate(raw):
            f.data[i] = b
        f.nbits, f.df, f.passed, f.crc = 112, 17, 1, 0
        f.secs = int(now)
        f.frac = now - int(now)
        r = self._dec.decode(self._arr, 1)[0]
        st = int(r["status"])
        if st & FS_CPR_STRADDLE:
            raise CPRBoundaryStraddleError
        if not (st & FS_HAS_POS):
            raise CPRNoPositionError
        if st & FS_HAS_RANGE:
            return [float(r["lat"]), float(r["lon"]), float(r["range"]), float(r["bearing"])]
        return [float(r["lat"]), float(r["lon"]), None, None]

    def close(self):
        if hasattr(self._dec, "close"):
            self._dec.close()


def record_to_dict(rec) -> dict:
    """One FIELDS_DTYPE record -> plain dict (ident as str, arrays as lists)."""
    d = {}
    for name in FIELDS_DTYPE.names:
        v = rec[name]
        if name == "ident":
            v = np.asarray(v).tobytes().rstrip(b"\0").decode("ascii")
        elif isinstance(v, np.ndarray):
            v = v.tolist()
        else:
            v = v.item()
        d[name] = v
    return d


def frame_bits(frame: Frame, start: int, num: int) -> int:
    """data_field.get_bits(start, num) on a frame's payload (parse.py:71-87), for raw sub-fields."""
    return int(_lib.load().amb_frame_bits(C.byref(frame), int(start), int(num)))
