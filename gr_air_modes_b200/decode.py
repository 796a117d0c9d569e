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
import functools
import math

import numpy as np

from . import _lib
from ._lib import Aircraft, AircraftExt, Fields, Frame, check

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
# op status / integrity outcome of a record (decoder option opstatus; include/airmodes_b200.h AMB_ES_*), read by
# opstatus_outcome()
ES_NOT_TRIED, ES_OPSTATUS, ES_TARGET_STATE, ES_NIC, ES_NUC, ES_UNSUPPORTED = (
    _lib.ES_NOT_TRIED, _lib.ES_OPSTATUS, _lib.ES_TARGET_STATE, _lib.ES_NIC, _lib.ES_NUC, _lib.ES_UNSUPPORTED)
ES_NO_VERSION = _lib.ES_NO_VERSION
OPSTATUS_MAX = _lib.OPSTATUS_MAX
# per-aircraft table (decoder option track; include/airmodes_b200.h amb_aircraft, AMB_AC_*)
AC_HAS_ALT, AC_HAS_SQUAWK, AC_HAS_IDENT, AC_HAS_POS, AC_HAS_RANGE = (
    _lib.AC_HAS_ALT, _lib.AC_HAS_SQUAWK, _lib.AC_HAS_IDENT, _lib.AC_HAS_POS, _lib.AC_HAS_RANGE)
AC_HAS_VELOCITY, AC_HAS_HEADING, AC_HAS_EPS, AC_ON_GROUND = (
    _lib.AC_HAS_VELOCITY, _lib.AC_HAS_HEADING, _lib.AC_HAS_EPS, _lib.AC_ON_GROUND)
TRACK_MAX = _lib.TRACK_MAX
# extension of the per-aircraft table (decoder option track_ext; include/airmodes_b200.h amb_aircraft_ext, AMB_AXG_*)
AXG_OPS, AXG_TS, AXG_INTEG, AXG_B40, AXG_B50, AXG_B60 = (
    _lib.AXG_OPS, _lib.AXG_TS, _lib.AXG_INTEG, _lib.AXG_B40, _lib.AXG_B50, _lib.AXG_B60)
TRACK_EXT_MAX = _lib.TRACK_EXT_MAX
# SBS-1 feed (decoder options sbs1 and sbs1_tz; include/airmodes_b200.h AMB_SBS1_TZ_*)
SBS1_TZ_MIN, SBS1_TZ_MAX = _lib.SBS1_TZ_MIN, _lib.SBS1_TZ_MAX
# coverage map (decoder option coverage; include/airmodes_b200.h AMB_COVERAGE_*): 72 bearing rows of 5 degrees, and the
# upper edges in feet of the nine altitude bands (az_map.py:42)
COVERAGE_ROWS, COVERAGE_BANDS, COVERAGE_ALTITUDES = _lib.COVERAGE_ROWS, _lib.COVERAGE_BANDS, _lib.COVERAGE_ALTITUDES

FIELDS_DTYPE = np.dtype(Fields)
FRAME_DTYPE = np.dtype(Frame)
AIRCRAFT_DTYPE = np.dtype(Aircraft)
AIRCRAFT_EXT_DTYPE = np.dtype(AircraftExt)


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


# The decoder options (amb_decoder_set_option): name -> (kind, lowest, highest value). A "switch" is off or on; the
# other kinds take integers in the unit they name, "seconds" from 0 (off).
OPTIONS = {"local_cpr": ("seconds", 0, LOCAL_CPR_MAX), "track": ("seconds", 0, TRACK_MAX),
           "commb": ("seconds", 0, COMMB_MAX), "opstatus": ("seconds", 0, OPSTATUS_MAX),
           "track_ext": ("seconds", 0, TRACK_EXT_MAX), "sbs1": ("switch", 0, 1),
           "sbs1_tz": ("minutes", SBS1_TZ_MIN, SBS1_TZ_MAX), "coverage": ("switch", 0, 1), "reports": ("switch", 0, 1)}
# the maxima of the options in seconds
OPTION_MAX = {name: top for name, (kind, _, top) in OPTIONS.items() if kind == "seconds"}


def check_option(name: str, value) -> int:
    """Validate a setting of decoder option `name` (OPTIONS): a switch takes False / True or 0 / 1, the other kinds an
    int in their range. Returns it as an int; raises ValueError otherwise."""
    kind, low, top = OPTIONS[name]
    if kind == "switch":
        if isinstance(value, (bool, np.bool_)) or (isinstance(value, (int, np.integer)) and int(value) in (0, 1)):
            return int(value)
        raise ValueError("%s: False / True (0 / 1), got %r" % (name, value))
    try:
        ok = not isinstance(value, bool) and int(value) == value and low <= int(value) <= top
    except (TypeError, ValueError):
        ok = False
    if not ok:
        span = "0 (off) .. %d" % top if kind == "seconds" else "%d .. %d" % (low, top)
        raise ValueError("%s: an integer number of %s in %s, got %r" % (name, kind, span, value))
    return int(value)


# check_option bound to one option, under the names the module has always exported
check_local_cpr = functools.partial(check_option, "local_cpr")
check_commb = functools.partial(check_option, "commb")
check_track = functools.partial(check_option, "track")
check_opstatus = functools.partial(check_option, "opstatus")
check_sbs1 = functools.partial(check_option, "sbs1")
check_sbs1_tz = functools.partial(check_option, "sbs1_tz")
check_coverage = functools.partial(check_option, "coverage")
check_reports = functools.partial(check_option, "reports")


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


def opstatus_outcome(records):
    """AMB_FIELDS_ES of a FIELDS_DTYPE record or array: ES_* per record (byte 5 of `pad_`)."""
    return (np.asarray(records["pad_"], dtype=np.uint64) >> np.uint64(40)) & np.uint64(0xFF)


def _aux_bytes(record):
    return np.asarray([int(x) for x in record["aux"]], dtype="<u4").view(np.uint8)


def opstatus_values(record):
    """What the decoder option opstatus wrote into a record, as named values; None for a record it did not decode.
      OPSTATUS      {"kind": "opstatus", "version", "subtype" (0 airborne, 1 surface), "capability", "op_mode" (the
                    16-bit words)}, and for versions 1 and 2 "nic_a", "nacp", "gva", "sil", "hrd", "sil_supplement",
                    "nic_baro" (airborne) or "trk_hdg" (surface), "nic_c" and "length_width" (surface)
      TARGET_STATE  {"kind": "target_state", "version": 2, "alt_source" ("MCP/FCU" / "FMS"), "selected_alt" (ft),
                    "baro" (mb), "heading" (deg; None when absent), "nacp", "nic_baro", "sil", "sil_supplement",
                    "autopilot", "vnav", "alt_hold", "approach", "lnav" (bool, None when the mode status bit is 0),
                    "tcas" (bool)}
      NIC / NUC     {"kind": "nic" / "nuc", "version" (None when there is no op status), "nic" or "nucp", "nic_a",
                    "nic_b", "nic_c", "rc" (m, None when unknown)}
    `record`: a FIELDS_DTYPE record or the dict from record_to_dict()."""
    pad = int(record["pad_"])
    es, ver, nic = (pad >> 40) & 0xFF, (pad >> 48) & 0xFF, (pad >> 56) & 0xFF
    b = _aux_bytes(record)
    u16 = b.view("<u2")
    if es == ES_OPSTATUS:
        out = {"kind": "opstatus", "version": ver, "subtype": int(b[4]), "capability": int(u16[0]),
               "op_mode": int(u16[1])}
        if ver:
            out.update(nic_a=int(b[5]), nacp=int(b[6]), gva=int(b[7]), sil=int(b[8]), hrd=int(b[10]),
                       sil_supplement=int(b[11]))
            if b[4]:
                out.update(trk_hdg=int(b[9]), nic_c=int(b[12]), length_width=int(b[13]))
            else:
                out["nic_baro"] = int(b[9])
        return out
    if es == ES_TARGET_STATE:
        alt, baro, hdg, modes = int(u16[0]), int(u16[1]), int(u16[2]), int(b[12])
        valid = bool(modes & 0x80)
        out = {"kind": "target_state", "version": ver, "alt_source": "FMS" if b[7] else "MCP/FCU",
               "selected_alt": None if alt == 0 else (alt - 1) * 32, "baro": None if baro == 0 else 800.0 + (baro - 1) * 0.8,
               "heading": hdg * 180.0 / 256 if b[8] else None, "nacp": int(b[9]), "nic_baro": int(b[10]),
               "sil": int(b[11]), "sil_supplement": int(b[6])}
        for name, bit in (("autopilot", 0x40), ("vnav", 0x20), ("alt_hold", 0x10), ("approach", 0x04), ("lnav", 0x01)):
            out[name] = bool(modes & bit) if valid else None
        out["tcas"] = bool(modes & 0x02)
        return out
    if es in (ES_NIC, ES_NUC):
        rc = float(b[4:8].view("<f4")[0])
        return {"kind": "nic" if es == ES_NIC else "nuc", "version": None if ver == ES_NO_VERSION else ver,
                ("nic" if es == ES_NIC else "nucp"): nic, "nic_a": int(b[0]), "nic_b": int(b[1]), "nic_c": int(b[2]),
                "rc": None if math.isnan(rc) else rc}
    return None


# aircraft_to_dict: a column and the flag that says it is set
_AC_COLUMNS = (("altitude", AC_HAS_ALT), ("squawk", AC_HAS_SQUAWK), ("ident", AC_HAS_IDENT), ("ftc", AC_HAS_IDENT),
               ("cat", AC_HAS_IDENT), ("lat", AC_HAS_POS), ("lon", AC_HAS_POS), ("pos_t", AC_HAS_POS),
               ("range", AC_HAS_RANGE), ("bearing", AC_HAS_RANGE), ("speed", AC_HAS_VELOCITY),
               ("vertical", AC_HAS_VELOCITY), ("heading", AC_HAS_HEADING), ("eps", AC_HAS_EPS))


def coverage_to_dict(grid, location) -> dict:
    """A coverage grid (batch_decoder.coverage(): COVERAGE_ROWS x COVERAGE_BANDS ranges) -> plain dict for JSON:
      location  the receiver's [lat, lon] the ranges were measured from
      unit      "statute miles", the unit of the records' range (cpr.py:162)
      sectors   per row i: "bearing" 5 i, and the bearings [from, to) it holds, from = 5 i - 2.5 (357.5 for row 0), to =
                5 i + 2.5; a bearing b lands in row int(b + 2.5) // 5 % 72 with the sum in IEEE double, so a bearing
                within rounding of an edge may land on the other side (include/airmodes_b200.h rule 3)
      bands     per band j: "altitude" = COVERAGE_ALTITUDES[j] in feet; band j holds the greatest range of the positions
                at or below that altitude, and the last band that of every position ("altitude" null)
      ranges    the grid, ranges[row][band]; 0.0 where nothing was heard."""
    grid = np.asarray(grid, dtype=np.float64).reshape(COVERAGE_ROWS, COVERAGE_BANDS)
    sectors = [{"bearing": 5.0 * i, "from": 357.5 if i == 0 else 5.0 * i - 2.5, "to": 5.0 * i + 2.5}
               for i in range(COVERAGE_ROWS)]
    bands = [{"altitude": a if j < COVERAGE_BANDS - 1 else None} for j, a in enumerate(COVERAGE_ALTITUDES)]
    return {"location": None if location is None else [float(location[0]), float(location[1])],
            "unit": "statute miles", "sectors": sectors, "bands": bands, "altitudes": list(COVERAGE_ALTITUDES),
            "ranges": grid.tolist()}


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


# aircraft_ext_to_dict: the key of each group, in the order of the AXG_* bits
_AXG_KEYS = ("opstatus", "target_state", "integrity", "bds40", "bds50", "bds60")


def _group_record(ext, i) -> dict:
    """The `pad_` and `aux` slots of the record that wrote group i of an AIRCRAFT_EXT_DTYPE row, rebuilt from the copy
    the group keeps (every slot the group does not keep is 0)."""
    words = [0, 0, 0, 0]
    if i == 0:
        words, pad = [int(x) for x in ext["ops"]], (ES_OPSTATUS << 40) | (int(ext["ops_version"]) << 48)
    elif i == 1:
        words, pad = [int(x) for x in ext["ts"]], (ES_TARGET_STATE << 40) | (2 << 48)
    elif i == 2:
        words[:2] = [int(x) for x in ext["integ"]]
        pad = (int(ext["integ_es"]) << 40) | (int(ext["integ_version"]) << 48) | (int(ext["integ_nic"]) << 56)
    else:
        c = i - 3
        raw = [int(x) & 0xFFFF for x in ext["commb"][c]] + [0]
        words = [raw[0] | raw[1] << 16, raw[2] | raw[3] << 16, raw[4], 0]
        pad = (int(ext["commb_outcome"][c]) << 8) | ((0x40 + 0x10 * c) << 16) | (int(ext["commb_mask"][c]) << 24)
    return {"pad_": pad, "aux": words}


def aircraft_ext_to_dict(row, ext) -> dict:
    """One AIRCRAFT_DTYPE row and its AIRCRAFT_EXT_DTYPE extension -> aircraft_to_dict(row) plus the keys "opstatus",
    "target_state", "integrity", "bds40", "bds50" and "bds60": None for a group that is not shown, else {"t": the time of
    the record that wrote it} merged with opstatus_values() / commb_values() of that record."""
    d = aircraft_to_dict(row)
    shown = int(ext["shown"])
    for i, key in enumerate(_AXG_KEYS):
        if not shown & (1 << i):
            d[key] = None
            continue
        rec = _group_record(ext, i)
        d[key] = {"t": float(ext["t"][i]), **(opstatus_values(rec) if i < 3 else commb_values(rec))}
    return d


class batch_decoder:
    """cpr_decoder(my_location) (cpr.py:184-190) + parser, for batches. my_location = [lat, lon] or None.

    local_cpr = S > 0 also decodes every position message the global decode leaves without a fix relative to the
    aircraft's last position of at most S seconds before (DESIGN.md §8); 0, the default, is the reference's decoder.
    track = S > 0 also keeps a per-aircraft table on the device, read with aircraft() / aircraft_device(): one row per
    address heard in a DF17 squitter, dropped S seconds after its last message (DESIGN.md §8 "Aircraft table").
    commb = S > 0 also infers the register (BDS 4,0 / 5,0 / 6,0) of the DF20/21 replies the parser does not handle,
    with the address's ADS-B velocity of at most S seconds before deciding between 5,0 and the others; read with
    commb_outcome() / commb_values() (DESIGN.md §8 "Comm-B inference").
    opstatus = S > 0 also decodes the DF17 operational status (TC 31) and target state (TC 29 subtype 1) squitters, and
    gives every DF17 position its NIC and containment radius from the address's op status of at most S seconds before,
    or its NUCp; read with opstatus_outcome() / opstatus_values() (DESIGN.md §8 "Operational status and NIC").
    track_ext = S2 > 0, with track on, also keeps beside every aircraft row the latest op status, target state, position
    integrity and Comm-B 4,0 / 5,0 / 6,0 of the address, each shown for S2 seconds; read with aircraft_ext() /
    aircraft_ext_device() (DESIGN.md §8 "Aircraft table extension").
    sbs1 = True also writes, on the device, the SBS-1 (BaseStation) lines the reference's output_sbs1 would send for the
    decoded messages, with aircraft ids carried from call to call and the date and time of each frame's stamp shifted
    by sbs1_tz minutes; read the last decode's lines with sbs1_text() / sbs1_text_device() (DESIGN.md §8 "SBS-1
    feed").
    coverage = True also keeps, on the device, the reference's azimuth map model: the greatest range heard in every
    5-degree bearing sector for each of nine altitude bands, from the positions with a range (a receiver location is
    needed); read with coverage() / coverage_device(), clear with reset_coverage() (DESIGN.md §8 "Receiver
    coverage").
    reports = True also writes, on the device, the text reports the reference's stdout printer (msprint.py, what
    modes_rx prints by default) prints for the decoded messages: report.format_report of each frame's slicer text and
    its record, the stream's first queued message at the slicer's precision 6; read the last decode's lines with
    report_text() / report_text_device() (DESIGN.md §8 "Text reports")."""

    def __init__(self, my_location=None, device: int = 0, local_cpr: int = 0, track: int = 0, commb: int = 0,
                 opstatus: int = 0, track_ext: int = 0, sbs1=False, sbs1_tz: int = 0, coverage=False,
                 reports=False):
        values = dict(local_cpr=local_cpr, track=track, commb=commb, opstatus=opstatus, track_ext=track_ext, sbs1=sbs1,
                      sbs1_tz=sbs1_tz, coverage=coverage, reports=reports)
        settings = {name: check_option(name, values[name]) for name in OPTIONS}
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
        self._options = dict.fromkeys(OPTIONS, 0)
        for name, value in settings.items():
            if value:
                self._set_option(name, value)

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
        """Forget every stored report, reference position, velocity, op status and aircraft, and clear the coverage
        grid; the option settings stay."""
        self._check(self._lib.amb_decoder_reset(self._h))

    def _set_option(self, name, value):
        value = check_option(name, value)
        self._check(self._lib.amb_decoder_set_option(self._h, name.encode(), value))
        self._options[name] = value

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

    def set_opstatus(self, seconds: int):
        """Option opstatus = S seconds (0 = off); applies from the next decode."""
        self._set_option("opstatus", seconds)

    def get_opstatus(self) -> int:
        return self._options["opstatus"]

    def set_track_ext(self, seconds: int):
        """Option track_ext = S2 seconds (0 = off); applies from the next decode, while track is on too."""
        self._set_option("track_ext", seconds)

    def get_track_ext(self) -> int:
        return self._options["track_ext"]

    def set_sbs1(self, on):
        """Option sbs1 on (True) or off (False); applies from the next decode."""
        self._set_option("sbs1", on)

    def get_sbs1(self) -> bool:
        return bool(self._options["sbs1"])

    def set_sbs1_tz(self, minutes: int):
        """Option sbs1_tz = minutes added to UTC in the SBS-1 date and time (0 = UTC); applies from the next decode."""
        self._set_option("sbs1_tz", minutes)

    def get_sbs1_tz(self) -> int:
        return self._options["sbs1_tz"]

    def _text(self, fetch) -> bytes:
        n = C.c_size_t()
        rc = fetch(self._h, None, 0, C.byref(n))
        if rc == _lib.ERR_OVERFLOW:
            buf = C.create_string_buffer(n.value)
            self._check(fetch(self._h, buf, n.value, C.byref(n)))
            return buf.raw[: n.value]
        self._check(rc)
        return b""

    def _text_device(self, fetch, name, out_dev) -> int:
        import torch
        if out_dev.dtype != torch.uint8 or not out_dev.is_cuda or not out_dev.is_contiguous():
            raise ValueError("%s: out_dev must be a contiguous CUDA uint8 tensor" % name)
        n = C.c_size_t()
        torch.cuda.current_stream(out_dev.device).synchronize()          # the decoder runs on its own stream
        rc = fetch(self._h, C.c_void_p(out_dev.data_ptr()), int(out_dev.numel()), C.byref(n))
        if rc == _lib.ERR_OVERFLOW:
            raise RuntimeError("%s: %d bytes needed, out_dev holds %d" % (name, n.value, out_dev.numel()))
        self._check(rc)
        return int(n.value)

    def sbs1_text(self) -> bytes:
        """The SBS-1 lines of the last decode, concatenated ("\\r\\n" after each). Needs the option sbs1 on."""
        return self._text(self._lib.amb_decoder_sbs1)

    def sbs1_text_device(self, out_dev) -> int:
        """sbs1_text() into out_dev, a CUDA uint8 tensor; returns the byte count. Only the count crosses PCIe. Raises
        RuntimeError (with the size needed) when out_dev is too small."""
        return self._text_device(self._lib.amb_decoder_sbs1_device, "sbs1_text_device", out_dev)

    def set_reports(self, on):
        """Option reports on (True) or off (False); applies from the next decode."""
        self._set_option("reports", on)

    def get_reports(self) -> bool:
        return bool(self._options["reports"])

    def report_text(self) -> bytes:
        """The text reports of the last decode, concatenated ("\\n" after each line). Needs the option reports on."""
        return self._text(self._lib.amb_decoder_reports)

    def report_text_device(self, out_dev) -> int:
        """report_text() into out_dev, a CUDA uint8 tensor; returns the byte count. Only the count crosses PCIe. Raises
        RuntimeError (with the size needed) when out_dev is too small."""
        return self._text_device(self._lib.amb_decoder_reports_device, "report_text_device", out_dev)

    def set_coverage(self, on):
        """Option coverage on (True) or off (False); applies from the next decode. The grid is kept while it is off."""
        self._set_option("coverage", on)

    def get_coverage(self) -> bool:
        return bool(self._options["coverage"])

    def coverage(self) -> np.ndarray:
        """The coverage grid: a (COVERAGE_ROWS, COVERAGE_BANDS) float64 array, [bearing row, altitude band], statute
        miles; all zeros before the first decode with the option on. Needs the option coverage on."""
        out = np.zeros((COVERAGE_ROWS, COVERAGE_BANDS), dtype=np.float64)
        self._check(self._lib.amb_decoder_coverage(self._h, C.c_void_p(out.ctypes.data)))
        return out

    def coverage_device(self, out_dev=None):
        """coverage() into device memory: a CUDA float64 tensor of shape (COVERAGE_ROWS, COVERAGE_BANDS) (out_dev when
        one is given: contiguous, float64, that many elements). Nothing but the call crosses PCIe."""
        import torch
        if out_dev is None:
            out_dev = torch.empty((COVERAGE_ROWS, COVERAGE_BANDS), dtype=torch.float64,
                                  device=torch.device("cuda", self._device))
        if out_dev.dtype != torch.float64 or not out_dev.is_cuda or not out_dev.is_contiguous() or \
                out_dev.numel() != COVERAGE_ROWS * COVERAGE_BANDS:
            raise ValueError("coverage_device: out_dev must be a contiguous CUDA float64 tensor of %d elements"
                             % (COVERAGE_ROWS * COVERAGE_BANDS))
        torch.cuda.current_stream(out_dev.device).synchronize()          # the decoder runs on its own stream
        self._check(self._lib.amb_decoder_coverage_device(self._h, C.c_void_p(out_dev.data_ptr())))
        return out_dev

    def reset_coverage(self):
        """Clear the coverage grid and nothing else (az_map_model.reset, az_map.py:77-82). Needs the option on."""
        self._check(self._lib.amb_decoder_coverage_reset(self._h))

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

    def aircraft_ext(self, now=None):
        """aircraft(now) and the extension of every row: (AIRCRAFT_DTYPE rows, AIRCRAFT_EXT_DTYPE rows), ext[i] beside
        rows[i]. Needs the options track and track_ext on."""
        now = self._now(now)
        n = self._check(self._lib.amb_decoder_aircraft_ext(self._h, now, None, None, 0))
        out = np.zeros(n, dtype=AIRCRAFT_DTYPE)
        ext = np.zeros(n, dtype=AIRCRAFT_EXT_DTYPE)
        if n:
            n = self._check(self._lib.amb_decoder_aircraft_ext(self._h, now, C.c_void_p(out.ctypes.data),
                                                               C.c_void_p(ext.ctypes.data), n))
        return out[:n], ext[:n]

    def aircraft_ext_device(self, now=None, out_dev=None, ext_dev=None):
        """aircraft_ext() into device memory: returns two CUDA uint8 tensors, of 128-byte amb_aircraft rows and of
        144-byte amb_aircraft_ext rows (views of the first rows of out_dev / ext_dev when they are given; give both or
        neither). Only the row count crosses PCIe."""
        import torch
        now = self._now(now)
        if (out_dev is None) != (ext_dev is None):
            raise ValueError("aircraft_ext_device: give both out_dev and ext_dev, or neither")
        if out_dev is None:
            n = self._check(self._lib.amb_decoder_aircraft_ext_device(self._h, now, None, None, 0))
            dev = torch.device("cuda", self._device)
            out_dev = torch.empty(n * 128, dtype=torch.uint8, device=dev)
            ext_dev = torch.empty(n * 144, dtype=torch.uint8, device=dev)
        torch.cuda.current_stream(out_dev.device).synchronize()          # the decoder runs on its own stream
        cap = int(min(out_dev.numel() // 128, ext_dev.numel() // 144))
        n = self._check(self._lib.amb_decoder_aircraft_ext_device(self._h, now, C.c_void_p(out_dev.data_ptr()),
                                                                  C.c_void_p(ext_dev.data_ptr()), cap))
        return out_dev[: n * 128], ext_dev[: n * 144]

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
