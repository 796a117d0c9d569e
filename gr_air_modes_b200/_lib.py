"""ctypes binding of libairmodes_b200.so (include/airmodes_b200.h).

There is no CPU implementation behind this module: if the CUDA library cannot be loaded, or no sm_90
device is present, the constructors raise RuntimeError. That is deliberate (BASELINE north_star: no CPU
fallback); nothing here imports or calls oracle/.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libairmodes_b200.so")

OK = 0
MEM_HOST, MEM_DEVICE, MEM_HOST_SC16, MEM_DEVICE_SC16 = 0, 1, 2, 3
# amb_frame.ec (include/airmodes_b200.h AMB_EC_*)
EC_NOT_TRIED, EC_FIXED, EC_TOO_MANY, EC_NO_SOLUTION, EC_AMBIGUOUS = 0, 1, 2, 3, 4
EC_MAX = 23
EC_ANY_MAX = 2              # option "ec_any": at most 2 flipped bits
# AMB_FRAME_AP (include/airmodes_b200.h AMB_AP_*), option "ap_filter" = S seconds (0 = off)
AP_NOT_CHECKED, AP_KNOWN, AP_UNKNOWN = 0, 1, 2
AP_FILTER_MAX = 3600
# AMB_FIELDS_LOCAL (include/airmodes_b200.h AMB_LOCAL_*), decoder option "local_cpr" = S seconds (0 = off)
LOCAL_NOT_TRIED, LOCAL_DECODED, LOCAL_NO_REF, LOCAL_STALE, LOCAL_REJECTED = 0, 1, 2, 3, 4
LOCAL_CPR_MAX = 600
# AMB_FIELDS_COMMB (include/airmodes_b200.h AMB_COMMB_*), decoder option "commb" = S seconds (0 = off)
COMMB_NOT_TRIED, COMMB_DECODED, COMMB_RESOLVED, COMMB_AMBIGUOUS, COMMB_NONE = 0, 1, 2, 3, 4
COMMB_MAX = 600
# AMB_FIELDS_ES (include/airmodes_b200.h AMB_ES_*), decoder option "opstatus" = S seconds (0 = off)
ES_NOT_TRIED, ES_OPSTATUS, ES_TARGET_STATE, ES_NIC, ES_NUC, ES_UNSUPPORTED = 0, 1, 2, 3, 4, 5
ES_NO_VERSION = 0xFF
OPSTATUS_MAX = 600
# amb_aircraft.flags (include/airmodes_b200.h AMB_AC_*), decoder option "track" = S seconds (0 = off)
AC_HAS_ALT, AC_HAS_SQUAWK, AC_HAS_IDENT, AC_HAS_POS, AC_HAS_RANGE = 0x001, 0x002, 0x004, 0x008, 0x010
AC_HAS_VELOCITY, AC_HAS_HEADING, AC_HAS_EPS, AC_ON_GROUND = 0x020, 0x040, 0x080, 0x100
TRACK_MAX = 3600
# amb_aircraft_ext.shown (include/airmodes_b200.h AMB_AXG_*), decoder option "track_ext" = S2 seconds (0 = off)
AXG_OPS, AXG_TS, AXG_INTEG, AXG_B40, AXG_B50, AXG_B60 = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20
AXG_N = 6
TRACK_EXT_MAX = 3600
# SBS-1 feed (decoder options sbs1, sbs1_tz; include/airmodes_b200.h AMB_SBS1_TZ_*)
SBS1_TZ_MIN, SBS1_TZ_MAX = -720, 840
# coverage map (decoder option coverage; include/airmodes_b200.h AMB_COVERAGE_*)
COVERAGE_ROWS, COVERAGE_BANDS = 72, 9
COVERAGE_ALTITUDES = (0, 1000, 2000, 5000, 10000, 15000, 20000, 25000, 30000)
ERR_INVALID = -1                 # AMB_ERR_INVALID
ERR_OVERFLOW = -5                # AMB_ERR_OVERFLOW: the buffer is too small (amb_decoder_sbs1 reports the size needed)
ERR_STATE = -8                   # AMB_ERR_STATE: not valid in this state (e.g. a call after flush without reset)
BEAST_CARRY_MAX = 43             # AMB_BEAST_CARRY_MAX
BEAST_PUSH_MAX = 0x7FFF0000      # AMB_BEAST_PUSH_MAX


class Frame(C.Structure):
    """struct amb_frame (80 bytes) = modes_packet (types.h:29-41) + preamble tag.

    The header's `ec`, `ec_flips` and the four bytes of its `pad_[4]` (AMB_FRAME_EC_ANY / AMB_FRAME_EC_ANY_BIT /
    AMB_FRAME_AP) are the six tail bytes, which stay one `pad_` field here: the record layout that numpy views and per-field dumps of frames see (np.dtype(Frame)) is
    the one the frame had before error correction existed. They are read through the properties below."""
    _fields_ = [("sample_index", C.c_uint64), ("secs", C.c_uint64), ("frac", C.c_double),
                ("ref_level", C.c_float), ("crc", C.c_uint32), ("nbits", C.c_uint8), ("df", C.c_uint8),
                ("numlowconf", C.c_uint8), ("passed", C.c_uint8), ("lowconfbits", C.c_uint8 * 24),
                ("data", C.c_uint8 * 14), ("pad_", C.c_uint8 * 6)]

    @property
    def ec(self) -> int:
        """amb_frame.ec: error-correction outcome, EC_* (0 unless option "ec" tried this frame)."""
        return self.pad_[0]

    @property
    def ec_flips(self) -> int:
        """amb_frame.ec_flips: bits the correction flipped (EC_FIXED), else 0."""
        return self.pad_[1]

    @property
    def ec_any(self) -> int:
        """AMB_FRAME_EC_ANY (byte 76): outcome of the second pass (option "ec_any"): EC_NOT_TRIED, EC_FIXED or EC_NO_SOLUTION."""
        return self.pad_[2]

    @property
    def ec_any_bits(self) -> tuple:
        """AMB_FRAME_EC_ANY_BIT(f, 0..1) (bytes 77-78): the two positions that pass flipped, ascending; 0 = unused slot."""
        return (self.pad_[3], self.pad_[4])

    @property
    def ap(self) -> int:
        """AMB_FRAME_AP (byte 79): address/parity check (option "ap_filter"): AP_NOT_CHECKED, AP_KNOWN or AP_UNKNOWN."""
        return self.pad_[5]

    def payload(self) -> bytes:
        return bytes(self.data[: self.nbits // 8])


class Stats(C.Structure):
    _fields_ = [("samples_in", C.c_uint64), ("candidates", C.c_uint64), ("candidates_real", C.c_uint64),
                ("detections", C.c_uint64), ("frames_passed", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("ms_scan", C.c_float), ("ms_total", C.c_float), ("resolver_fallback", C.c_int),
                ("ec_fixed", C.c_int)]


class Geometry(C.Structure):
    _fields_ = [("samples_per_chip", C.c_float), ("samples_per_symbol", C.c_float), ("threshold", C.c_float),
                ("rate_int", C.c_int), ("history", C.c_int), ("check_width", C.c_int), ("pulse_offset", C.c_int * 4),
                ("quiet_a", C.c_int * 2), ("quiet_b", C.c_int * 2), ("max_late", C.c_int), ("packet_skip", C.c_int),
                ("pmf_len", C.c_int), ("floor_len", C.c_int), ("chip_offset_239", C.c_int),
                ("shard_back", C.c_int), ("shard_fwd", C.c_int)]


class WalkState(C.Structure):
    """struct amb_walk_state: where preamble_impl::general_work's loop stands (preamble_impl.cc:164,237)."""
    _fields_ = [("pos", C.c_int64), ("p", C.c_int64)]


class WalkSummary(C.Structure):
    """struct amb_walk_summary (speculative resolution of a time-sharded span)."""
    _fields_ = [("pos", C.c_int64), ("p", C.c_int64), ("first_real", C.c_int64), ("first_packet", C.c_int64),
                ("exact_span", C.c_int64), ("frames_passed", C.c_int64)]


class Fields(C.Structure):
    """struct amb_fields (144 bytes): one decoded message (parse.py / altitude.py / cpr.py results).

    The first byte of the header's `pad_` (AMB_FIELDS_LOCAL) holds the local CPR outcome; `pad_` stays one uint64 field
    here, so the record layout numpy sees (np.dtype(Fields)) is the one it had before local decoding existed."""
    _fields_ = [("icao", C.c_uint32), ("ecc", C.c_uint32), ("df", C.c_uint8), ("status", C.c_uint8), ("bds", C.c_uint8),
                ("subtype", C.c_uint8), ("ca", C.c_uint8), ("fs", C.c_uint8), ("vs", C.c_uint8), ("ri", C.c_uint8),
                ("sl", C.c_uint8), ("cc", C.c_uint8), ("dr", C.c_uint8), ("um", C.c_uint8), ("ftc", C.c_uint8),
                ("cat", C.c_uint8), ("cpr_format", C.c_uint8), ("surface", C.c_uint8), ("eps", C.c_uint8),
                ("ast", C.c_uint8), ("bds2", C.c_uint8), ("tti", C.c_uint8), ("altitude", C.c_int32),
                ("squawk", C.c_int32), ("threat_alt", C.c_int32), ("cpr_lat", C.c_uint32), ("cpr_lon", C.c_uint32),
                ("aux", C.c_uint32 * 4), ("ident", C.c_char * 8), ("lat", C.c_double), ("lon", C.c_double),
                ("range", C.c_double), ("bearing", C.c_double), ("val", C.c_double * 4), ("pad_", C.c_uint64)]

    @property
    def local(self) -> int:
        """AMB_FIELDS_LOCAL (byte 136): local CPR outcome (decoder option "local_cpr"), LOCAL_*."""
        return self.pad_ & 0xFF

    @property
    def commb(self) -> int:
        """AMB_FIELDS_COMMB (byte 137): Comm-B inference outcome (decoder option "commb"), COMMB_*."""
        return (self.pad_ >> 8) & 0xFF

    @property
    def es(self) -> int:
        """AMB_FIELDS_ES (byte 141): op status / integrity outcome (decoder option "opstatus"), ES_*."""
        return (self.pad_ >> 40) & 0xFF


class Aircraft(C.Structure):
    """struct amb_aircraft (128 bytes): one row of the decoder's per-aircraft table (option "track")."""
    _fields_ = [("icao", C.c_uint32), ("messages", C.c_uint32), ("first_seen", C.c_double), ("seen", C.c_double),
                ("ref_level", C.c_float), ("flags", C.c_uint16), ("ftc", C.c_int8), ("cat", C.c_int8),
                ("ident", C.c_char * 8), ("altitude", C.c_int32), ("squawk", C.c_int32), ("lat", C.c_double),
                ("lon", C.c_double), ("range", C.c_double), ("bearing", C.c_double), ("pos_t", C.c_double),
                ("speed", C.c_double), ("heading", C.c_double), ("vertical", C.c_double), ("eps", C.c_int8),
                ("pad_", C.c_uint8 * 15)]


class AircraftExt(C.Structure):
    """struct amb_aircraft_ext (144 bytes): the op-status and Comm-B groups beside one aircraft row (option
    "track_ext"); t[i] is the time of the group with bit 1 << i."""
    _fields_ = [("icao", C.c_uint32), ("shown", C.c_uint8), ("ops_version", C.c_uint8), ("integ_es", C.c_uint8),
                ("integ_version", C.c_uint8), ("t", C.c_double * 6), ("ops", C.c_uint32 * 4), ("ts", C.c_uint32 * 4),
                ("integ", C.c_uint32 * 2), ("integ_nic", C.c_uint8), ("commb_mask", C.c_uint8 * 3),
                ("commb_outcome", C.c_uint8 * 3), ("pad0_", C.c_uint8), ("commb", (C.c_int16 * 5) * 3),
                ("pad_", C.c_uint8 * 10)]


class MlatFix(C.Structure):
    """struct amb_mlat_fix (112 bytes): one multilateration fix (include/airmodes_b200.h amb_mlat)."""
    _fields_ = [("data", C.c_uint8 * 14), ("nbits", C.c_uint8), ("df", C.c_uint8), ("addr", C.c_uint32),
                ("status", C.c_uint8), ("n", C.c_uint8), ("steps", C.c_uint8), ("ref", C.c_uint8),
                ("stations", C.c_uint32), ("altitude", C.c_int32), ("secs", C.c_uint64), ("frac", C.c_double),
                ("lat", C.c_double), ("lon", C.c_double), ("height", C.c_double), ("x", C.c_double), ("y", C.c_double),
                ("z", C.c_double), ("rms", C.c_double), ("dop", C.c_double)]


class MlatCounts(C.Structure):
    """struct amb_mlat_counts (80 bytes): amb_mlat_stats."""
    _fields_ = [("eligible", C.c_uint64), ("carried", C.c_uint64), ("solved", C.c_uint64),
                ("no_convergence", C.c_uint64), ("degenerate", C.c_uint64), ("too_few", C.c_uint64),
                ("duplicate", C.c_uint64), ("span", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("ms_last", C.c_float), ("pad_", C.c_uint32)]


class BeastCounts(C.Structure):
    """struct amb_beast_counts (72 bytes): amb_beast_reader_stats."""
    _fields_ = [("bytes_in", C.c_uint64), ("modes", C.c_uint64), ("modeac", C.c_uint64), ("other", C.c_uint64),
                ("truncated", C.c_uint64), ("skipped", C.c_uint64), ("passed", C.c_uint64), ("carried", C.c_uint64),
                ("kernel_launches", C.c_uint64)]


# amb_mlat_fix.status (include/airmodes_b200.h AMB_MLAT_*)
MLAT_SOLVED, MLAT_NO_CONVERGENCE, MLAT_DEGENERATE = 1, 2, 3
MLAT_MIN_STATIONS, MLAT_MAX_STATIONS = 3, 32

assert C.sizeof(Frame) == 80
assert C.sizeof(Fields) == 144
assert C.sizeof(Aircraft) == 128
assert C.sizeof(AircraftExt) == 144
assert C.sizeof(MlatFix) == 112
assert C.sizeof(MlatCounts) == 80
assert C.sizeof(BeastCounts) == 72


class ModeacStats(C.Structure):
    _fields_ = [("candidates", C.c_uint64), ("replies", C.c_uint64), ("overlap_drops", C.c_uint64), ("with_altitude", C.c_uint64)]

assert C.sizeof(ModeacStats) == 32

# every symbol include/airmodes_b200.h declares: (name, restype, argtypes)
_vp, _f32p, _u64p = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_uint64)
SYMBOLS = [
    ("amb_create", C.c_int, [C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.POINTER(_vp)]),
    ("amb_destroy", None, [_vp]),
    ("amb_reset", C.c_int, [_vp]),
    ("amb_set_rate", C.c_int, [_vp, C.c_float]),
    ("amb_set_threshold", C.c_int, [_vp, C.c_float]),
    ("amb_get_rate", C.c_float, [_vp]),
    ("amb_get_threshold", C.c_float, [_vp]),
    ("amb_get_pmf", C.c_int, [_vp]),
    ("amb_set_start_time", C.c_int, [_vp, C.c_uint64, C.c_double]),
    ("amb_query_geometry", C.c_int, [C.c_float, C.c_float, C.c_int, C.POINTER(Geometry)]),
    ("amb_process", C.c_int, [_vp, _vp, C.c_size_t, C.c_int, C.c_int]),
    ("amb_poll_frames", C.c_int, [_vp, C.POINTER(Frame), C.c_int]),
    ("amb_pending_frames", C.c_int, [_vp]),
    ("amb_poll_ready", C.c_int, [_vp, C.POINTER(Frame), C.c_int]),
    ("amb_drain_device", C.c_int, [_vp, _vp, C.c_int]),
    ("amb_add_time_tag", C.c_int, [_vp, C.c_uint64, C.c_uint64, C.c_double]),
    ("amb_wait_stream", C.c_int, [_vp, _vp]),
    ("amb_format_message", C.c_int, [C.POINTER(Frame), C.c_int, C.c_char_p, C.c_size_t]),
    ("amb_format_messages", C.c_int, [_vp, C.c_int, C.c_int, C.c_char_p, C.c_size_t]),
    ("amb_modes_check_crc", C.c_uint32, [C.c_char_p, C.c_int]),
    ("amb_device_crc", C.c_int, [_vp, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_uint32)]),
    ("amb_preamble_process", C.c_int, [_vp, _f32p, _f32p, C.c_size_t, C.c_int, _f32p, _u64p, C.c_int]),
    ("amb_slicer_process", C.c_int, [_vp, _f32p, C.c_int, _u64p, C.POINTER(C.c_double), C.POINTER(Frame)]),
    ("amb_set_stream", C.c_int, [_vp, _vp]),
    ("amb_enable_timing", C.c_int, [_vp, C.c_int]),
    ("amb_get_stats", C.c_int, [_vp, C.POINTER(Stats)]),
    ("amb_get_scan_times", C.c_int, [_vp, _f32p, C.c_int]),
    ("amb_get_timeline", C.c_int, [_vp, _f32p, C.c_int]),
    ("amb_synchronize", C.c_int, [_vp]),
    ("amb_join", C.c_int, [_vp]),
    ("amb_debug_candidates", C.c_int, [_vp, _u64p, C.POINTER(C.c_uint32), C.c_int]),
    ("amb_set_option", C.c_int, [_vp, C.c_char_p, C.c_int]),
    ("amb_poll_modeac", C.c_int, [_vp, _vp, C.c_int]),
    ("amb_pending_modeac", C.c_int, [_vp]),
    ("amb_drain_modeac_device", C.c_int, [_vp, _vp, C.c_int]),
    ("amb_get_modeac_stats", C.c_int, [_vp, C.POINTER(ModeacStats)]),
    ("amb_dump_stage", C.c_int, [_vp, C.c_int, _f32p, C.c_size_t, _f32p]),
    ("amb_seek", C.c_int, [_vp, C.c_uint64, C.c_uint64, C.POINTER(WalkState)]),
    ("amb_resolve", C.c_int, [_vp, C.POINTER(WalkState)]),
    ("amb_get_walk_state", C.c_int, [_vp, C.POINTER(WalkState)]),
    ("amb_get_walk_summary", C.c_int, [_vp, C.POINTER(WalkSummary)]),
    ("amb_walk_summary_async", C.c_int, [_vp, _vp]),
    ("amb_compose_entries_async", C.c_int, [_vp, _vp, C.c_int, _vp, _vp]),
    ("amb_resolve_device", C.c_int, [_vp, _vp, _vp]),
    ("amb_join_stream", C.c_int, [_vp, _vp]),
    ("amb_decoder_create", C.c_int, [C.c_int, C.c_int, C.c_double, C.c_double, C.POINTER(_vp)]),
    ("amb_decoder_set_option", C.c_int, [_vp, C.c_char_p, C.c_int]),
    ("amb_decoder_destroy", None, [_vp]),
    ("amb_decoder_set_location", C.c_int, [_vp, C.c_int, C.c_double, C.c_double]),
    ("amb_decoder_reset", C.c_int, [_vp]),
    ("amb_decode_frames", C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp]),
    ("amb_decode_frames_device", C.c_int, [_vp, _vp, C.c_int, _vp]),
    ("amb_decoder_aircraft", C.c_int, [_vp, C.c_double, _vp, C.c_int]),
    ("amb_decoder_aircraft_device", C.c_int, [_vp, C.c_double, _vp, C.c_int]),
    ("amb_decoder_aircraft_ext", C.c_int, [_vp, C.c_double, _vp, _vp, C.c_int]),
    ("amb_decoder_aircraft_ext_device", C.c_int, [_vp, C.c_double, _vp, _vp, C.c_int]),
    ("amb_decoder_sbs1", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_sbs1_device", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_reports", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_reports_device", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_beast", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_beast_device", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_avr", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_avr_device", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_flightgear", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_flightgear_device", C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("amb_decoder_coverage", C.c_int, [_vp, _vp]),
    ("amb_decoder_coverage_device", C.c_int, [_vp, _vp]),
    ("amb_decoder_coverage_reset", C.c_int, [_vp]),
    ("amb_decoder_stats", C.c_int, [_vp, _u64p, _f32p]),
    ("amb_decoder_last_error", C.c_char_p, [_vp]),
    ("amb_mlat_create", C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                  C.POINTER(C.c_double), C.POINTER(_vp)]),
    ("amb_mlat_destroy", None, [_vp]),
    ("amb_mlat_set_option", C.c_int, [_vp, C.c_char_p, C.c_double]),
    ("amb_mlat_get_option", C.c_int, [_vp, C.c_char_p, C.POINTER(C.c_double)]),
    ("amb_mlat_set_offset", C.c_int, [_vp, C.c_int, C.c_double]),
    ("amb_mlat_reset", C.c_int, [_vp]),
    ("amb_mlat_process", C.c_int, [_vp, C.POINTER(_vp), C.POINTER(C.c_int), C.c_uint64, C.c_double, C.c_int, _vp,
                                   C.c_int, C.POINTER(C.c_int)]),
    ("amb_mlat_process_device", C.c_int, [_vp, C.POINTER(_vp), C.POINTER(C.c_int), C.c_uint64, C.c_double, C.c_int,
                                          _vp, C.c_int, C.POINTER(C.c_int)]),
    ("amb_mlat_stats", C.c_int, [_vp, C.POINTER(MlatCounts)]),
    ("amb_mlat_last_error", C.c_char_p, [_vp]),
    ("amb_beast_reader_create", C.c_int, [C.c_int, C.POINTER(_vp)]),
    ("amb_beast_reader_destroy", None, [_vp]),
    ("amb_beast_reader_reset", C.c_int, [_vp]),
    ("amb_beast_reader_push", C.c_int, [_vp, _vp, C.c_size_t, C.c_int, C.c_int]),
    ("amb_beast_reader_frames", C.c_int, [_vp, _vp, C.c_int]),
    ("amb_beast_reader_frames_device", C.c_int, [_vp, _vp, C.c_int]),
    ("amb_beast_reader_stats", C.c_int, [_vp, C.POINTER(BeastCounts)]),
    ("amb_beast_reader_last_error", C.c_char_p, [_vp]),
    ("amb_frame_bits", C.c_uint64, [C.POINTER(Frame), C.c_int, C.c_int]),
    ("amb_strerror", C.c_char_p, [C.c_int]),
    ("amb_last_error", C.c_char_p, [_vp]),
    ("amb_version", C.c_char_p, []),
]

_lib = None


def load() -> C.CDLL:
    """Load the CUDA library or raise; never falls back to anything else."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libairmodes_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                           "this package has no CPU fallback")
    try:
        lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    except OSError as first:
        # libcudart.so.12 ships inside the torch wheel set; make it resolvable and retry once
        try:
            import glob
            import sysconfig
            for pat in ("nvidia/cuda_runtime/lib/libcudart.so.12", "torch/lib/libcudart*.so*"):
                for path in glob.glob(os.path.join(sysconfig.get_paths()["purelib"], pat)):
                    C.CDLL(path, mode=C.RTLD_GLOBAL)
            lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        except OSError:
            raise RuntimeError("cannot load libairmodes_b200.so: %s" % first) from first
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)      # AttributeError here means the header and the library disagree
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def check(rc: int, ctx=None) -> int:
    if rc < 0:
        lib = load()
        msg = lib.amb_strerror(rc).decode()
        if ctx:
            detail = lib.amb_last_error(ctx).decode()
            if detail:
                msg += " (%s)" % detail
        raise RuntimeError("libairmodes_b200: " + msg)
    return rc
