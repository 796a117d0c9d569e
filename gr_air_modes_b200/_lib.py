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


class Frame(C.Structure):
    """struct amb_frame (80 bytes) = modes_packet (types.h:29-41) + preamble tag."""
    _fields_ = [("sample_index", C.c_uint64), ("secs", C.c_uint64), ("frac", C.c_double),
                ("ref_level", C.c_float), ("crc", C.c_uint32), ("nbits", C.c_uint8), ("df", C.c_uint8),
                ("numlowconf", C.c_uint8), ("passed", C.c_uint8), ("lowconfbits", C.c_uint8 * 24),
                ("data", C.c_uint8 * 14), ("pad_", C.c_uint8 * 6)]

    def payload(self) -> bytes:
        return bytes(self.data[: self.nbits // 8])


class Stats(C.Structure):
    _fields_ = [("samples_in", C.c_uint64), ("candidates", C.c_uint64), ("candidates_real", C.c_uint64),
                ("detections", C.c_uint64), ("frames_passed", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("ms_scan", C.c_float), ("ms_total", C.c_float), ("resolver_fallback", C.c_int),
                ("reserved_", C.c_int)]


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
    """struct amb_fields (144 bytes): one decoded message (parse.py / altitude.py / cpr.py results)."""
    _fields_ = [("icao", C.c_uint32), ("ecc", C.c_uint32), ("df", C.c_uint8), ("status", C.c_uint8), ("bds", C.c_uint8),
                ("subtype", C.c_uint8), ("ca", C.c_uint8), ("fs", C.c_uint8), ("vs", C.c_uint8), ("ri", C.c_uint8),
                ("sl", C.c_uint8), ("cc", C.c_uint8), ("dr", C.c_uint8), ("um", C.c_uint8), ("ftc", C.c_uint8),
                ("cat", C.c_uint8), ("cpr_format", C.c_uint8), ("surface", C.c_uint8), ("eps", C.c_uint8),
                ("ast", C.c_uint8), ("bds2", C.c_uint8), ("tti", C.c_uint8), ("altitude", C.c_int32),
                ("squawk", C.c_int32), ("threat_alt", C.c_int32), ("cpr_lat", C.c_uint32), ("cpr_lon", C.c_uint32),
                ("aux", C.c_uint32 * 4), ("ident", C.c_char * 8), ("lat", C.c_double), ("lon", C.c_double),
                ("range", C.c_double), ("bearing", C.c_double), ("val", C.c_double * 4), ("pad_", C.c_uint64)]


assert C.sizeof(Frame) == 80
assert C.sizeof(Fields) == 144

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
    ("amb_decoder_destroy", None, [_vp]),
    ("amb_decoder_set_location", C.c_int, [_vp, C.c_int, C.c_double, C.c_double]),
    ("amb_decoder_reset", C.c_int, [_vp]),
    ("amb_decode_frames", C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp]),
    ("amb_decode_frames_device", C.c_int, [_vp, _vp, C.c_int, _vp]),
    ("amb_decoder_stats", C.c_int, [_vp, _u64p, _f32p]),
    ("amb_decoder_last_error", C.c_char_p, [_vp]),
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
