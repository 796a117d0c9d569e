"""Multilateration across synchronized receivers (include/airmodes_b200.h amb_mlat, DESIGN.md §8 "Multilateration").

K receivers that share a GPS-disciplined clock hear the same transmission at different times; those differences, with
the barometric altitude the reply carries, locate the aircraft. This is what the reference's mlat.py sets out to do,
for transponders that never broadcast a position (DF4/DF20 altitude replies) as well as for ADS-B. Frames of the K
receivers go in (host arrays or the CUDA tensors `rx_path.drain_device` returns); the grouping and the solve run on the
device, and fixes come out as a numpy structured array (np.dtype(MlatFix)).

    m = mlat_solver([(lat, lon, height_m), ...])
    fixes = m.process([frames_0, frames_1, ...], end=(secs, frac))
    m.process([...], flush=True)

There is no CPU path: without the CUDA library or an sm_90 device the constructor raises. `llh2ecef` and `ecef2llh`
below are the reference's host geodesy (mlat.py:58-86), for callers and tests.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import Frame, MlatCounts, MlatFix, MLAT_SOLVED, MLAT_NO_CONVERGENCE, MLAT_DEGENERATE

__all__ = ["mlat_solver", "fix_to_dict", "llh2ecef", "ecef2llh", "FIX_DTYPE", "SPEED_OF_LIGHT",
           "MLAT_SOLVED", "MLAT_NO_CONVERGENCE", "MLAT_DEGENERATE"]

SPEED_OF_LIGHT = 299792458 / 1.0003          # mlat.py:95, in air
WGS84_A, WGS84_B, WGS84_E2 = 6378137.0, 6356752.314245, 0.0066943799901975848
FIX_DTYPE = np.dtype(MlatFix)
STATUS_NAMES = {MLAT_SOLVED: "solved", MLAT_NO_CONVERGENCE: "no_convergence", MLAT_DEGENERATE: "degenerate"}
_FRAME = C.sizeof(Frame)


def llh2ecef(lat, lon, height):
    """Geodetic (degrees, degrees, m above the WGS84 ellipsoid) to ECEF m, as mlat.py:77-86 computes it."""
    la, lo = lat * (math.pi / 180.0), lon * (math.pi / 180.0)
    sl = math.sin(la)
    n = WGS84_A / math.sqrt(1 - WGS84_E2 * (sl * sl))
    return ((n + height) * math.cos(la) * math.cos(lo), (n + height) * math.cos(la) * math.sin(lo),
            (n * (1 - WGS84_E2) + height) * sl)


def ecef2llh(x):
    """ECEF m to (lat, lon, height): Bowring's one-step form of mlat.py:58-75."""
    a, b = WGS84_A, WGS84_B
    ep = math.sqrt((a * a - b * b) / (b * b))
    p = math.sqrt(x[0] * x[0] + x[1] * x[1])
    th = math.atan2(a * x[2], b * p)
    lon = math.atan2(x[1], x[0])
    st, ct = math.sin(th), math.cos(th)
    lat = math.atan2(x[2] + ep * ep * b * (st * st * st), p - WGS84_E2 * a * (ct * ct * ct))
    sl = math.sin(lat)
    n = a / math.sqrt(1 - WGS84_E2 * (sl * sl))
    return lat * (180.0 / math.pi), lon * (180.0 / math.pi), p / math.cos(lat) - n


def fix_to_dict(fix) -> dict:
    """One row of the fixes array as a plain dict (the JSON line of tools/mlat_b200.py)."""
    nbits = int(fix["nbits"])
    return {"status": STATUS_NAMES.get(int(fix["status"]), int(fix["status"])), "df": int(fix["df"]),
            "addr": "%06x" % int(fix["addr"]), "payload": bytes(fix["data"][: nbits // 8]).hex(),
            "stations": [k for k in range(32) if (int(fix["stations"]) >> k) & 1], "ref": int(fix["ref"]),
            "n": int(fix["n"]), "steps": int(fix["steps"]), "altitude_ft": int(fix["altitude"]),
            "secs": int(fix["secs"]), "frac": float(fix["frac"]), "lat": float(fix["lat"]), "lon": float(fix["lon"]),
            "height": float(fix["height"]), "ecef": [float(fix["x"]), float(fix["y"]), float(fix["z"])],
            "rms": float(fix["rms"]), "dop": float(fix["dop"])}


def _end(end, flush):
    if end is None:
        if not flush:
            raise ValueError("process: give end=(secs, frac) or flush=True")
        return 0, 0.0
    secs, frac = end
    return int(secs), float(frac)


class mlat_solver:
    """K stations = [(lat, lon, height_m), ...] (3 <= K <= 32, heights above the ellipsoid). window_us: the grouping
    window W (default: the longest baseline / c + 2 us). offsets: per-station clock offsets in seconds."""

    def __init__(self, stations, device: int = 0, window_us=None, offsets=None):
        st = [tuple(float(v) for v in s) for s in stations]
        if any(len(s) != 3 for s in st):
            raise ValueError("stations: (lat, lon, height) each")
        self.K = len(st)
        self.stations = st
        self._lib = _lib.load()
        arr = C.c_double * max(1, self.K)
        h = C.c_void_p()
        rc = self._lib.amb_mlat_create(int(device), self.K, arr(*[s[0] for s in st]), arr(*[s[1] for s in st]),
                                       arr(*[s[2] for s in st]), C.byref(h))
        if rc < 0:
            detail = self._lib.amb_mlat_last_error(None).decode()
            raise (ValueError if rc == _lib.ERR_INVALID else RuntimeError)(
                "libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(), (" (%s)" % detail) if detail else ""))
        self._h = h
        self._device = int(device)
        self._cap = 0
        self._out = None
        if window_us is not None:
            self.set_window_us(window_us)
        for k, off in enumerate(offsets or []):
            self.set_offset(k, off)

    def _check(self, rc):
        if rc < 0:
            detail = self._lib.amb_mlat_last_error(self._h).decode()
            msg = "libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(), (" (%s)" % detail) if detail else "")
            raise ValueError(msg) if rc == _lib.ERR_INVALID else RuntimeError(msg)
        return rc

    def set_window_us(self, us):
        self._check(self._lib.amb_mlat_set_option(self._h, b"window_us", float(us)))

    def get_window_us(self) -> float:
        v = C.c_double()
        self._check(self._lib.amb_mlat_get_option(self._h, b"window_us", C.byref(v)))
        return v.value

    def set_offset(self, k: int, seconds: float):
        self._check(self._lib.amb_mlat_set_offset(self._h, int(k), float(seconds)))

    def reset(self):
        """Drop the frames carried from earlier calls."""
        self._check(self._lib.amb_mlat_reset(self._h))

    def stats(self) -> dict:
        s = MlatCounts()
        self._check(self._lib.amb_mlat_stats(self._h, C.byref(s)))
        return {name: getattr(s, name) for name, _ in MlatCounts._fields_ if name != "pad_"}

    def _counts(self, per_station):
        if len(per_station) != self.K:
            raise ValueError("process: %d stations expected, %d given" % (self.K, len(per_station)))
        return (C.c_int * self.K)(*[int(n) for n in per_station])

    def _run(self, fn, ptrs, counts, end, flush, out_ptr, cap):
        secs, frac = _end(end, flush)
        n = C.c_int()
        rc = fn(self._h, ptrs, counts, secs, frac, 1 if flush else 0, out_ptr, int(cap), C.byref(n))
        return rc, n.value

    def process(self, frames_per_station, end=None, flush=False) -> np.ndarray:
        """frames_per_station[k]: station k's frames (ctypes Frame arrays or sequences, numpy arrays of np.dtype(Frame)
        or bytes of 80-byte records) in stream order. end = (secs, frac): every station has delivered every frame with
        t <= end; flush=True completes every run. Returns the fixes as a structured array."""
        bufs = [_as_frames(f) for f in frames_per_station]
        counts = self._counts([len(b) // _FRAME for b in bufs])
        keep = [(C.c_char * max(1, len(b))).from_buffer_copy(b if b else b"\0") for b in bufs]
        ptrs = (C.c_void_p * self.K)(*[C.addressof(k) for k in keep])
        # a transmission is a group only when three stations heard it: room for that many fixes mostly avoids a second
        # pass (an overflow changes nothing, and the call is made again with the count it reported)
        self._cap = max(self._cap, sum(counts) // 3 + 16)
        while True:
            out = np.zeros(max(1, self._cap), FIX_DTYPE)
            rc, n = self._run(self._lib.amb_mlat_process, ptrs, counts, end, flush, out.ctypes.data, self._cap)
            if rc == _lib.ERR_OVERFLOW:
                self._cap = max(n, 2 * self._cap)
                continue
            self._check(rc)
            return out[:n].copy()

    def process_device(self, frames_per_station, end=None, flush=False, out_dev=None):
        """The same with each station's frames a CUDA uint8 tensor of n * 80 bytes (what rx_path.drain_device returns);
        returns a CUDA uint8 tensor of fixes (n * 112 bytes) that never crossed PCIe. out_dev: a caller's tensor to
        write into (grown when too small)."""
        import torch
        dev = torch.device("cuda", self._device)
        tensors = []
        for t in frames_per_station:
            if not (t.is_cuda and t.dtype == torch.uint8 and t.numel() % _FRAME == 0):
                raise ValueError("process_device: CUDA uint8 tensors of 80-byte frames expected")
            tensors.append(t.contiguous())
        counts = self._counts([t.numel() // _FRAME for t in tensors])
        ptrs = (C.c_void_p * self.K)(*[t.data_ptr() for t in tensors])
        torch.cuda.current_stream(dev).synchronize()          # the stage runs on its own stream
        out = out_dev
        if out is None:
            out = torch.empty((sum(counts) // 3 + 16) * FIX_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        while True:
            cap = 0 if out is None else out.numel() // FIX_DTYPE.itemsize
            rc, n = self._run(self._lib.amb_mlat_process_device, ptrs, counts, end, flush,
                              None if out is None else out.data_ptr(), cap)
            if rc == _lib.ERR_OVERFLOW:
                out = torch.empty(max(n, 1) * FIX_DTYPE.itemsize, dtype=torch.uint8, device=dev)
                continue
            self._check(rc)
            return out[: n * FIX_DTYPE.itemsize]

    @staticmethod
    def fixes_from_device(t) -> np.ndarray:
        """A tensor process_device returned, copied to the host as a structured array."""
        return np.frombuffer(t.cpu().numpy().tobytes(), FIX_DTYPE).copy()

    def close(self):
        if getattr(self, "_h", None):
            self._lib.amb_mlat_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _as_frames(f) -> bytes:
    if isinstance(f, (bytes, bytearray, memoryview)):
        b = bytes(f)
    elif isinstance(f, np.ndarray):
        b = f.tobytes()
    elif isinstance(f, C.Array):
        b = bytes(f)
    else:
        b = b"".join(bytes(x) for x in f)
    if len(b) % _FRAME:
        raise ValueError("frames: whole 80-byte records expected")
    return b
