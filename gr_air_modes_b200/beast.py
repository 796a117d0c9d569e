"""Beast binary input (include/airmodes_b200.h amb_beast_reader, DESIGN.md §8 "Beast input").

Most receivers in the field are an RTL-SDR stick running dump1090 or readsb, which serve their frames as Beast binary
on TCP port 30005. beast_reader parses such a byte stream on the device into amb_frame records - the same records
rx_path.drain_device gives - so that another receiver's frames reach the batch decoder, multilateration and every
output built on them.

    r = beast_reader()
    frames = r.process(chunk)                    # numpy FRAME_DTYPE array, in stream order
    t = r.process_device(cuda_bytes, flush=True) # CUDA uint8 tensor of n * 80 bytes: batch_decoder.decode_device input

A stream may be cut into calls anywhere: what cannot be decided yet is carried on the device. There is no CPU path:
without the CUDA library or an sm_90 device the constructor raises.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import BeastCounts, Frame

__all__ = ["beast_reader", "FRAME_DTYPE"]

FRAME_DTYPE = np.dtype(Frame)
_FRAME = C.sizeof(Frame)


class beast_reader:
    """A Beast binary byte stream on `device`, parsed on the device into frames."""

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = C.c_void_p()
        rc = self._lib.amb_beast_reader_create(int(device), C.byref(h))
        if rc < 0:
            detail = self._lib.amb_beast_reader_last_error(None).decode()
            raise RuntimeError("libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(),
                                                           (" (%s)" % detail) if detail else ""))
        self._h = h
        self._device = int(device)

    def _check(self, rc):
        if rc < 0:
            detail = self._lib.amb_beast_reader_last_error(self._h).decode()
            msg = "libairmodes_b200: %s%s" % (self._lib.amb_strerror(rc).decode(), (" (%s)" % detail) if detail else "")
            raise ValueError(msg) if rc == _lib.ERR_INVALID else RuntimeError(msg)
        return rc

    def _push(self, data, flush):
        """Hand the bytes to the library; returns the frame count. A CUDA tensor is read in place, after everything
        torch's current stream has queued (its producer included)."""
        if _is_tensor(data) and data.is_cuda:
            import torch
            if data.dtype != torch.uint8:
                raise ValueError("process: a CUDA tensor must be uint8")
            t = data.contiguous().view(-1)
            torch.cuda.current_stream(t.device).synchronize()
            return self._check(self._lib.amb_beast_reader_push(self._h, C.c_void_p(t.data_ptr() if t.numel() else None),
                                                               t.numel(), _lib.MEM_DEVICE, 1 if flush else 0))
        buf = _host_bytes(data)
        ptr = buf.ctypes.data if buf.size else None
        return self._check(self._lib.amb_beast_reader_push(self._h, C.c_void_p(ptr), buf.size, _lib.MEM_HOST,
                                                           1 if flush else 0))

    def process(self, data, flush: bool = False) -> np.ndarray:
        """The next bytes of the stream (bytes, bytearray, memoryview, a numpy uint8 array or a torch uint8 tensor,
        CUDA ones read in place); flush=True ends the stream. Returns this call's frames as a FRAME_DTYPE array."""
        n = self._push(data, flush)
        out = np.zeros(n, FRAME_DTYPE)
        if n:
            self._check(self._lib.amb_beast_reader_frames(self._h, C.c_void_p(out.ctypes.data), n))
        return out

    def process_device(self, data, flush: bool = False, out=None):
        """The same, with the frames returned as a CUDA uint8 tensor of n * 80 bytes that never crossed PCIe: the input
        of batch_decoder.decode_device and of mlat_solver.process_device. out: a caller's CUDA uint8 tensor to write
        into (a ValueError when it is too small)."""
        import torch
        n = self._push(data, flush)
        dev = torch.device("cuda", self._device)
        if out is None:
            out = torch.empty(n * _FRAME, dtype=torch.uint8, device=dev)
        elif not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()):
            raise ValueError("process_device: out must be a contiguous CUDA uint8 tensor")
        elif out.numel() < n * _FRAME:
            raise ValueError("process_device: out holds %d bytes, %d needed" % (out.numel(), n * _FRAME))
        if n:
            torch.cuda.current_stream(dev).synchronize()          # the library writes `out` on its own stream
            self._check(self._lib.amb_beast_reader_frames_device(self._h, C.c_void_p(out.data_ptr()),
                                                                 out.numel() // _FRAME))
        return out[: n * _FRAME]

    @staticmethod
    def frames_from_device(t) -> np.ndarray:
        """A tensor process_device returned, copied to the host as a FRAME_DTYPE array."""
        return np.frombuffer(t.cpu().numpy().tobytes(), FRAME_DTYPE).copy()

    def stats(self) -> dict:
        """Counters of the stream since create or reset (include/airmodes_b200.h amb_beast_counts)."""
        s = BeastCounts()
        self._check(self._lib.amb_beast_reader_stats(self._h, C.byref(s)))
        return {name: getattr(s, name) for name, _ in BeastCounts._fields_}

    def reset(self):
        """Start a new stream: the carry is dropped, offsets and counters restart, flush is undone."""
        self._check(self._lib.amb_beast_reader_reset(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.amb_beast_reader_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _is_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and hasattr(x, "is_cuda")


def _host_bytes(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        if data.dtype != np.uint8:
            raise ValueError("process: a numpy array must be uint8")
        return np.ascontiguousarray(data).reshape(-1)
    if _is_tensor(data):
        import torch
        if data.dtype != torch.uint8:
            raise ValueError("process: a tensor must be uint8")
        return data.contiguous().view(-1).numpy()
    if isinstance(data, (bytes, bytearray, memoryview)):
        return np.frombuffer(memoryview(data).cast("B"), np.uint8) if len(memoryview(data)) else np.zeros(0, np.uint8)
    raise ValueError("process: bytes, bytearray, memoryview, a numpy uint8 array or a torch uint8 tensor expected")
