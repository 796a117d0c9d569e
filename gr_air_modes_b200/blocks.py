"""Host-side mirror of the reference block surface for the Mode S receive hot path.

  air_modes.preamble(channel_rate, threshold_db)   include/gr_air_modes/preamble.h:36-45, lib/preamble_impl.cc:37-76
  air_modes.slicer(queue)                          include/gr_air_modes/slicer.h:37-42,  lib/slicer_impl.cc:46-63
  air_modes.rx_path(rate, threshold, queue, use_pmf=False, use_dcblock=False)   python/rx_path.py:25-87
  modes_check_crc(data, length)                    include/gr_air_modes/modes_crc.h:26

Same names, argument meaning and defaults. The GNU Radio scheduler is replaced by explicit
`process()` calls (a GNU Radio adapter that forwards work() to them lives in gr_adapter.py and is only
importable where gnuradio is). All arithmetic happens in libairmodes_b200.so on the GPU.
"""
from __future__ import annotations

import collections
import ctypes as C
import threading

import numpy as np

from . import _lib
from ._lib import Frame, Geometry, ModeacStats, Stats, WalkState, WalkSummary, check

# amb_modeac (include/airmodes_b200.h, option "modeac"): one Mode A/C reply, 48 bytes
MODEAC_DTYPE = np.dtype([("sample_index", "<u8"), ("secs", "<u8"), ("frac", "<f8"), ("peak", "<f4"), ("floor", "<f4"),
                         ("altitude", "<i4"), ("code", "<u2"), ("squawk", "<u2"), ("spi", "u1"), ("pad_", "u1", (7,))])
assert MODEAC_DTYPE.itemsize == 48
NO_ALTITUDE = -(1 << 31)    # AMB_NO_ALTITUDE


# ---------------------------------------------------------------------------------------------
# gr.msg_queue / gr.message stand-ins (radio.py:43,84-87 only uses handle/insert_tail/delete_head
# and msg.to_string()); a real gr.msg_queue can be passed instead wherever `queue` is accepted.
# ---------------------------------------------------------------------------------------------
class message:
    def __init__(self, s: str):
        self._s = s

    def to_string(self) -> str:
        return self._s


def message_from_string(s: str) -> message:
    return message(s)


class msg_queue:
    """gr.msg_queue stand-in (gnuradio/msg_queue.h): handle / insert_tail, delete_head (BLOCKS until a message is
    there, as gr.msg_queue.delete_head does - radio.py:84-87 relies on it), delete_head_nowait, empty_p, count, flush."""

    def __init__(self, limit: int = 0):
        self._q = collections.deque()
        self._limit = limit
        self._cv = threading.Condition()

    def handle(self, msg) -> None:
        with self._cv:
            self._q.append(msg)
            self._cv.notify()

    insert_tail = handle

    def delete_head_nowait(self):
        with self._cv:
            return self._q.popleft() if self._q else None

    def delete_head(self, timeout: float | None = None):
        """Blocks until a message arrives (timeout in seconds is an extension; None = wait for ever)."""
        with self._cv:
            if not self._cv.wait_for(lambda: len(self._q) > 0, timeout):
                return None
            return self._q.popleft()

    def empty_p(self) -> bool:
        return not self._q

    def count(self) -> int:
        return len(self._q)

    def flush(self) -> None:
        with self._cv:
            self._q.clear()

    def strings(self):
        return [m.to_string() for m in list(self._q)]


def _make_gr_message(queue, text: str):
    """Wrap `text` in whatever message type `queue` expects."""
    if isinstance(queue, msg_queue):
        return message(text)
    try:  # a real gnuradio msg_queue
        from gnuradio import gr  # type: ignore
        return gr.message_from_string(text)
    except Exception:
        return message(text)


def modes_check_crc(data, length: int | None = None) -> int:
    """modes_check_crc(unsigned char data[], int length) (lib/modes_crc.cc:55-63): CRC of the first
    `length` bytes. Host table routine exported by the library (the slicer kernel has its own device CRC)."""
    data = bytes(data)
    if length is None:
        length = len(data)
    return int(_lib.load().amb_modes_check_crc(data, length))


modes_crc = modes_check_crc


def query_geometry(rate, threshold_db=7.0, use_pmf=True) -> Geometry:
    """What preamble_impl::set_rate/set_threshold derive from the rate (preamble_impl.cc:56-68) plus the halos
    of a time-sharded span. Host only."""
    g = Geometry()
    check(_lib.load().amb_query_geometry(float(rate), float(threshold_db), int(bool(use_pmf)), C.byref(g)))
    return g


def _as_iq(iq):
    """Return (pointer, n_complex, mem_kind, keepalive) for numpy (host) or torch (host / CUDA) input.

    complex64 / interleaved float32 = gr_complex (rx_path.py:29); complex128 is narrowed to complex64; interleaved
    int16 I,Q (full scale 32768, the receivers' wire format) is shipped as it is and widened on the device. Anything
    else is refused: silently reinterpreting it would decode garbage."""
    try:
        import torch
        if isinstance(iq, torch.Tensor):
            t = iq
            if t.is_complex():
                t = torch.view_as_real(t.to(torch.complex64))
            if t.dtype == torch.int16:
                kind = _lib.MEM_DEVICE_SC16 if t.is_cuda else _lib.MEM_HOST_SC16
            elif t.dtype == torch.float32:
                kind = _lib.MEM_DEVICE if t.is_cuda else _lib.MEM_HOST
            else:
                raise TypeError("IQ tensor must be complex64 / complex128, interleaved float32 or interleaved int16, not %s" % t.dtype)
            t = t.contiguous()
            return C.c_void_p(t.data_ptr()), t.numel() // 2, kind, t
    except ImportError:
        pass
    a = np.asarray(iq)
    if a.dtype == np.complex128:
        a = a.astype(np.complex64)
    if a.dtype == np.complex64:
        a = np.ascontiguousarray(a).view(np.float32)
    if a.dtype == np.int16:
        a = np.ascontiguousarray(a).reshape(-1)
        return C.c_void_p(a.ctypes.data), a.size // 2, _lib.MEM_HOST_SC16, a
    if a.dtype != np.float32:
        raise TypeError("IQ array must be complex64 / complex128, interleaved float32 or interleaved int16, not %s" % a.dtype)
    a = np.ascontiguousarray(a).reshape(-1)
    return C.c_void_p(a.ctypes.data), a.size // 2, _lib.MEM_HOST, a


class _Context:
    """Owner of one amb_ctx (one IQ stream on one GPU)."""

    def __init__(self, rate, threshold_db, use_pmf, use_dcblock, device=0):
        self._lib = _lib.load()
        h = C.c_void_p()
        check(self._lib.amb_create(int(device), float(rate), float(threshold_db), int(bool(use_pmf)),
                                   int(bool(use_dcblock)), C.byref(h)))
        self._h = h
        self.device = int(device)
        self.ec = 0                 # option "ec" as last set (the library keeps it; there is no getter in the C ABI)
        self.ec_any = 0             # option "ec_any", likewise
        self.ap_filter = 0          # option "ap_filter", likewise

    def close(self):
        if getattr(self, "_h", None):
            self._lib.amb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def call(self, name, *args):
        return check(getattr(self._lib, name)(self._h, *args), self._h)

    def poll_array(self):
        """(ctypes Frame array, count) of everything pending, in stream order."""
        n = self.call("amb_pending_frames")
        buf = (Frame * max(n, 1))()
        got = self.call("amb_poll_frames", buf, n) if n else 0
        return buf, got

    def poll(self):
        buf, got = self.poll_array()
        return list(buf)[:got]

    def poll_ready_array(self, max_frames: int = 4096):
        """Non-blocking: (ctypes Frame array, count) of the frames whose calls have completed on the device. The
        array is reused from call to call."""
        buf = getattr(self, "_ready_buf", None)
        if buf is None or len(buf) < max_frames:
            buf = self._ready_buf = (Frame * max_frames)()
        got = self.call("amb_poll_ready", buf, max_frames)
        return buf, got

    def wait_stream(self, cuda_stream_ptr: int):
        """Order the context's work after everything enqueued so far on another CUDA stream."""
        self.call("amb_wait_stream", C.c_void_p(cuda_stream_ptr))

    def stats(self) -> Stats:
        s = Stats()
        self.call("amb_get_stats", C.byref(s))
        return s

    def scan_times_ms(self, max_n: int = 64):
        buf = (C.c_float * max_n)()
        n = self.call("amb_get_scan_times", buf, max_n)
        return [buf[i] for i in range(n)]

    def join(self):
        """Make the caller-visible CUDA stream wait for everything enqueued so far (no host sync)."""
        self.call("amb_join")

    def use_stream(self, cuda_stream_ptr: int):
        self.call("amb_set_stream", C.c_void_p(cuda_stream_ptr))


def format_message(frame: Frame, first: bool) -> str:
    buf = C.create_string_buffer(200)
    check(_lib.load().amb_format_message(C.byref(frame), int(first), buf, 200))
    return buf.value.decode()


class slicer:
    """air_modes.slicer(queue): turns 240-chip packets into queue messages (slicer_impl.cc:102-198).

    ec=K (1..23, extension; default 0 = off, the reference's behaviour): DF11/DF17 packets that fail only their CRC
    are corrected over at most K low-confidence bits when exactly one set of flips fits (see amb_frame.ec).
    ec_any=M (1 or 2, extension; default 0 = off): DF17 packets still dropped for their CRC after that are corrected
    by at most M flipped bits anywhere in 5..111, whatever their confidence (see AMB_FRAME_EC_ANY)."""

    def __init__(self, queue, device: int = 0, _ctx: _Context | None = None, ec: int = 0, ec_any: int = 0):
        self._queue = queue
        self._ctx = _ctx or _Context(4e6, 7.0, False, False, device)
        self._first = True          # d_payload precision: 6 until the first message (slicer_impl.cc:192)
        if ec:
            self.set_ec(ec)
        if ec_any:
            self.set_ec_any(ec_any)

    def set_ec(self, k: int):
        """Error correction over at most k low-confidence bits (0 = off); takes effect at the next call."""
        self._ctx.call("amb_set_option", b"ec", int(k))
        self._ctx.ec = int(k)

    def get_ec(self) -> int:
        return self._ctx.ec

    def set_ec_any(self, m: int):
        """DF17 correction by at most m (1, 2) bits anywhere in 5..111 (0 = off); takes effect at the next call."""
        self._ctx.call("amb_set_option", b"ec_any", int(m))
        self._ctx.ec_any = int(m)

    def get_ec_any(self) -> int:
        return self._ctx.ec_any

    def emit(self, frames, n: int | None = None) -> int:
        """Queue one message per frame that passed the slicer rules (slicer_impl.cc:186-194). Returns how many.
        `frames`: a ctypes Frame array (first n entries) or any sequence of Frame. The text of the whole batch is
        formatted by one library call."""
        if isinstance(frames, (list, tuple)):
            n = len(frames) if n is None else n
            frames = (Frame * max(n, 1))(*frames[:n])
        elif n is None:
            n = len(frames)
        if n == 0:
            return 0
        cap = 128 * n + 16
        buf = C.create_string_buffer(cap)
        k = check(_lib.load().amb_format_messages(C.cast(frames, C.c_void_p), int(n), int(self._first), buf, cap))
        if k:
            handle, q = self._queue.handle, self._queue
            for text in buf.value.decode("ascii").split("\n"):
                handle(_make_gr_message(q, text))
            self._first = False
        return k

    def process(self, chips, tags) -> list:
        """chips: (ndet, 240) float32 packets; tags: per packet (secs, frac) = the preamble_found tag value.
        Returns the frames (all packets; see .passed) after queueing the messages."""
        chips = np.ascontiguousarray(chips, dtype=np.float32).reshape(-1, 240)
        ndet = chips.shape[0]
        secs = np.ascontiguousarray([t[0] for t in tags], dtype=np.uint64)
        frac = np.ascontiguousarray([t[1] for t in tags], dtype=np.float64)
        out = (Frame * max(ndet, 1))()
        self._ctx.call("amb_slicer_process", chips.ctypes.data_as(C.POINTER(C.c_float)), ndet,
                       secs.ctypes.data_as(C.POINTER(C.c_uint64)), frac.ctypes.data_as(C.POINTER(C.c_double)), out)
        self.emit(out, ndet)
        return list(out)[:ndet]


class preamble:
    """air_modes.preamble(channel_rate, threshold_db) (preamble.h:39-45)."""

    def __init__(self, channel_rate, threshold_db, device: int = 0):
        self._ctx = _Context(channel_rate, threshold_db, False, False, device)

    def set_rate(self, channel_rate):
        self._ctx.call("amb_set_rate", float(channel_rate))

    def set_threshold(self, threshold_db):
        self._ctx.call("amb_set_threshold", float(threshold_db))

    def get_rate(self):
        return float(self._ctx._lib.amb_get_rate(self._ctx._h))

    def get_threshold(self):
        return float(self._ctx._lib.amb_get_threshold(self._ctx._h))

    def process(self, in0, in1, flush: bool = True, max_det: int | None = None):
        """Whole streams in0 (signal) / in1 (moving-average reference) -> (chips[ndet,240], tags) with
        tags = [(sample_index, secs, frac)], i.e. the 240-item packets and preamble_found tags of
        preamble_impl.cc:219-232."""
        in0 = np.ascontiguousarray(in0, dtype=np.float32)
        in1 = np.ascontiguousarray(in1, dtype=np.float32)
        n = min(in0.size, in1.size)
        if max_det is None:
            max_det = n // 200 + 16
        chips = np.empty((max_det, 240), np.float32)
        idx = np.empty(max_det, np.uint64)
        nd = self._ctx.call("amb_preamble_process", in0.ctypes.data_as(C.POINTER(C.c_float)),
                            in1.ctypes.data_as(C.POINTER(C.c_float)), n, int(flush),
                            chips.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_uint64)), max_det)
        rate = int(self.get_rate())
        tags = [(int(i), int(i) // rate, (int(i) % rate) / float(rate)) for i in idx[:nd]]
        return chips[:nd].copy(), tags


class rx_path:
    """air_modes.rx_path(rate, threshold, queue, use_pmf=False, use_dcblock=False) (rx_path.py:27).

    A sink of gr_complex: feed it with process(iq) (numpy complex64 / interleaved float32 on the host, or a
    torch CUDA tensor that is read in place). Decoded frames are pushed to `queue` as the reference's
    ASCII messages.

    ec=K (extension, default 0 = off): error correction over at most K (1..23) low-confidence bits of the DF11/DF17
    frames the reference drops for their CRC (slicer_impl.cc:182); a frame with exactly one fitting set of flips becomes
    an ordinary message with crc token 000000. Frames record the outcome in .ec / .ec_flips.

    ec_any=M (extension, default 0 = off): DF17 frames still dropped for their CRC after that are corrected by at most
    M (1, 2) flipped bits anywhere in 5..111, whatever their confidence; the one- and two-bit fits are unique there.
    Frames record the outcome in .ec_any / .ec_any_bits.

    ap_filter=S (extension, default 0 = off): address/parity check. Replies whose parity carries the address (DF0/4/5/
    16/20/21 and any other DF but 11/17) are dropped unless a CRC-clean DF11/DF17 frame of that address arrived in the
    last S seconds of the stream (counted in samples, S * int(rate)); DF11 replies whose parity carries a non-zero
    interrogator code (syndrome 1..0x7F) are accepted when their address is known that way. Frames record the outcome in
    .ap. reset() / set_rate() forget the confirmed addresses and keep the option. Not available with seek() /
    defer_resolve().

    modeac=True (extension, default off): also find Mode A/C replies (F1, 13 code pulses, F2 at 20.3 us, SPI) in the same
    front end, by the rules of include/airmodes_b200.h; modeac() / modeac_device() return them in stream order. Set
    before the first process() of a stream (set_modeac); kept across reset() / set_rate(). Not available with seek() /
    defer_resolve()."""

    def __init__(self, rate, threshold, queue, use_pmf=False, use_dcblock=False, device: int = 0, ec: int = 0,
                 ec_any: int = 0, ap_filter: int = 0, modeac: bool = False):
        self._rate = int(rate)                      # rx_path.py:32
        self._threshold = threshold
        self._queue = queue
        self._spc = int(rate / 2e6)                 # rx_path.py:35
        self._use_pmf = bool(use_pmf)
        self._ctx = _Context(rate, threshold, use_pmf, use_dcblock, device)
        self._slicer = slicer(queue, device, _ctx=self._ctx, ec=ec, ec_any=ec_any)
        if ap_filter:
            self.set_ap_filter(ap_filter)
        self._modeac = False
        if modeac:
            self.set_modeac(True)
        self.frames = []                            # every detection of the last process() call
        self._keep = []                             # device inputs still being read

    # -- the reference's methods (rx_path.py:67-87)
    def set_rate(self, rate):
        self._ctx.call("amb_set_rate", float(int(rate)))    # rx_path.py:68 passes int(rate)
        self._rate = int(rate)
        self._spc = int(rate / 2e6)

    def set_threshold(self, threshold):
        self._ctx.call("amb_set_threshold", float(threshold))
        self._threshold = threshold

    def set_start_time(self, secs: int, frac: float):
        """rx_time tag of the stream's first item (what a UHD source provides; preamble_impl.cc:164-170)."""
        self._ctx.call("amb_set_start_time", int(secs), float(frac))

    def set_pmf(self, pmf):
        pass                                        # rx_path.py:79-81: "must be done when top block is stopped"

    def get_pmf(self, pmf=None):
        return bool(self._ctx._lib.amb_get_pmf(self._ctx._h))

    def get_threshold(self):
        return float(self._ctx._lib.amb_get_threshold(self._ctx._h))

    # -- extension: error correction (see the class docstring); persists across reset() and set_rate()
    def set_ec(self, k: int):
        self._slicer.set_ec(k)

    def get_ec(self) -> int:
        return self._slicer.get_ec()

    def set_ec_any(self, m: int):
        self._slicer.set_ec_any(m)

    def get_ec_any(self) -> int:
        return self._slicer.get_ec_any()

    def set_ap_filter(self, seconds: int):
        """Address/parity check against the aircraft confirmed in the last `seconds` (0 = off, up to 3600); takes effect
        at the next call. Not available together with seek() / defer_resolve()."""
        self._ctx.call("amb_set_option", b"ap_filter", int(seconds))
        self._ctx.ap_filter = int(seconds)

    def get_ap_filter(self) -> int:
        return self._ctx.ap_filter

    # -- extension: Mode A/C replies (see the class docstring)
    def set_modeac(self, on: bool):
        """Find Mode A/C replies from the next stream on: only before the first process() after construction, reset()
        or set_rate()."""
        self._ctx.call("amb_set_option", b"modeac", int(bool(on)))
        self._modeac = bool(on)

    def get_modeac(self) -> bool:
        return self._modeac

    def modeac(self) -> np.ndarray:
        """Every reply not handed out yet, in stream order and stamped: a numpy array of MODEAC_DTYPE (waits for the
        work given so far)."""
        n = self._ctx.call("amb_pending_modeac")
        out = np.zeros(n, MODEAC_DTYPE)
        got = self._ctx.call("amb_poll_modeac", out.ctypes.data_as(C.c_void_p), n) if n else 0
        return out[:got]

    def modeac_device(self, out=None):
        """The device-side modeac(): a torch CUDA uint8 tensor of n * 48 bytes (amb_modeac records in stream order,
        stamped) that never crosses to the host. Replies modeac() already fetched are not included."""
        import torch
        n = self._ctx.call("amb_drain_modeac_device", None, 0)
        dev = torch.device("cuda", self._ctx.device)
        if out is None:
            out = torch.empty(n * 48, dtype=torch.uint8, device=dev)
        elif out.numel() < n * 48:
            raise ValueError("modeac_device: out holds %d bytes, %d needed" % (out.numel(), n * 48))
        torch.cuda.current_stream(dev).synchronize()
        got = self._ctx.call("amb_drain_modeac_device", C.c_void_p(out.data_ptr()), int(out.numel() // 48)) if n else 0
        return out[:got * 48]

    def modeac_stats(self) -> ModeacStats:
        """Counts since the stream began: candidates (rules 1-2), replies, overlap drops (rule 7), with altitude."""
        st = ModeacStats()
        self._ctx.call("amb_get_modeac_stats", C.byref(st))
        return st

    # -- data path
    def process(self, iq, flush: bool = False, collect: bool = True) -> int:
        """Consume a stretch of the stream; returns the number of messages queued (0 if collect=False:
        results then stay on the device until drain() / poll_ready()).

        Host arrays (numpy, CPU tensors; float32 / complex64 / int16 I,Q) are consumed before this returns. A torch
        CUDA tensor is read in place: the call is ordered after the work already enqueued on torch's current stream,
        and the tensor is kept alive until drain() (or a collecting process()) has synchronised."""
        ptr, n, kind, keep = _as_iq(iq)
        if kind in (_lib.MEM_DEVICE, _lib.MEM_DEVICE_SC16):
            try:
                import torch
                self._ctx.wait_stream(torch.cuda.current_stream(keep.device).cuda_stream)
            except ImportError:
                pass
            self._keep.append(keep)
        self._ctx.call("amb_process", ptr, n, kind, int(flush))
        return self.drain() if collect else 0

    def drain(self) -> int:
        """Wait for everything given so far and queue its messages."""
        buf, got = self._ctx.poll_array()
        self.frames = list(buf)[:got] if got else []
        self._keep.clear()
        return self._slicer.emit(buf, got)

    def drain_device(self, out=None):
        """The device-side drain(): waits for everything given so far and returns its frames as a torch CUDA uint8 tensor
        of n * 80 bytes (amb_frame records in stream order, stamped) WITHOUT copying them to the host - the input of
        batch_decoder.decode_device(). No messages are queued for these frames (that needs them on the host: drain())."""
        import torch
        n = self._ctx.call("amb_drain_device", None, 0)
        dev = torch.device("cuda", self._ctx.device)
        if out is None:
            out = torch.empty(n * 80, dtype=torch.uint8, device=dev)
        elif out.numel() < n * 80:
            raise ValueError("drain_device: out holds %d bytes, %d needed" % (out.numel(), n * 80))
        # the library writes `out` on its own stream: whatever torch's stream still does with that memory (a recycled
        # block, a producer of a caller-supplied tensor) comes first
        torch.cuda.current_stream(dev).synchronize()
        got = self._ctx.call("amb_drain_device", C.c_void_p(out.data_ptr()), int(out.numel() // 80)) if n else 0
        self.frames = []
        self._keep.clear()
        return out[:got * 80]

    def poll_ready(self, max_frames: int = 4096) -> int:
        """Non-blocking drain: queue the messages of the calls that have already completed on the device (what a GNU
        Radio work() function calls after handing over its items). Returns how many were queued."""
        buf, got = self._ctx.poll_ready_array(max_frames)
        if not got:
            self.frames = []
            return 0
        arr = (Frame * got).from_buffer_copy(buf)            # own copy: the poll buffer is reused
        self.frames = list(arr)
        return self._slicer.emit(arr, got)

    def add_time_tag(self, offset: int, secs: int, frac: float):
        """A later rx_time tag at absolute item `offset` (see amb_add_time_tag)."""
        self._ctx.call("amb_add_time_tag", int(offset), int(secs), float(frac))

    def use_stream(self, cuda_stream_ptr: int):
        """Run the streaming pass on a caller-owned cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream)."""
        self._ctx.use_stream(cuda_stream_ptr)

    def join(self):
        """Make the caller-visible stream wait for everything enqueued so far (no host synchronisation)."""
        self._ctx.join()

    def set_option(self, name: str, value: int):
        """Library options: "coalesce", "ingest_chunk", "copy_threads", "resolver", "overlap", "keep_chips", "exact_dense",
        "scan_ctas", "order_tile", "ec", "ec_any", "ap_filter", "modeac"."""
        if name == "ec":
            return self.set_ec(value)
        if name == "ec_any":
            return self.set_ec_any(value)
        if name == "ap_filter":
            return self.set_ap_filter(value)
        if name == "modeac":
            return self.set_modeac(value)
        self._ctx.call("amb_set_option", name.encode(), int(value))

    def reset(self):
        self._ctx.call("amb_reset")

    # -- one stream time-sharded over several rx_paths / GPUs (include/airmodes_b200.h, amb_seek)
    def seek(self, first_sample: int, first_decision: int, entry=None):
        """Restart the stream at global sample `first_sample`; decisions start at reported index
        `first_decision`. entry = (pos, p) handed over by the previous span, None = fresh."""
        st = WalkState(int(entry[0]), int(entry[1])) if entry is not None else None
        self._ctx.call("amb_seek", int(first_sample), int(first_decision), C.byref(st) if st is not None else None)

    def defer_resolve(self, on: bool = True):
        self._ctx.call("amb_set_option", b"defer_resolve", int(bool(on)))

    def resolve(self, entry=None):
        st = WalkState(int(entry[0]), int(entry[1])) if entry is not None else None
        self._ctx.call("amb_resolve", C.byref(st) if st is not None else None)

    def walk_state(self):
        st = WalkState()
        self._ctx.call("amb_get_walk_state", C.byref(st))
        return int(st.pos), int(st.p)

    def walk_summary(self) -> WalkSummary:
        s = WalkSummary()
        self._ctx.call("amb_get_walk_summary", C.byref(s))
        return s

    # -- the same hand-over with nothing waiting on the host (amb_walk_summary_async and friends): device pointers
    def walk_summary_async(self, dev_ptr: int):
        self._ctx.call("amb_walk_summary_async", C.c_void_p(dev_ptr))

    def compose_entries_async(self, gathered_ptr: int, n_spans: int, out_ptr: int, stream_ptr: int = 0):
        self._ctx.call("amb_compose_entries_async", C.c_void_p(gathered_ptr), int(n_spans), C.c_void_p(out_ptr), C.c_void_p(stream_ptr))

    def resolve_device(self, entry_ptr: int, after_stream_ptr: int = 0):
        self._ctx.call("amb_resolve_device", C.c_void_p(entry_ptr), C.c_void_p(after_stream_ptr))

    def join_stream(self, stream_ptr: int = 0):
        """Make another CUDA stream of the caller's wait for everything enqueued so far (0: the caller-visible one)."""
        self._ctx.call("amb_join_stream", C.c_void_p(stream_ptr))

    def dump_stage(self, stage: str, iq) -> np.ndarray:
        """Parity dump: "m2" | "bb" | "avg" | "dc" of a short host buffer taken as a whole stream (amb_dump_stage)."""
        iq = np.ascontiguousarray(np.asarray(iq).view(np.float32).reshape(-1))
        out = np.empty(iq.size if stage == "dc" else iq.size // 2, np.float32)
        self._ctx.call("amb_dump_stage", {"m2": 0, "bb": 1, "avg": 2, "dc": 3}[stage],
                       iq.ctypes.data_as(C.POINTER(C.c_float)), iq.size // 2, out.ctypes.data_as(C.POINTER(C.c_float)))
        return out

    def stats(self) -> Stats:
        return self._ctx.stats()

    def close(self):
        self._ctx.close()
