"""Independent checker of Beast binary input (include/airmodes_b200.h "Beast binary input"; DESIGN.md §8 "Beast input"):
a byte-by-byte sequential parser written from rules 1-5 with plain Python integers and floats. It knows nothing of the
device's scans: it reads the stream left to right, one byte at a time, as a reader on a socket would. It gives the
frames (a numpy FRAME_DTYPE array), the counters of amb_beast_counts and the bytes a call carries."""
import numpy as np

ESC = 0x1A
CLOCK = 12_000_000
NEED = {0x31: 9, 0x32: 14, 0x33: 21}          # '1' Mode A/C, '2' Mode S short, '3' Mode S long: data tokens of a body
LONG_DF = (16, 17, 20, 21)
COUNTERS = ("modes", "modeac", "other", "truncated", "skipped", "passed")


def frame_dtype():
    from gr_air_modes_b200._lib import Frame      # the record layout only
    return np.dtype(Frame)


def _crc_table():
    t = []
    for n in range(256):
        c = n << 16
        for _ in range(8):
            c = (((c << 1) ^ 0xFFF409) if c & 0x800000 else c << 1) & 0xFFFFFF
        t.append(c)
    return t


_CRC = _crc_table()


def crc24(data) -> int:
    """modes_check_crc (modes_crc.cc:33-63): polynomial 0xFFF409, most significant bit first, a byte at a time."""
    c = 0
    for b in data:
        c = _CRC[((c >> 16) ^ b) & 0xFF] ^ ((c << 8) & 0xFFFFFF)
    return c


def stamp(T: int):
    """(secs, frac) of a 48-bit count T at 12 MHz (rule 3): one correctly rounded division."""
    return T // CLOCK, (T % CLOCK) / 12e6


def level(S: int) -> float:
    """ref_level of a signal byte S (rule 3), as a float32 value."""
    return float(np.float32((S * S) / 65025.0))


def passed(data: bytes, nbits: int, crc: int) -> int:
    """Rule 4: the reference slicer's drop rules that need no samples."""
    df = data[0] >> 3
    if not any(data):
        return 0
    if nbits != (112 if df in LONG_DF else 56):
        return 0
    if crc and df in (11, 17):
        return 0
    return 1


def frame_fields(body, at):
    """The fields of the frame of a complete Mode S message: body = the data tokens after its sync token."""
    T = int.from_bytes(bytes(body[:6]), "big")
    S = body[6]
    payload = bytes(body[7:])
    nb = len(payload)
    crc = crc24(payload[: nb - 3]) ^ int.from_bytes(payload[nb - 3:], "big")
    secs, frac = stamp(T)
    return {"sample_index": at, "secs": secs, "frac": frac, "ref_level": level(S), "crc": crc, "nbits": 8 * nb,
            "df": payload[0] >> 3, "passed": passed(payload, 8 * nb, crc), "data": payload + bytes(14 - nb)}


class Parser:
    """The stream since create or reset. feed(buf, flush) reads the next bytes and returns this call's frames (a list of
    field dicts); carry() is what a call cut here would have to keep."""

    def __init__(self):
        self.counts = dict.fromkeys(COUNTERS, 0)
        self.pos = 0                    # stream offset of the next byte
        self.esc_at = None              # a 0x1a token start whose second byte is still to come
        self.body = None                # (need, sync offset, type, data tokens so far) of the open message
        self.flushed = False

    def _data(self, v, out):
        if self.body is None:
            self.counts["skipped"] += 1
            return
        need, at, ty, toks = self.body
        toks.append(v)
        if len(toks) == need:
            self.body = None
            if ty == 0x31:
                self.counts["modeac"] += 1
            else:
                self.counts["modes"] += 1
                f = frame_fields(toks, at)
                self.counts["passed"] += f["passed"]
                out.append(f)

    def _sync(self, ty, at):
        if self.body is not None:
            self.counts["truncated"] += 1
            self.body = None
        if ty in NEED:
            self.body = (NEED[ty], at, ty, [])
        else:
            self.counts["other"] += 1

    def feed(self, buf, flush=False):
        if self.flushed:
            raise RuntimeError("flushed")
        out = []
        for b in bytes(buf):
            if self.esc_at is not None:
                at, self.esc_at = self.esc_at, None
                if b == ESC:
                    self._data(ESC, out)
                else:
                    self._sync(b, at)
            elif b == ESC:
                self.esc_at = self.pos
            else:
                self._data(b, out)
            self.pos += 1
        if flush:
            self.esc_at = None                       # a lone final 0x1a: dropped, not counted
            if self.body is not None:
                self.counts["truncated"] += 1
                self.body = None
            self.flushed = True
        return out

    def carry(self) -> int:
        """Bytes a call ending here carries: from the open message's sync byte, else a lone final 0x1a, else none."""
        if self.body is not None:
            return self.pos - self.body[1]
        return 1 if self.esc_at is not None else 0


def to_array(frames) -> np.ndarray:
    arr = np.zeros(len(frames), frame_dtype())
    for k, f in enumerate(frames):
        for name in ("sample_index", "secs", "frac", "ref_level", "crc", "nbits", "df", "passed"):
            arr[name][k] = f[name]
        arr["data"][k] = np.frombuffer(f["data"], np.uint8)
    return arr


def parse(buf, flush=True):
    """One call over the whole stream: (frames as a FRAME_DTYPE array, counters, bytes carried)."""
    p = Parser()
    fr = p.feed(buf, flush)
    return to_array(fr), dict(p.counts), p.carry()


# ---- streams that test the rules -----------------------------------------------------------------------------------
def escape(raw: bytes) -> bytes:
    return raw.replace(b"\x1a", b"\x1a\x1a")


def message(ty: int, T: int, S: int, payload: bytes) -> bytes:
    """A well-formed Beast message of type ty ('1', '2' or '3') with the given T, S and payload."""
    return bytes([ESC, ty]) + escape(T.to_bytes(6, "big") + bytes([S]) + payload)


def garbage(rng, n, density=0.4) -> bytes:
    """n random bytes, a share `density` of them 0x1a and a few type bytes among the rest."""
    v = rng.integers(0, 256, n).astype(np.uint8)
    r = rng.random(n)
    typ = r < 0.1
    v[typ] = rng.choice(np.array([0x31, 0x32, 0x33, 0x34], np.uint8), int(typ.sum()))
    v[r > 1.0 - density] = ESC
    return v.tobytes()
