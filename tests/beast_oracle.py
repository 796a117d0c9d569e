"""Independent checker of the Beast binary and AVR raw feeds (include/airmodes_b200.h, "Beast binary and AVR raw
feeds"; DESIGN.md §8): an encoder of both formats over a numpy FRAME_DTYPE array, written from the rules with Python
integers and floats, and byte-by-byte parsers of both formats for round trips."""
import math

import numpy as np

FS_NOT_QUEUED = 0x80
ESC = 0x1A
CLOCK = 12_000_000               # Beast timestamp ticks per second
TYPE_LEN = {0x32: 7, 0x33: 14}   # '2': Mode S short, '3': Mode S long


def timestamp(secs, frac) -> int:
    """T (rule 2): the stamp as a 48-bit count at 12 MHz; 0 when frac * 12e6 is not finite or at least 2^62."""
    x = float(frac) * 12e6
    if not math.isfinite(x) or abs(x) >= 2.0 ** 62:
        return 0
    return (int(secs) * CLOCK + round(x)) % (1 << 48)       # round(): half to even, exact for |x| < 2^62


def signal(ref_level) -> int:
    """S (rule 3) of a float32 reference level."""
    v = float(np.float32(ref_level))
    if math.isnan(v) or v <= 0.0:
        return 0
    if v >= 1.0:
        return 255
    return max(1, round(255.0 * math.sqrt(v)))


def payload(frame) -> bytes:
    return bytes(frame["data"][: 14 if int(frame["nbits"]) == 112 else 7])


def beast_message(frame) -> bytes:
    body = payload(frame)
    raw = timestamp(frame["secs"], frame["frac"]).to_bytes(6, "big") + bytes([signal(frame["ref_level"])]) + body
    return bytes([ESC, 0x33 if len(body) == 14 else 0x32]) + raw.replace(b"\x1a", b"\x1a\x1a")


def avr_line(frame, form) -> bytes:
    stamp = "%012X" % timestamp(frame["secs"], frame["frac"]) if form == 2 else ""
    return ("%s%s%s;\n" % ("@" if form == 2 else "*", stamp, payload(frame).hex().upper())).encode("ascii")


def queued(frames, records=None):
    """Which frames are written (rule 1): records lacking FS_NOT_QUEUED, or frames with passed != 0."""
    if records is None:
        return np.asarray(frames["passed"]) != 0
    return (np.asarray(records["status"]) & FS_NOT_QUEUED) == 0


def beast(frames, records=None) -> bytes:
    """The Beast messages of the queued frames, in order."""
    q = queued(frames, records)
    return b"".join(beast_message(f) for f, on in zip(frames, q) if on)


def avr(frames, form, records=None) -> bytes:
    """The AVR lines (form 1: "*", 2: "@" with the timestamp) of the queued frames, in order."""
    q = queued(frames, records)
    return b"".join(avr_line(f, form) for f, on in zip(frames, q) if on)


def parse_beast(buf: bytes):
    """Messages of a Beast stream, byte by byte: a list of (T, S, payload). Raises ValueError on anything but whole
    Mode S short / long messages with every 0x1a after the type byte doubled."""
    out, i, n = [], 0, len(buf)
    while i < n:
        if buf[i] != ESC or i + 1 >= n or buf[i + 1] not in TYPE_LEN:
            raise ValueError("no message start at byte %d" % i)
        want, body, i = 7 + TYPE_LEN[buf[i + 1]], bytearray(), i + 2
        while len(body) < want:
            if i >= n:
                raise ValueError("truncated message")
            b = buf[i]
            if b == ESC:
                if i + 1 >= n or buf[i + 1] != ESC:
                    raise ValueError("lone 0x1a at byte %d" % i)
                i += 1
            body.append(b)
            i += 1
        out.append((int.from_bytes(body[:6], "big"), body[6], bytes(body[7:])))
    return out


def parse_avr(text: bytes):
    """Lines of an AVR stream: a list of (T or None for a "*" line, payload). Raises ValueError on a malformed line."""
    out = []
    if text and not text.endswith(b"\n"):
        raise ValueError("truncated line")
    for line in text.split(b"\n")[:-1] if text else []:
        s = line.decode("ascii")
        if len(s) < 2 or s[-1] != ";" or s[0] not in "*@":
            raise ValueError("bad line %r" % s)
        body = s[1:-1]
        t = None
        if s[0] == "@":
            t, body = int(body[:12], 16), body[12:]
        if len(body) not in (14, 28) or body != body.upper():
            raise ValueError("bad payload %r" % s)
        out.append((t, bytes.fromhex(body)))
    return out


# ---- adversarial frames -------------------------------------------------------------------------------------------
PAYLOADS = ("8D4840D6202CC371C32CE0576098", "8D1A1A1A201A1A1A1A1A1A1A1A1A", "5D4840D6AAAAAA", "5D1A1A1A1A1A1A",
            "A8001A1A30000000000000123456")
WRAP_SECS = (1 << 48) // CLOCK               # secs * 12e6 is just below 2^48
T_1A = 0x1A1A1A1A1A1A
STAMPS = [(1, 0.5), (T_1A // CLOCK, (T_1A % CLOCK) / 12e6), (0, 0.0), (WRAP_SECS, 0.0), (WRAP_SECS, 0.05),
          (WRAP_SECS, 0.9999999), (WRAP_SECS + 1, 0.25), (2 ** 64 - 1, 0.999), (2 ** 64 - 2, 0.5), (2 ** 63, 0.125),
          (7, 2.0 ** -9), (7, 3 * 2.0 ** -9), (7, 5 * 2.0 ** -9), (0, -0.25), (5, -1e-9), (3, 1.75),
          (1, float("nan")), (1, float("inf")), (1, float("-inf")), (1, 1e300),
          (1, float(np.nextafter(2.0 ** 62 / 12e6, 0))), (1, 2.0 ** 62 / 12e6), (1, -2.0 ** 62 / 12e6)]
LEVELS = [0.25, float(np.float32((26 / 255) ** 2)), float("nan"), -1.0, 0.0, 1e-45, 1e-10, 0.999, 1.0, 2.0,
          float("inf"), -float("inf"), float(np.float32((0.5 / 255) ** 2))]


def adversarial_frames():
    """Frames at every edge of the rules: payloads with 0x1a bytes (long and short), timestamps of 0x1a bytes, at the
    2^48 wrap, secs near 2^64, half-tick ties, negative and non-finite fracs, |frac * 12e6| on both sides of 2^62, and
    signal levels NaN, negative, 0, tiny, (26/255)^2 (S = 0x1a), 1 and above; every fifth frame not queued, every
    seventh marked as fixed by error correction."""
    from gr_air_modes_b200 import decode
    rows = [(p, s, lv) for s in STAMPS for p in PAYLOADS[:2] for lv in LEVELS[:2]]
    rows += [(PAYLOADS[k % len(PAYLOADS)], STAMPS[k % len(STAMPS)], lv) for k, lv in enumerate(LEVELS * 3)]
    rows += [(p, STAMPS[1], LEVELS[1]) for p in PAYLOADS]
    fr = np.zeros(len(rows), dtype=decode.FRAME_DTYPE)
    for k, (p, (secs, frac), lv) in enumerate(rows):
        raw = bytes.fromhex(p)
        fr["data"][k][: len(raw)] = np.frombuffer(raw, np.uint8)
        fr["nbits"][k], fr["df"][k] = 8 * len(raw), raw[0] >> 3
        fr["secs"][k], fr["frac"][k], fr["ref_level"][k] = secs, frac, np.float32(lv)
        fr["passed"][k] = 0 if k % 5 == 4 else 1
        fr["pad_"][k][0] = 1 if k % 7 == 3 else 0      # amb_frame.ec = AMB_EC_FIXED
        fr["sample_index"][k] = 1000 * k
    return fr
