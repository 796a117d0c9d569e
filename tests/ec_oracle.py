"""TEST INFRASTRUCTURE ONLY: an independent restatement of the error correction behind option "ec".

The library solves each candidate with a GF(2) elimination over per-bit syndromes (amb_ec_kernel). This checker does
neither: it enumerates every subset of the search set, flips those bits in a copy of the payload and recomputes the
CRC with the plain bytewise table arithmetic of modes_crc.cc:55-63, then applies the drop rule of slicer_impl.cc:173-182.
The product never imports it (tests/test_host_logic.py).

Semantics (DESIGN.md section 0):
  candidate   passed == 0 and crc != 0 (only DF11 / DF17 frames can be: every other rule leaves crc == 0)
  L           lowconfbits[:numlowconf] minus positions 0-4 (the DF field is never flipped)
  too many    numlowconf > K (a saturated count of 24 always)
  otherwise   the non-empty subsets S of L whose flips zero the syndrome: none / several / exactly one (fixed:
              data flipped, crc = 0, passed = 1; numlowconf and lowconfbits keep what the slicer saw)
"""
from __future__ import annotations

import ctypes as C

import numpy as np

EC_NOT_TRIED, EC_FIXED, EC_TOO_MANY, EC_NO_SOLUTION, EC_AMBIGUOUS = 0, 1, 2, 3, 4


def _crc_table():
    """crc_table of modes_crc.cc:31-53 (polynomial 0xFFF409, MSB first)."""
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i << 16
        for _ in range(8):
            c = ((c << 1) ^ 0xFFF409) if c & 0x800000 else (c << 1)
        t[i] = c & 0xFFFFFF
    return t


TABLE = _crc_table()


def crc_rows(data: np.ndarray, length: int) -> np.ndarray:
    """modes_check_crc(row, length) for every row of a uint8 array: crc = table[((crc >> 16) ^ byte) & 0xff] ^ (crc << 8)."""
    crc = np.zeros(data.shape[0], np.uint32)
    for i in range(length):
        crc = TABLE[((crc >> 16) ^ data[:, i].astype(np.uint32)) & 0xFF] ^ ((crc << 8) & 0xFFFFFFFF)
    return crc & 0xFFFFFF


def syndromes(data: np.ndarray, nbits: int) -> np.ndarray:
    """slicer_impl.cc:173-177 per row: CRC of the first nbits/8 - 3 bytes XOR the last three bytes."""
    nb = nbits // 8
    ap = (data[:, nb - 3].astype(np.uint32) << 16) | (data[:, nb - 2].astype(np.uint32) << 8) | data[:, nb - 1]
    return crc_rows(data, nb - 3) ^ ap


def search_set(frame):
    return [int(p) for p in list(frame.lowconfbits)[:int(frame.numlowconf)] if int(p) >= 5]


def correct(frame, k: int):
    """(status, flips, corrected copy of `frame`) for a cpu_oracle.Frame or an amb_frame, by brute force. flips: the
    sorted bit positions flipped (empty unless fixed). The copy equals the frame unless the status is EC_FIXED."""
    g = type(frame).from_buffer_copy(frame)
    if not k or frame.passed or frame.crc == 0:
        return EC_NOT_TRIED, (), g
    if int(frame.numlowconf) > k:
        return EC_TOO_MANY, (), g
    nbits = int(frame.nbits)
    L = search_set(frame)
    base = np.frombuffer(bytes(frame.data), np.uint8)[: nbits // 8]
    masks = np.arange(1, 1 << len(L), dtype=np.int64)
    rows = np.repeat(base[None, :], masks.size, axis=0)
    for i, p in enumerate(L):
        sel = ((masks >> i) & 1).astype(bool)
        rows[sel, p // 8] ^= np.uint8(0x80 >> (p % 8))
    hits = np.nonzero(syndromes(rows, nbits) == 0)[0] if masks.size else np.zeros(0, np.int64)
    if hits.size == 0:
        return EC_NO_SOLUTION, (), g
    if hits.size > 1:
        return EC_AMBIGUOUS, (), g
    flips = tuple(sorted(p for i, p in enumerate(L) if (masks[hits[0]] >> i) & 1))
    data = bytearray(bytes(g.data))
    data[: nbits // 8] = rows[hits[0]].tobytes()
    C.memmove(C.addressof(g) + type(g).data.offset, bytes(data), len(data))
    g.crc = 0
    g.passed = 1
    return EC_FIXED, flips, g


def expected_frames(frames, k: int):
    """[(status, flips, corrected frame)] for every frame."""
    return [correct(f, k) for f in frames]


def merged_messages(port, frames, k: int, first: bool = True):
    """The message stream with correction: the oracle's messages plus those of the fixed frames, in stream order, with
    the first-message precision rule of slicer_impl.cc:192 applied over the merged sequence. `frames`: the oracle's
    frames (all detections, stream order)."""
    out = []
    for f in frames:
        st, _, g = correct(f, k)
        if f.passed or st == EC_FIXED:
            out.append(port.format_message(g, first and not out))
    return out
