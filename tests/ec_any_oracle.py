"""TEST INFRASTRUCTURE ONLY: an independent restatement of the DF17 correction behind option "ec_any".

The library looks each candidate's syndrome up among the one- and two-bit syndromes (amb_ec_kernel, second phase). This
checker does not: it enumerates every pattern of at most M bits over positions 5..nbits-1, flips them in a copy of the
payload and recomputes the CRC with the bytewise arithmetic of modes_crc.cc (tests/ec_oracle.py). It composes after
ec_oracle.correct, as the library runs the "ec" pass first. The product never imports it (tests/test_host_logic.py).

Semantics (DESIGN.md section 0):
  candidate   df == 17, passed == 0 and crc != 0 after the "ec" pass (a frame "ec" fixed is not tried again;
              numlowconf does not matter)
  search set  bit positions 5..111 (the DF field is never flipped)
  fixed       exactly one pattern of at most M bits zeroes the syndrome: data flipped, crc = 0, passed = 1,
              bits = the flipped positions, ascending
  otherwise   no solution; the frame stays dropped
"""
from __future__ import annotations

import ctypes as C
import os
import sys
from itertools import combinations

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_oracle as eo  # noqa: E402

EC_NOT_TRIED, EC_FIXED, EC_NO_SOLUTION = eo.EC_NOT_TRIED, eo.EC_FIXED, eo.EC_NO_SOLUTION
LO = 5                      # first position that may be flipped


def patterns(nbits: int, m: int):
    """Every pattern of 1..m positions in LO..nbits-1, as sorted tuples (one bits first, then pairs, ...)."""
    return [p for r in range(1, m + 1) for p in combinations(range(LO, nbits), r)]


def flipped_rows(base: np.ndarray, pats) -> np.ndarray:
    """One copy of the uint8 payload `base` per pattern, with that pattern's bits flipped."""
    rows = np.repeat(base[None, :], len(pats), axis=0)
    for r in range(max((len(p) for p in pats), default=0)):
        sel = np.array([len(p) > r for p in pats])
        pos = np.array([p[r] if len(p) > r else 0 for p in pats])
        np.bitwise_xor.at(rows, (np.nonzero(sel)[0], pos[sel] // 8), (0x80 >> (pos[sel] % 8)).astype(np.uint8))
    return rows


def _is_candidate(frame, m: int) -> bool:
    return bool(m) and int(frame.df) == 17 and not frame.passed and frame.crc != 0


def _apply(frame, bits):
    """A copy of `frame` with `bits` flipped, crc = 0 and passed = 1."""
    g = type(frame).from_buffer_copy(frame)
    data = bytearray(bytes(g.data))
    for p in bits:
        data[p // 8] ^= 0x80 >> (p % 8)
    C.memmove(C.addressof(g) + type(g).data.offset, bytes(data), len(data))
    g.crc = 0
    g.passed = 1
    return g


def correct_any(frame, m: int):
    """(status, bits, corrected copy of `frame`) by brute force over every pattern of at most m bits. bits: the sorted
    positions flipped (empty unless fixed). The copy equals the frame unless the status is EC_FIXED."""
    if not _is_candidate(frame, m):
        return EC_NOT_TRIED, (), type(frame).from_buffer_copy(frame)
    nbits = int(frame.nbits)
    pats = patterns(nbits, m)
    base = np.frombuffer(bytes(frame.data), np.uint8)[: nbits // 8]
    hits = np.nonzero(eo.syndromes(flipped_rows(base, pats), nbits) == 0)[0]
    if hits.size != 1:
        return EC_NO_SOLUTION, (), type(frame).from_buffer_copy(frame)
    bits = tuple(pats[int(hits[0])])
    return EC_FIXED, bits, _apply(frame, bits)


class SyndromeTable:
    """syndrome -> every pattern of at most m bits with that syndrome, built by the same enumeration on an all-zero
    112-bit packet (the syndrome is linear: a packet's own syndrome is that of its error pattern). Equal to correct_any
    on every frame (tests/test_ec_any_cpu.py); fast enough for long scenes."""

    def __init__(self, m: int, nbits: int = 112):
        self.m, self.nbits = m, nbits
        pats = patterns(nbits, m)
        syn = eo.syndromes(flipped_rows(np.zeros(nbits // 8, np.uint8), pats), nbits)
        self.table = {}
        for p, s in zip(pats, syn.tolist()):
            self.table.setdefault(int(s), []).append(p)

    def correct(self, frame):
        if not _is_candidate(frame, self.m):
            return EC_NOT_TRIED, (), type(frame).from_buffer_copy(frame)
        assert int(frame.nbits) == self.nbits
        fits = self.table.get(int(frame.crc), [])
        if len(fits) != 1:
            return EC_NO_SOLUTION, (), type(frame).from_buffer_copy(frame)
        return EC_FIXED, tuple(fits[0]), _apply(frame, fits[0])


def correct_both(frame, k: int, m: int, table: SyndromeTable | None = None):
    """The two passes in the library's order: ((ec status, ec flips), (ec_any status, ec_any bits), final frame)."""
    st, flips, g = eo.correct(frame, k)
    if st == EC_FIXED:
        return (st, flips), (EC_NOT_TRIED, ()), g
    st2, bits, g2 = table.correct(g) if table is not None else correct_any(g, m)
    return (st, flips), (st2, bits), g2


def merged_messages(port, frames, k: int, m: int, first: bool = True, table: SyndromeTable | None = None):
    """The message stream with both passes: the oracle's messages plus those of the frames either pass fixed, in stream
    order, with the first-message precision rule of slicer_impl.cc:192 applied over the merged sequence (as
    ec_oracle.merged_messages). `frames`: the oracle's frames (all detections, stream order)."""
    out = []
    for f in frames:
        _, _, g = correct_both(f, k, m, table)
        if g.passed:
            out.append(port.format_message(g, first and not out))
    return out
