"""Sequential checker of the decoder option "coverage" (include/airmodes_b200.h, DESIGN.md §8 "Receiver coverage"):
rules 1-4 replayed in Python over the decoder's own records, one record at a time in stream order, into a 72 x 9 grid of
floats. add() is az_map_model.addRecord (python/az_map.py:56-75) restated with npoints = 72; tests/golden's
coverage_golden.json.gz pins it against the unmodified az_map.py."""
from __future__ import annotations

import numpy as np

ROWS, BANDS = 72, 9
ALTITUDES = (0, 1000, 2000, 5000, 10000, 15000, 20000, 25000, 30000)
FS_NO_HANDLER, FS_HAS_RANGE, FS_NOT_QUEUED = 0x01, 0x20, 0x80


def cell(bearing: float, altitude: int):
    """Rule 3: (row, col). The sum bearing + 2.5 is a Python float (IEEE double), truncated, then divided as an
    integer (az_map.py:66: int(int(b + 180./72) / (360./72)) % 72, which is the same for b + 2.5 >= 0)."""
    row = int(bearing + 2.5) // 5 % ROWS
    col = BANDS - 1 if altitude >= ALTITUDES[-1] else next(j for j, a in enumerate(ALTITUDES) if a >= altitude)
    return row, col


def add(grid, bearing: float, altitude: int, rng: float) -> None:
    """Rule 4: every band from col up takes the range when it is strictly greater."""
    row, col = cell(bearing, altitude)
    for j in range(col, BANDS):
        if rng > grid[row][j]:
            grid[row][j] = rng


def counted(rec):
    """Rules 1-2: (bearing, altitude, range) of a record that counts, else None. `rec`: a FIELDS_DTYPE record or an
    oracle/decode_oracle.py record dict."""
    st = int(rec["status"])
    if st & (FS_NOT_QUEUED | FS_NO_HANDLER) or int(rec["df"]) != 17 or int(rec["bds"]) not in (0x05, 0x06):
        return None
    if not st & FS_HAS_RANGE:
        return None
    alt = 0 if int(rec["bds"]) == 0x06 else int(rec["altitude"])
    return float(rec["bearing"]), alt, float(rec["range"])


def empty():
    return [[0.0] * BANDS for _ in range(ROWS)]


class CoverageChecker:
    """The grid of one decoder: feed() the records of every call in stream order; reset() = amb_decoder_reset or
    amb_decoder_coverage_reset."""

    def __init__(self):
        self.grid = empty()

    def reset(self):
        self.grid = empty()

    def feed(self, recs) -> np.ndarray:
        for r in recs:
            c = counted(r)
            if c is not None:
                add(self.grid, *c)
        return self.array()

    def array(self) -> np.ndarray:
        return np.array(self.grid, dtype=np.float64)


def grid_of(recs) -> np.ndarray:
    return CoverageChecker().feed(recs)
