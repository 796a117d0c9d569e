"""TEST INFRASTRUCTURE ONLY: an independent restatement of the address/parity check behind option "ap_filter".

The library buckets confirmers and subjects by address, sorts each bucket and keeps a table of the latest confirmer per
address across calls (amb_kernels.cu, amb_ap_*). This checker does none of that: for every subject it scans every
earlier confirmer of the stream (O(subjects x confirmers), no table, no buckets). It takes the oracle's frames (all
detections, stream order) and composes after the correction checkers (tests/ec_oracle.py, tests/ec_any_oracle.py), as
the library runs the correction passes first. The product never imports it.

Semantics (include/airmodes_b200.h, AMB_FRAME_AP):
  confirmer      df in {11, 17}, passed, crc == 0, fixed by neither correction pass; address AA (data[1..3])
  AP subject     passed, df not in {11, 17}; address crc (AP xor parity)
  II/SI subject  df == 11, not passed, 0 < crc < 0x80; address AA
  known          a confirmer g of the same address with g.si < f.si <= g.si + S * rate_int
  effect         known AP: unchanged; unknown AP: passed = 0; known II/SI: passed = 1; unknown II/SI: stays dropped
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_any_oracle as ea  # noqa: E402
import ec_oracle as eo  # noqa: E402

AP_NOT_CHECKED, AP_KNOWN, AP_UNKNOWN = 0, 1, 2
NONE, CONF, SUBJECT, IISI = 0, 1, 2, 3


def aa(frame) -> int:
    return (frame.data[1] << 16) | (frame.data[2] << 8) | frame.data[3]


def classify(frame, ec_status: int = eo.EC_NOT_TRIED, any_status: int = ea.EC_NOT_TRIED):
    """(kind, address) of a frame after the correction passes, whose outcomes are ec_status / any_status."""
    df, crc = int(frame.df), int(frame.crc)
    if frame.passed:
        if df not in (11, 17):
            return SUBJECT, crc & 0xFFFFFF
        if crc == 0 and ec_status != eo.EC_FIXED and any_status != ea.EC_FIXED:
            return CONF, aa(frame)
        return NONE, None
    if df == 11 and 0 < crc < 0x80:
        return IISI, aa(frame)
    return NONE, None


def check(items, seconds: int, rate_int: int):
    """items: [(sample_index, kind, address)] of one stream (any order). Returns the AP_* outcome of each item by brute
    force over every confirmer."""
    conf = [(si, a) for si, k, a in items if k == CONF]
    csi = np.array([c[0] for c in conf], np.uint64)
    cad = np.array([c[1] for c in conf], np.int64)
    w = np.uint64(seconds * rate_int)
    out = []
    for si, k, a in items:
        if k in (NONE, CONF) or not seconds:
            out.append(AP_NOT_CHECKED)
            continue
        s = np.uint64(si)
        hit = (cad == a) & (csi < s) & (s - csi <= w) if len(conf) else np.zeros(0, bool)
        out.append(AP_KNOWN if hit.any() else AP_UNKNOWN)
    return out


def apply(frames, k: int, m: int, seconds: int, rate_int: int, table: ea.SyndromeTable | None = None):
    """Every frame (the oracle's, cpu_oracle.Frame: .index is the sample index) through both correction checkers and
    this one: [(ec (status, flips), ec_any (status, bits), ap status, final frame)]."""
    corr = [ea.correct_both(f, k, m, table) for f in frames]
    items = []
    for f, (ec_st, any_st, g) in zip(frames, corr):
        kind, addr = classify(g, ec_st[0], any_st[0])
        items.append((int(f.index), kind, addr))
    aps = check(items, seconds, rate_int)
    out = []
    for (ec_st, any_st, g), (_, kind, _), ap in zip(corr, items, aps):
        if kind == SUBJECT and ap == AP_UNKNOWN:
            g.passed = 0
        if kind == IISI and ap == AP_KNOWN:
            g.passed = 1
        out.append((ec_st, any_st, ap, g))
    return out


def merged_messages(port, frames, k: int, m: int, seconds: int, rate_int: int, first: bool = True,
                    table: ea.SyndromeTable | None = None):
    """The message stream with the corrections and the check: the frames that end up passed, in stream order, with the
    first-message precision rule of slicer_impl.cc:192 applied over the resulting sequence."""
    out = []
    for _, _, _, g in apply(frames, k, m, seconds, rate_int, table):
        if g.passed:
            out.append(port.format_message(g, first and not out))
    return out
