"""Sequential checker of the decoder option "commb" (Comm-B register inference, DESIGN.md §8 "Comm-B inference"),
written from the rules in include/airmodes_b200.h and not from the kernel: it takes the decoder's own option-off
records and their frames and returns the records the option must produce. Each record's velocity reference is found by
a scan of the earlier records. Also an encoder of the three registers, independent of the decoder, for the scenes and
the round trips."""
from __future__ import annotations

import math

import numpy as np

NOT_TRIED, DECODED, RESOLVED, AMBIGUOUS, NONE = 0, 1, 2, 3, 4
FS_NO_HANDLER, FS_NOT_QUEUED = 0x01, 0x80
REGS = (0x40, 0x50, 0x60)

# Per register, fields 0..4: (status bit, sign bit or None, first magnitude bit, magnitude bits). MB bits 1..56.
LAYOUT = {
    0x40: ((1, None, 2, 12), (14, None, 15, 12), (27, None, 28, 12), (48, None, 49, 3), (54, None, 55, 2)),
    0x50: ((1, 2, 3, 9), (12, 13, 14, 10), (24, None, 25, 10), (35, 36, 37, 9), (46, None, 47, 10)),
    0x60: ((1, 2, 3, 10), (13, None, 14, 10), (24, None, 25, 10), (35, 36, 37, 9), (46, 47, 48, 9)),
}
RESERVED = {0x40: tuple(range(40, 48)) + (52, 53), 0x50: (), 0x60: ()}


def bit(mb, k):
    return (mb >> (56 - k)) & 1


def bits(mb, first, n):
    return (mb >> (57 - first - n)) & ((1 << n) - 1)


def put(mb, first, n, v):
    return mb | ((v & ((1 << n) - 1)) << (57 - first - n))


def raw_range(reg, i):
    """The raw values field i can carry: (lowest, highest)."""
    _, sign, _, n = LAYOUT[reg][i]
    return (-(1 << n), (1 << n) - 1) if sign else (0, (1 << n) - 1)


def encode(reg, values, reserved=0):
    """MB word of register `reg` with fields {i: raw value} present (others absent, all-zero); `reserved` is OR-ed into
    the 4,0 reserved bits as a mask over their positions."""
    mb = 0
    for i, v in values.items():
        st, sign, first, n = LAYOUT[reg][i]
        mb = put(mb, st, 1, 1)
        if sign is not None:
            mb = put(mb, sign, 1, 1 if v < 0 else 0)
            v = v + (1 << n) if v < 0 else v
        mb = put(mb, first, n, v)
    for j, k in enumerate(RESERVED[reg]):
        if (reserved >> j) & 1:
            mb = put(mb, k, 1, 1)
    return mb


def read(mb, reg):
    """(is a candidate, raw values of fields 0..4 with 0 for absent ones, status mask)."""
    raws, mask, ok = [0] * 5, 0, True
    for i, (st, sign, first, n) in enumerate(LAYOUT[reg]):
        mag = bits(mb, first, n)
        s = bit(mb, sign) if sign is not None else 0
        if bit(mb, st):
            mask |= 1 << i
            raws[i] = mag - (1 << n) if s else mag
        elif mag or s:
            ok = False
    if mask == 0 or any(bit(mb, k) for k in RESERVED[reg]):
        ok = False
    r = raws
    if reg == 0x40:
        if r[0] > 3125 or r[1] > 3125 or (mask & 4 and not 700 <= r[2] <= 3000):
            ok = False
    elif reg == 0x50:
        if abs(r[0]) > 284 or r[2] > 400 or r[4] > 300 or (mask & 4 and mask & 16 and abs(r[2] - r[4]) > 125):
            ok = False
    else:
        if r[1] > 500 or r[2] > 250 or abs(r[3]) > 187 or abs(r[4]) > 187:
            ok = False
    return ok, raws, mask


def candidates(mb):
    return [reg for reg in REGS if read(mb, reg)[0]]


def agree(gs_raw, trk_raw, speed, track):
    trk = trk_raw * 90.0 / 512.0
    d = math.fmod(abs(trk - track), 360.0)
    d = min(d, 360.0 - d)
    return abs(2.0 * gs_raw - speed) <= 20.0 and d <= 10.0


def t_of(frames):
    return frames["secs"].astype(np.float64) + frames["frac"]


def mb_of(frame):
    return int.from_bytes(bytes(frame["data"][4:11]), "big")


def eligible(frame, rec):
    if not frame["passed"] or frame["nbits"] != 112 or rec["status"] != FS_NO_HANDLER or rec["df"] not in (20, 21):
        return False
    b1 = mb_of(frame) >> 48
    return not (b1 & 0x0F == 0 and b1 >> 4 <= 3)


def is_reference(rec):
    return (not rec["status"] & FS_NOT_QUEUED and rec["df"] == 17 and rec["bds"] == 0x09 and rec["subtype"] in (0, 1)
            and not math.isnan(rec["val"][0]) and not math.isnan(rec["val"][1]))


def decide(mb, ref, t, S):
    """(outcome, register or None, candidate list) of one eligible word; ref = (t, speed, track) or None."""
    c = candidates(mb)
    if not c:
        return NONE, None, c
    if len(c) == 1:
        return DECODED, c[0], c
    _, r50, m50 = read(mb, 0x50)
    if 0x50 in c and m50 & 6 == 6 and ref is not None and 0.0 <= t - ref[0] <= S:
        left = [0x50] if agree(r50[2], r50[1], ref[1], ref[2]) else [g for g in c if g != 0x50]
        if len(left) == 1:
            return RESOLVED, left[0], c
    return AMBIGUOUS, None, c


class Checker:
    """Feed (frames, option-off records) call by call in stream order; get the option-on records back."""

    def __init__(self, S):
        self.S = S
        # every earlier record: its address when it is a velocity reference (else -1), t, speed, track
        self.icao = np.zeros(0, dtype=np.int64)
        self.t = self.speed = self.track = np.zeros(0)

    def reset(self):
        self.__init__(self.S)

    def feed(self, frames, recs):
        n0 = len(self.icao)
        ts = t_of(frames)
        refs = np.array([int(r["icao"]) if is_reference(r) else -1 for r in recs], dtype=np.int64)
        self.icao = np.concatenate([self.icao, refs])
        self.t = np.concatenate([self.t, ts])
        self.speed = np.concatenate([self.speed, recs["val"][:, 0]])
        self.track = np.concatenate([self.track, recs["val"][:, 1]])
        out = recs.copy()
        for k in range(len(recs)):
            f, r = frames[k], recs[k]
            if not eligible(f, r):
                continue
            mb = mb_of(f)
            hits = np.flatnonzero(self.icao[:n0 + k] == int(r["icao"]))   # a scan of every earlier record
            ref = None if len(hits) == 0 else (float(self.t[hits[-1]]), float(self.speed[hits[-1]]),
                                                 float(self.track[hits[-1]]))   # the latest earlier velocity record
            outcome, reg, cand = decide(mb, ref, float(ts[k]), self.S)
            set_record(out[k:k + 1], mb, outcome, reg, cand)
        return out


def set_record(rec1, mb, outcome, reg, cand):
    """Write the option's fields into a 1-element FIELDS_DTYPE slice."""
    raws, mask = [0] * 5, 0
    if reg is not None:
        _, raws, mask = read(mb, reg)
    aux = np.array(raws + [0, 0, 0], dtype="<i2").view("<u4")
    rec1["aux"][0] = aux
    cbits = sum(1 << REGS.index(g) for g in cand)
    pad = int(rec1["pad_"][0]) & ~0xFFFFFFFF00
    pad |= (outcome << 8) | ((reg or 0) << 16) | (mask << 24) | (cbits << 32)
    rec1["pad_"][0] = pad


def replay(frames, recs, S):
    return Checker(S).feed(frames, recs)


def outcome_of(recs):
    return (np.asarray(recs["pad_"], dtype=np.uint64) >> np.uint64(8)) & np.uint64(0xFF)


def assert_records_equal(got, want, tag):
    if got.tobytes() == want.tobytes():
        return
    bad = [k for k in range(len(got)) if got[k].tobytes() != want[k].tobytes()]
    k = bad[0]
    raise AssertionError("%s: %d records differ, first #%d: got pad_ %#x aux %s, want pad_ %#x aux %s"
                         % (tag, len(bad), k, int(got["pad_"][k]), list(got["aux"][k]), int(want["pad_"][k]),
                            list(want["aux"][k])))
