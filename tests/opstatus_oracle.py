"""Sequential checker of the decoder option "opstatus" (ADS-B operational status, target state and position integrity,
DESIGN.md §8 "Operational status and NIC"), written from the rules in include/airmodes_b200.h and not from the kernel:
it takes the decoder's own option-off records and their frames and returns the records the option must produce. A
position's op status A and surface op status C are found by a scan of every earlier op-status record; the NIC tables
are this file's own literal copy of DESIGN.md's."""
from __future__ import annotations

import numpy as np

NOT_TRIED, OPSTATUS, TARGET_STATE, NIC, NUC, UNSUPPORTED = 0, 1, 2, 3, 4, 5
NO_VERSION = 0xFF
FS_NO_HANDLER, FS_NOT_QUEUED = 0x01, 0x80

# type code -> {(NIC-A, NIC-B) or (NIC-A, NIC-C): (NIC, Rc in m or None)}; None as key: any supplements
AIRBORNE = {
    9: {None: (11, 7.5)}, 10: {None: (10, 25.0)},
    11: {(1, 1): (9, 75.0), (0, 0): (8, 185.2)},
    12: {None: (7, 370.4)},
    13: {(0, 1): (6, 555.6), (0, 0): (6, 926.0), (1, 1): (6, 1111.2)},
    14: {None: (5, 1852.0)},
    16: {(1, 1): (3, 7408.0), (0, 0): (2, 14816.0)},
    17: {None: (1, 37040.0)}, 18: {None: (0, None)},
}
SURFACE = {
    5: {None: (11, 7.5)}, 6: {None: (10, 25.0)},
    7: {(1, 0): (9, 75.0), (0, 0): (8, 185.2)},
    8: {(1, 1): (7, 370.4), (1, 0): (6, 555.6), (0, 1): (6, 1111.2), (0, 0): (0, None)},
}
NUCP = {9: 9, 10: 8, 11: 7, 12: 6, 13: 5, 14: 4, 16: 2, 17: 1, 18: 0, 5: 9, 6: 8, 7: 7, 8: 6}


def lookup(tc, s1, s2):
    """(NIC, Rc or None) of the tables; an unlisted combination is (0, None)."""
    row = (SURFACE if tc <= 8 else AIRBORNE)[tc]
    if None in row:
        return row[None]
    return row.get((s1, s2), (0, None))


def me_bits(me, first, n):
    """ME bits first..first+n-1 (1..56) of the 56-bit ME word."""
    return (me >> (57 - first - n)) & ((1 << n) - 1)


def me_of(frame):
    """The ME field; 0 for a 56-bit frame, whose "me" the parser reads past the end (parse.py:83-86)."""
    return int.from_bytes(bytes(frame["data"][4:11]), "big") if frame["nbits"] == 112 else 0


def t_of(frames):
    return frames["secs"].astype(np.float64) + frames["frac"]


def set_record(rec1, aux_bytes, outcome, version, nic):
    """Write the option's fields into a 1-element FIELDS_DTYPE slice: aux (16 bytes) and pad_ bytes 5..7."""
    rec1["aux"][0] = np.frombuffer(bytes(aux_bytes), dtype="<u4")
    pad = int(rec1["pad_"][0]) & 0xFFFFFFFFFF
    rec1["pad_"][0] = pad | (outcome << 40) | (version << 48) | (nic << 56)


def _f32(x):
    return np.float32(np.nan if x is None else x).tobytes()


class Checker:
    """Feed (frames, option-off records) call by call in stream order; get the option-on records back."""

    def __init__(self, S):
        self.S = S
        # every earlier op-status record: address, t, subtype, version, NIC-A, NIC-C
        self.w_icao = np.zeros(0, dtype=np.int64)
        self.w_t = np.zeros(0)
        self.w = []

    def reset(self):
        self.__init__(self.S)

    def _add_writer(self, icao, t, sub, ver, nica, nicc):
        self.w_icao = np.append(self.w_icao, icao)
        self.w_t = np.append(self.w_t, t)
        self.w.append((sub, ver, nica, nicc))

    def _position(self, out1, icao, t, tc, me):
        hits = np.flatnonzero(self.w_icao == icao)                 # a scan of every earlier op-status record
        surf = [h for h in hits if self.w[h][0] == 1]
        a = int(hits[-1]) if len(hits) else None
        c = int(surf[-1]) if surf else None
        a_ok = a is not None and 0.0 <= t - self.w_t[a] <= self.S
        c_ok = c is not None and 0.0 <= t - self.w_t[c] <= self.S
        if not a_ok or self.w[a][1] == 0:
            set_record(out1, bytes(4) + _f32(None) + bytes(8), NUC, 0 if a_ok else NO_VERSION, NUCP[tc])
            return
        ver, nica = self.w[a][1], self.w[a][2]
        surface = tc <= 8
        nicb = 0 if surface else (me_bits(me, 8, 1) if ver == 2 else nica)
        nicc = self.w[c][3] if (surface and ver == 2 and c_ok) else 0
        if ver == 1 and tc == 8:
            nic, rc = 0, None                                      # pyModeS's version-1 table
        else:
            nic, rc = lookup(tc, nica, nicc if surface else nicb)
        set_record(out1, bytes([nica, nicb, nicc, 0]) + _f32(rc) + bytes(8), NIC, ver, nic)

    def feed(self, frames, recs):
        ts = t_of(frames)
        out = recs.copy()
        for k in range(len(recs)):
            f, r = frames[k], recs[k]
            if not f["passed"] or r["df"] != 17 or r["status"] & FS_NOT_QUEUED:
                continue
            me, icao, t = me_of(f), int(r["icao"]), float(ts[k])
            if r["bds"] in (0x05, 0x06):
                self._position(out[k:k + 1], icao, t, int(r["ftc"]), me)
                continue
            if r["status"] != FS_NO_HANDLER:
                continue
            tc = me_bits(me, 1, 5)
            aux = bytearray(16)
            if tc == 31:
                sub, ver = me_bits(me, 6, 3), me_bits(me, 41, 3)
                if sub > 1 or ver > 2:
                    set_record(out[k:k + 1], aux, UNSUPPORTED, ver, 0)
                    continue
                aux[0:2] = me_bits(me, 9, 16).to_bytes(2, "little")
                aux[2:4] = me_bits(me, 25, 16).to_bytes(2, "little")
                aux[4] = sub
                nica = nicc = 0
                if ver:
                    nica = me_bits(me, 44, 1)
                    aux[5:12] = bytes([nica, me_bits(me, 45, 4), me_bits(me, 49, 2), me_bits(me, 51, 2),
                                       me_bits(me, 53, 1), me_bits(me, 54, 1), me_bits(me, 55, 1)])
                    if sub == 1:
                        nicc = me_bits(me, 20, 1)
                        aux[12:14] = bytes([nicc, me_bits(me, 21, 4)])
                set_record(out[k:k + 1], aux, OPSTATUS, ver, 0)
                self._add_writer(icao, t, sub, ver, nica, nicc)
            elif tc == 29:
                if me_bits(me, 6, 2) != 1:
                    set_record(out[k:k + 1], aux, UNSUPPORTED, NO_VERSION, 0)
                    continue
                aux[0:2] = me_bits(me, 10, 11).to_bytes(2, "little")
                aux[2:4] = me_bits(me, 21, 9).to_bytes(2, "little")
                aux[4:6] = me_bits(me, 31, 9).to_bytes(2, "little")
                aux[6:13] = bytes([me_bits(me, 8, 1), me_bits(me, 9, 1), me_bits(me, 30, 1), me_bits(me, 40, 4),
                                   me_bits(me, 44, 1), me_bits(me, 45, 2), me_bits(me, 47, 8)])
                set_record(out[k:k + 1], aux, TARGET_STATE, 2, 0)
        return out


def replay(frames, recs, S):
    return Checker(S).feed(frames, recs)


def outcome_of(recs):
    return (np.asarray(recs["pad_"], dtype=np.uint64) >> np.uint64(40)) & np.uint64(0xFF)


def eligible(frame, rec):
    """A record the option may write: a queued DF17 position or TC 29 / TC 31 squitter."""
    if not frame["passed"] or rec["df"] != 17 or rec["status"] & FS_NOT_QUEUED:
        return False
    if rec["bds"] in (0x05, 0x06):
        return True
    return rec["status"] == FS_NO_HANDLER and me_bits(me_of(frame), 1, 5) in (29, 31)


def assert_records_equal(got, want, tag):
    if got.tobytes() == want.tobytes():
        return
    bad = [k for k in range(len(got)) if got[k].tobytes() != want[k].tobytes()]
    k = bad[0]
    raise AssertionError("%s: %d records differ, first #%d: got pad_ %#x aux %s, want pad_ %#x aux %s"
                         % (tag, len(bad), k, int(got["pad_"][k]), [hex(x) for x in got["aux"][k]],
                            int(want["pad_"][k]), [hex(x) for x in want["aux"][k]]))
