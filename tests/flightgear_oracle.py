"""Sequential checker of the decoder option "flightgear" (include/airmodes_b200.h rules 1-5, DESIGN.md §8 "FlightGear
multiplayer feed"), written from the rules with Python floats and dicts: FgChecker.feed(frames, records) returns the
packets a decode of those records writes, continuing the state of earlier calls; packet() is rule 5 on its own.
tests/test_flightgear_cpu.py pins it to the unmodified reference (tests/golden/flightgear_golden.json.gz)."""
from __future__ import annotations

import math
import struct

NOT_QUEUED, NO_HANDLER, HAS_POS = 0x80, 0x01, 0x10
PACKET_BYTES = 232
WGS_A, WGS_E2 = 6378137.0, 0.0066943799901975848

MODELS = ["Aircraft/777-200/Models/777-200ER.xml", "Aircraft/c172p/Models/c172p.xml",
          "Aircraft/CitationX/Models/Citation-X.xml", "Aircraft/CRJ700-family/Models/CRJ700.xml",
          "Aircraft/757-200/Models/757-200.xml", "Aircraft/IDG-A32X/Models/A320neo-CFM.xml",
          "Aircraft/SR71-BlackBird/Models/Blackbird-SR71B.xml", "Aircraft/ec130/Models/ec130b4.xml",
          "Aircraft/ASK21-MI/Models/ask21mi.xml", "Aircraft/ZLT-NT/Models/ZLT-NT.xml",
          "Aircraft/cri-cri/Models/MC-15.xml", "Aircraft/YardStik/Models/yardstik.xml",
          "Aircraft/SpaceShip-One/Models/spaceshipone.xml", "Aircraft/followme/Models/follow_me.xml",
          "Aircraft/pushback/Models/Pushback.xml", "Aircraft/santa/Models/santa.xml"]
SANTA = 15
# categories[ftc - 1][cat] of parse.py:270-275 as model indices (SANTA where modelmap has no entry); row 2 has 7 entries
ROWS = [[0, SANTA, SANTA, SANTA, SANTA, SANTA, SANTA, SANTA],
        [0, 13, 14, SANTA, SANTA, SANTA, SANTA],
        [0, 8, 9, SANTA, 10, SANTA, 11, 12],
        [0, 1, 2, 3, 4, 5, 6, 7]]


def model(ftc: int, cat: int):
    """Rule 2: the model index, or None where the reference raises IndexError."""
    if not 1 <= ftc <= 4 or not 0 <= cat < len(ROWS[ftc - 1]):
        return None
    return ROWS[ftc - 1][cat]


def orientation(lat: float, lon: float, hdg: float):
    """The three orientation floats (as Python floats before packing), or None where the reference raises TypeError."""
    pi = math.pi
    lon_r, lat_r = lon * (pi / 180.), lat * (pi / 180.)
    zd2, yd2 = 0.5 * lon_r, -0.25 * pi - 0.5 * lat_r
    S, Sy, C, Cy = math.sin(zd2), math.sin(yd2), math.cos(zd2), math.cos(yd2)
    a = [-S * Sy, C * Sy, S * Cy, C * Cy]
    ra, dec, roll = hdg * (pi / 180.0), 0.0 * (pi / 180.0), 0.0 * (pi / 180.0)
    ca, sa, cd, sd, cr, sr = math.cos(ra), math.sin(ra), math.cos(dec), math.sin(dec), math.cos(roll), math.sin(roll)
    T = [[ca * cd, sa * cd, sd],
         [-ca * sd * sr - sa * cr, -sa * sd * sr + ca * cr, cd * sr],
         [-ca * sd * cr + sa * sr, -sa * sd * cr - ca * sr, cd * cr]]
    den = [1.0 + T[0][0] - T[1][1] - T[2][2], 1.0 - T[0][0] + T[1][1] - T[2][2],
           1.0 - T[0][0] - T[1][1] + T[2][2], 1.0 + T[0][0] + T[1][1] + T[2][2]]
    m = 0
    for i in range(1, 4):
        if den[i] > den[m]:
            m = i
    b = [0.0] * 4
    b[m] = 0.5 * math.sqrt(den[m])
    d = 4.0 * b[m]
    if m == 0:
        b[1], b[2], b[3] = (T[1][0] + T[0][1]) / d, (T[2][0] + T[0][2]) / d, -(T[2][1] - T[1][2]) / d
    elif m == 1:
        b[0], b[2], b[3] = (T[1][0] + T[0][1]) / d, (T[2][1] + T[1][2]) / d, -(T[0][2] - T[2][0]) / d
    elif m == 2:
        b[0], b[1], b[3] = (T[2][0] + T[0][2]) / d, (T[2][1] + T[1][2]) / d, -(T[1][0] - T[0][1]) / d
    else:
        b[0], b[1], b[2] = -(T[2][1] - T[1][2]) / d, -(T[0][2] - T[2][0]) / d, -(T[1][0] - T[0][1]) / d
    q = [a[3] * b[0] - a[2] * b[1] + a[1] * b[2] + a[0] * b[3],
         a[2] * b[0] + a[3] * b[1] - a[0] * b[2] + a[1] * b[3],
         -a[1] * b[0] + a[0] * b[1] + a[3] * b[2] + a[2] * b[3],
         -a[0] * b[0] - a[1] * b[1] - a[2] * b[2] + a[3] * b[3]]
    if not q[3] > 0:
        q = [-x for x in q]
    norm = math.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    if norm < 1e-12:
        return None
    rnorm = 1.0 / norm
    c = rnorm * q[3]
    angle = math.acos(1.0 if c > 1 else -1.0 if c < -1 else c)
    s = math.sin(angle)
    if s < 1e-12:
        return None
    angle *= 2
    return [angle * ((rnorm / s) * x) for x in q[:3]]


def llh2ecef(lat: float, lon: float, alt: float):
    lat, lon = lat * (math.pi / 180.0), lon * (math.pi / 180.0)
    sl = math.sin(lat)
    n = WGS_A / math.sqrt(1 - WGS_E2 * (sl * sl))
    return [(n + alt) * math.cos(lat) * math.cos(lon), (n + alt) * math.cos(lat) * math.sin(lon),
            (n * (1 - WGS_E2) + alt) * sl]


def packet(ident: bytes, m: int, lat: float, lon: float, alt: float, t: float, hdg: float, vel_ms: float,
           turn: float):
    """Rule 5: the 232 bytes, or None where the orientation does not exist. alt in feet; vel_ms and turn are the
    float32 values (already rounded)."""
    o = orientation(lat, lon, hdg)
    if o is None:
        return None
    pos = llh2ecef(lat, lon, alt * 0.3048)
    head = struct.pack("!4sLLLLL8s", b"FGFS", 0x00010001, 7, PACKET_BYTES, 0, 0, bytes(ident))
    body = struct.pack("!96sdd3d3f3f3f3f3fI", MODELS[m].encode("ascii"), t, 0.0, *pos, *o, vel_ms, 0, 0, 0, 0, turn,
                       0, 0, 0, 0, 0, 0, 0)
    return head + body


def f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


def kind(r) -> str | None:
    """Rules 1-4: what record r does ("callsign", "velocity", "position") or None."""
    if int(r["status"]) & (NOT_QUEUED | NO_HANDLER) or int(r["df"]) != 17:
        return None
    bds = int(r["bds"])
    if bds == 0x08:
        return "callsign" if model(int(r["ftc"]), int(r["cat"])) is not None else None
    if bds == 0x09:
        return "velocity" if int(r["subtype"]) in (0, 1) else None
    if bds in (0x05, 0x06):
        return "position" if int(r["status"]) & HAS_POS else None
    return None


class FgChecker:
    """The state of one decoder since its last reset: address -> (ident, model) and address -> (hdg, vel_ms, turn)."""

    def __init__(self):
        self.callsigns: dict[int, tuple] = {}
        self.velocities: dict[int, tuple] = {}

    def reset(self):
        self.__init__()

    def record(self, frame, r):
        """The packet record r writes (or None), after updating the state."""
        k = kind(r)
        a = int(r["icao"])
        if k == "callsign":
            self.callsigns[a] = (bytes(r["ident"]).ljust(8, b"\0")[:8], model(int(r["ftc"]), int(r["cat"])))
        elif k == "velocity":
            v = [float(x) for x in r["val"]]
            turn = v[3] if int(r["subtype"]) == 0 else 0
            self.velocities[a] = (v[1], f32(v[0] * 0.514444444), f32(turn * (math.pi / 180.)))
        elif k == "position" and a in self.callsigns and a in self.velocities:
            ident, m = self.callsigns[a]
            hdg, vel, turn = self.velocities[a]
            alt = float(int(r["altitude"])) if int(r["bds"]) == 0x05 else 0.0
            t = float(int(frame["secs"])) + float(frame["frac"])
            return packet(ident, m, float(r["lat"]), float(r["lon"]), alt, t, hdg, vel, turn)
        return None

    def feed(self, frames, records) -> bytes:
        """The packets of one decode call, concatenated."""
        return b"".join(p for p in (self.record(f, r) for f, r in zip(frames, records)) if p is not None)
