"""Generates tests/golden/flightgear_golden.json.gz (the decoder option "flightgear", DESIGN.md §8 "FlightGear
multiplayer feed"). Run in the build container:

    python tests/golden/make_flightgear_golden.py

Every message of tests/flightgear_cases.scenes() (every frame queued) is pushed through the UNMODIFIED reference
modules python/parse.py, altitude.py, cpr.py, mlat.py, Quaternion.py and flightgear.py, imported where they lie in the
gr-air-modes tree ($AMB_REFERENCE_TREE) behind a stub `air_modes` package, as make_sbs1_golden.py does; nothing is
copied. Per message it does what make_parser (parse.py:422-436) and output_flightgear.output (flightgear.py:30-64) do:
modes_reply, then for DF17 output() on an object made with object.__new__. Only module and instance attributes are
patched, no file is touched: numpy.float (gone from numpy, mlat.py names it); an `air_modes.sql` stub (flightgear.py
imports output_sql and never uses it); flightgear.struct with a pack that ASCII-encodes str arguments - the one Python 3
repair, without which every pack raises struct.error; flightgear.time and cpr.time return the message's own secs +
frac; the socket is a recorder of sendto; print is silenced. The IndexError / TypeError that escape output() are
recorded as such. The packer grid of flightgear_cases.grid() goes through fg_posmsg(...).pack() directly. Nothing in the
output is hand-edited.
"""
import gzip
import json
import os
import struct
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import make_decode_golden as mdg  # noqa: E402
import make_sbs1_golden as msg  # noqa: E402

GRID_CALLSIGN, GRID_MODEL, GRID_VEL, GRID_TURN, GRID_T = "GRID1234", "HEAVY", 451.5, -1.5, 1700000000.25


class _Struct:
    """flightgear.struct: struct.pack with str arguments ASCII-encoded (the reference passes str to '4s' / '8s' /
    '96s')."""

    @staticmethod
    def pack(fmt, *args):
        return struct.pack(fmt, *[a.encode("ascii") if isinstance(a, str) else a for a in args])


class _Sock:
    def __init__(self):
        self.sent = []

    def sendto(self, data, addr):
        self.sent.append(bytes(data))


def load_reference():
    import numpy
    exc, parse, cpr, _ = msg.load_reference()
    if not hasattr(numpy, "float"):
        numpy.float = float
    if mdg.REF not in sys.path:
        sys.path.insert(0, mdg.REF)                     # flightgear.py: from Quaternion import Quat
    pkg = sys.modules["air_modes"]
    mlat = mdg._load("air_modes.mlat", os.path.join(mdg.REF, "mlat.py"))
    pkg.mlat = mlat
    sql = types.ModuleType("air_modes.sql")
    sql.output_sql = None
    sys.modules["air_modes.sql"] = sql
    fg = mdg._load("air_modes.flightgear", os.path.join(mdg.REF, "flightgear.py"))
    fg.struct = _Struct
    fg.print = lambda *a, **k: None
    return exc, parse, cpr, fg


def run_reference(location, msgs, mods=None):
    """-> one entry per message: [the packets it sent (hex), the escaping exception's name or None]."""
    exc, parse, cpr, fg = mods or load_reference()
    clock = mdg.Clock()
    cpr.time = types.SimpleNamespace(time=clock.time)
    fg.time = types.SimpleNamespace(time=clock.time)
    out = object.__new__(fg.output_flightgear)
    out.hostname, out.port = "127.0.0.1", 5000
    out.positions, out.velocities, out.callsigns = {}, {}, {}
    out._cpr = cpr.cpr_decoder(list(location) if location is not None else None)
    out.sock = _Sock()
    pkg = sys.modules["air_modes"]
    res = []
    for hexs, ecc, secs, frac in msgs:
        clock.now = float(secs) + float(frac)
        try:
            data = parse.modes_reply(int(hexs, 16))
            df = data.get_type()
        except exc.ADSBError:
            res.append([[], None])
            continue
        if df != 17:
            res.append([[], None])
            continue
        m = pkg.modes_report(data, int(ecc), 0.0, pkg.stamp(int(secs), float(frac)))
        n0, err = len(out.sock.sent), None
        try:
            out.output(m)
        except (IndexError, TypeError) as e:
            err = type(e).__name__                      # escapes output() in the reference
        res.append([[p.hex() for p in out.sock.sent[n0:]], err])
    return res


def run_grid(mods=None):
    """-> per grid point [lat, lon, alt, heading, the packet (hex) or None, the exception's name or None]."""
    _, _, _, fg = mods or load_reference()
    fg.time = types.SimpleNamespace(time=lambda: GRID_T)
    import flightgear_cases as fc
    out = []
    for lat, lon, alt, hdg in fc.grid():
        p, err = None, None
        try:
            p = fg.fg_posmsg(GRID_CALLSIGN, GRID_MODEL, lat, lon, alt, hdg, GRID_VEL, 0, GRID_TURN).pack().hex()
        except (IndexError, TypeError) as e:
            err = type(e).__name__
        out.append([lat, lon, alt, hdg, p, err])
    return out


def main():
    import flightgear_cases as fc
    mods = load_reference()
    out = []
    for name, loc, msgs in fc.scenes():
        res = run_reference(loc, msgs, mods)
        out.append({"name": name, "location": loc, "msgs": [[h, e, s, f] for h, e, s, f in msgs], "out": res})
        print("%-18s %5d messages, %5d packets, %d IndexError, %d TypeError" % (
            name, len(msgs), sum(len(r[0]) for r in res), sum(r[1] == "IndexError" for r in res),
            sum(r[1] == "TypeError" for r in res)))
    grid = run_grid(mods)
    print("grid %d points, %d TypeError" % (len(grid), sum(g[5] == "TypeError" for g in grid)))
    mdg.unload_reference()
    path = os.path.join(HERE, "flightgear_golden.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps({"scenes": out, "grid": grid, "grid_args": [GRID_CALLSIGN, GRID_MODEL, GRID_VEL, GRID_TURN,
                                                                       GRID_T]}, separators=(",", ":")).encode())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
