"""Generates tests/golden/coverage_golden.json.gz (the decoder option "coverage", DESIGN.md §8 "Receiver coverage").
Run in the build container:

    python tests/golden/make_coverage_golden.py

The UNMODIFIED reference module python/az_map.py is imported where it lies in the gr-air-modes tree
($AMB_REFERENCE_TREE) behind the stub `air_modes` package of make_decode_golden.py, with parse.py, altitude.py and cpr.py
unmodified beside it; nothing is copied. az_map.py imports PyQt4 for its widget; a small stand-in defined below supplies
QtCore.QObject, a no-op pyqtSignal and inert QtGui / Qt names for the class attributes evaluated at import.

az_map_model.npoints is set to 72 before the model is constructed. That is the attribute's value under the Python 2 the
GUI ran on, where 360/5 is the integer 72; under Python 3 it is 72.0 and range(0, 72.0) raises in __init__. Row
arithmetic is unaffected: az_map.py:66 divides by 180./npoints and 360./npoints, floats either way.

Two further patches, both module or instance attributes, no file touched: cpr.py's time.time returns the message's own
secs + frac (as make_decode_golden.py), and az_map.py's global `air_modes` - the package name it calls parseBDS05 /
parseBDS06 through (az_map.py:195,198) without importing it - is bound to the stub package carrying parse.py's
functions. The model's addRecord is wrapped on the instance to record its arguments, then called unchanged.

It records:
  (a) "calls": az_map_model.addRecord on boundary triples - bearings 0, every 5i + 2.5 and its neighbouring doubles,
      360 - ulp and 360; altitudes -1300, -1000, 0, 1 and every band edge and its neighbours up to 30001 and 10^5;
      ranges 0, the smallest subnormal, a new largest value, that value again (equal to the cell), half of it - and for
      every call the cells it changed, [row, col, new value]; "final" the grid at the end.
  (b) "scenes": az_map_output.output (an object made with object.__new__, no publisher) over every DF17 message that
      make_parser would publish (parse.py:422-436), for tests/decode_cases.CASES, the scenes of tests/track_cases.py and
      tests/local_cpr_cases.chain_scene, each with a receiver location: the messages' digest, the addRecord calls with
      a range ([message index, bearing, altitude, range]) and the final grid. It also confirms that no record the
      decoder counts (oracle/decode_oracle.py's records, rule 1) is a BDS0,5 without an altitude. The same
      messages without a location: the TypeErrors addRecord(None, ...) raises are counted and the grid is checked to
      stay all zeros.
Nothing in the output is hand-edited.
"""
import copy
import gzip
import hashlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import make_decode_golden as mdg  # noqa: E402

DEFAULT_LOCATION = [47.9, 11.1]          # for the scenes that come without one


class _Signal:
    def __init__(self, *a, **k):
        pass

    def emit(self, *a):
        pass

    def connect(self, *a):
        pass


class _Inert:
    """Any attribute, any call: an inert stand-in for the Qt names az_map.py evaluates at import."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Inert()

    def __getattr__(self, name):
        return _Inert()


def _qt_stand_in():
    core = types.ModuleType("PyQt4.QtCore")

    class QObject:
        def __init__(self, parent=None):
            pass

    core.QObject, core.pyqtSignal, core.Qt = QObject, _Signal, _Inert()
    core.QSize = core.QRectF = core.QPointF = _Inert
    gui = types.ModuleType("PyQt4.QtGui")

    class QWidget:
        def __init__(self, parent=None):
            pass

    gui.QWidget = QWidget
    for name in ("QPen", "QColor", "QBrush", "QPainter", "QPainterPath", "QGridLayout", "QApplication"):
        setattr(gui, name, _Inert)
    pkg = types.ModuleType("PyQt4")
    pkg.QtCore, pkg.QtGui = core, gui
    sys.modules.update({"PyQt4": pkg, "PyQt4.QtCore": core, "PyQt4.QtGui": gui})


def load_reference():
    exc, alt, parse, cpr = mdg.load_reference()
    pkg = sys.modules["air_modes"]
    pkg.parseBDS05, pkg.parseBDS06 = parse.parseBDS05, parse.parseBDS06
    pkg.exceptions = exc
    _qt_stand_in()
    az = mdg._load("air_modes.az_map", os.path.join(mdg.REF, "az_map.py"))
    az.air_modes = pkg
    az.az_map_model.npoints = 72
    return exc, parse, cpr, az


def _model(az, calls):
    m = az.az_map_model()
    add = m.addRecord

    def recording(bearing, altitude, distance):
        calls.append((bearing, altitude, distance))
        add(bearing, altitude, distance)
    m.addRecord = recording
    return m


def boundary_calls(az):
    """(a): [[bearing, altitude, range, [[row, col, value], ...]], ...] and the final grid."""
    bearings = [0.0]
    for i in range(72):
        e = 5.0 * i + 2.5
        bearings += [float(np.nextafter(e, 0.0)), e, float(np.nextafter(e, 400.0))]
    bearings += [float(np.nextafter(360.0, 0.0)), 360.0]
    alts = [-1300, -1000, 0, 1]
    for a in (0, 1000, 2000, 5000, 10000, 15000, 20000, 25000, 30000):
        alts += [a - 1, a, a + 1]
    alts = sorted(set(alts + [100000]))
    pairs = [(b, alts[k % len(alts)]) for k, b in enumerate(bearings)]
    pairs += [(b, a) for a in alts for b in (0.0, float(np.nextafter(2.5, 0.0)), 2.5, 177.5, 357.5, 360.0)]
    m = az.az_map_model()
    out, big = [], 1.0
    for b, a in pairs:
        big += 0.37
        for r in (0.0, 5e-324, big, big, big * 0.5):
            before = copy.deepcopy(m._data)
            m.addRecord(b, a, r)
            changed = [[i, j, m._data[i][j]] for i in range(72) for j in range(9) if m._data[i][j] != before[i][j]]
            out.append([b, a, r, changed])
    return out, [list(map(float, row)) for row in m._data]


def digest(msgs) -> str:
    return hashlib.sha1(json.dumps([[h, int(e), int(s), float(f)] for h, e, s, f in msgs]).encode()).hexdigest()


def run_output(mods, location, msgs):
    """az_map_output.output over the DF17 messages make_parser publishes -> (addRecord calls with a range as
    [index, bearing, altitude, range], grid, TypeErrors)."""
    exc, parse, cpr, az = mods
    pkg = sys.modules["air_modes"]
    clock = mdg.Clock()
    cpr.time = types.SimpleNamespace(time=clock.time)
    calls = []
    out = object.__new__(az.az_map_output)
    out._cpr = cpr.cpr_decoder(list(location) if location is not None else None)
    out.model = _model(az, calls)
    got, type_errors = [], 0
    for k, (hexs, ecc, secs, frac) in enumerate(msgs):
        clock.now = float(secs) + float(frac)
        try:
            data = parse.modes_reply(int(hexs, 16))
        except exc.ADSBError:
            continue                                    # make_parser publishes nothing
        if data.get_type() != 17:
            continue
        del calls[:]
        try:
            out.output(pkg.modes_report(data, int(ecc), 0.0, pkg.stamp(int(secs), float(frac))))
        except TypeError:
            type_errors += 1                            # addRecord(None, ...) without a receiver location
        assert len(calls) <= 1
        if 5 <= data["ftc"] <= 18:                      # else output() adds (0, 0, 0), which changes nothing
            got += [[k, float(b), int(a), float(r)] for b, a, r in calls if b is not None]
    return got, [list(map(float, row)) for row in out.model._data], type_errors


def scenes():
    """(name, location, msgs): the decode golden's cases, the track scenes and the local CPR chain scene."""
    import decode_cases
    import local_cpr_cases
    import track_cases
    for kw in decode_cases.CASES:
        loc, msgs = decode_cases.make_case(**kw)
        yield "decode_seed%d" % kw["seed"], loc if loc is not None else DEFAULT_LOCATION, msgs
    for name, loc, msgs, _ in track_cases.scenes():
        if not name.startswith("case"):
            yield "track_" + name, loc if loc is not None else DEFAULT_LOCATION, msgs
    yield "local_chain", [48.0, 11.0], local_cpr_cases.chain_scene()


def main():
    import coverage_oracle
    from oracle import decode_oracle
    mods = load_reference()
    calls, final = boundary_calls(mods[3])
    print("boundary: %d addRecord calls, %d cells changed" % (len(calls), sum(len(c[3]) for c in calls)))
    out = []
    for name, loc, msgs in scenes():
        got, grid, te = run_output(mods, loc, msgs)
        assert te == 0, name
        recs = decode_oracle.decode_batch(msgs, loc)
        assert all(r["bds"] == 0x06 or r["altitude"] != decode_oracle.NO_ALT   # no counted BDS0,5 lacks its altitude
                   for r in recs if coverage_oracle.counted(r) is not None), name
        n_got, grid0, te0 = run_output(mods, None, msgs)
        assert not n_got and all(v == 0 for row in grid0 for v in row), name
        out.append({"name": name, "location": loc, "digest": digest(msgs), "records": got, "grid": grid,
                    "type_errors_without_location": te0})
        print("%-20s %5d messages, %5d ranges, %3d cells set; without a location %d TypeErrors, grid empty" % (
            name, len(msgs), len(got), sum(v > 0 for row in grid for v in row), te0))
    mdg.unload_reference()
    for k in ("PyQt4", "PyQt4.QtCore", "PyQt4.QtGui"):
        sys.modules.pop(k, None)
    path = os.path.join(HERE, "coverage_golden.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps({"calls": calls, "final": final, "scenes": out}, separators=(",", ":")).encode())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
