"""Generates tests/golden/sbs1_golden.json.gz (the decoder option "sbs1", DESIGN.md §8 "SBS-1 feed"). Run in the build
container:

    python tests/golden/make_sbs1_golden.py

Every message of tests/decode_cases.CASES and tests/sbs1_cases.scenes() (every frame queued) is pushed through the
UNMODIFIED reference modules python/parse.py, python/altitude.py, python/cpr.py and python/sbs1.py, imported where they
lie in the gr-air-modes tree ($AMB_REFERENCE_TREE) behind a stub `air_modes` package, as make_decode_golden.py does;
nothing is copied. Per message it does what make_parser (parse.py:422-436) and output_sbs1.output (sbs1.py:92-103) do:
modes_reply, then for DF0/4/5/11/17 output_sbs1.parse on an object made with object.__new__ (so no socket is bound
and no thread starts). Three patches, all module or instance attributes, no file touched: cpr.py's time.time returns
the message's own secs + frac (as make_decode_golden.py); output_sbs1.current_time returns the rule-5 strings of the
message's stamp (tests/sbs1_oracle.stamp, UTC); and the ValueError / IndexError that escape output() are recorded as
such. Each scene stays under 10000 aircraft, where sbs1.py's Python 2 pruning never runs. Nothing in the output is
hand-edited.
"""
import gzip
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import make_decode_golden as mdg  # noqa: E402

SBS1_LOCATION = [47.9, 11.1]


def load_reference():
    exc, alt, parse, cpr = mdg.load_reference()
    pkg = sys.modules["air_modes"]
    pkg.decode_alt, pkg.decode_id = alt.decode_alt, parse.decode_id
    for name in ("parseBDS05", "parseBDS06", "parseBDS08", "parseBDS09_0", "parseBDS09_1"):
        setattr(pkg, name, getattr(parse, name))
    pkg.exceptions = exc
    sbs1 = mdg._load("air_modes.sbs1", os.path.join(mdg.REF, "sbs1.py"))
    return exc, parse, cpr, sbs1


def run_reference(location, msgs, mods=None):
    """-> one entry per message: [published (0/1), aircraft id or 0, the line or None, the escaping exception's name or
    None]."""
    import types

    import sbs1_oracle as so
    exc, parse, cpr, sbs1 = mods or load_reference()
    clock = mdg.Clock()
    cpr.time = types.SimpleNamespace(time=clock.time)
    out = object.__new__(sbs1.output_sbs1)
    out._s = types.SimpleNamespace(close=lambda: None)     # __del__ closes the listening socket it never made
    out._aircraft_id_map, out._aircraft_id_count = {}, 0
    out._cpr = cpr.cpr_decoder(list(location) if location is not None else None)
    stamp = [None]
    out.current_time = lambda: list(stamp[0])
    pkg = sys.modules["air_modes"]
    res = []
    for hexs, ecc, secs, frac in msgs:
        clock.now = float(secs) + float(frac)
        try:
            data = parse.modes_reply(int(hexs, 16))
            df = data.get_type()
        except exc.ADSBError:
            res.append([0, 0, None, None])
            continue
        if df not in (0, 4, 5, 11, 17):
            res.append([0, 0, None, None])
            continue
        msg = pkg.modes_report(data, int(ecc), 0.0, pkg.stamp(int(secs), float(frac)))
        stamp[0] = so.stamp(int(secs), float(frac))
        line, err = None, None
        try:
            line = out.parse(msg)
        except exc.ADSBError:
            pass                                        # output() swallows it (sbs1.py:102-103)
        except (ValueError, IndexError) as e:
            err = type(e).__name__                      # escapes output() in the reference
        addr = data["aa"] if df in (11, 17) else int(ecc)
        res.append([1, out._aircraft_id_map[addr], line, err])
    return res


def scenes():
    """(name, location, msgs) of the golden: the decode golden's cases and the SBS-1 scenes."""
    import decode_cases
    import sbs1_cases
    for kw in decode_cases.CASES:
        loc, msgs = decode_cases.make_case(**kw)
        yield "decode_seed%d" % kw["seed"], loc, msgs
    for name, msgs in sbs1_cases.scenes():
        yield name, SBS1_LOCATION, msgs


def main():
    mods = load_reference()
    out = []
    for name, loc, msgs in scenes():
        res = run_reference(loc, msgs, mods)
        ids = {r[1] for r in res if r[0]}
        assert len(ids) < 10000, name
        out.append({"name": name, "location": loc, "msgs": [[h, e, s, f] for h, e, s, f in msgs], "out": res})
        print("%-18s %5d messages, %5d published, %5d lines, %d aircraft, %d ValueError, %d IndexError" % (
            name, len(msgs), sum(r[0] for r in res), sum(r[2] is not None for r in res), len(ids),
            sum(r[3] == "ValueError" for r in res), sum(r[3] == "IndexError" for r in res)))
    mdg.unload_reference()
    path = os.path.join(HERE, "sbs1_golden.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps({"scenes": out}, separators=(",", ":")).encode())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
