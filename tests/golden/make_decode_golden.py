"""Generates tests/golden/decode_golden.json.gz (SURVEY.md 8 row f4). Run in the build container:

    python tests/golden/make_decode_golden.py

Every message of tests/decode_cases.CASES is pushed through the UNMODIFIED reference modules python/parse.py,
python/altitude.py and python/cpr.py (imported where they lie in the gr-air-modes tree, $AMB_REFERENCE_TREE, behind a stub `air_modes`
package; nothing is copied), calling exactly what the reference's own consumer python/msprint.py calls per DF
(handle0/4/5/11/17, printTCAS). The only patch: cpr.py stamps reports with time.time() (cpr.py:219-221); here
time.time returns the message's own timestamp secs + frac, which is the clock a batch decoder has.
Nothing in the output is hand-edited.
"""
import importlib.util
import json
import math
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    pkg = types.ModuleType("air_modes")
    pkg.__path__ = []
    sys.modules["air_modes"] = pkg
    exc = _load("air_modes.exceptions", os.path.join(REF, "exceptions.py"))
    alt = _load("air_modes.altitude", os.path.join(REF, "altitude.py"))
    mt = _load("air_modes.modes_types", os.path.join(REF, "modes_types.py"))
    pkg.modes_report, pkg.stamp = mt.modes_report, mt.stamp
    parse = _load("air_modes.parse", os.path.join(REF, "parse.py"))
    cpr = _load("air_modes.cpr", os.path.join(REF, "cpr.py"))
    return exc, alt, parse, cpr


def unload_reference():
    for k in [k for k in sys.modules if k == "air_modes" or k.startswith("air_modes.")]:
        del sys.modules[k]


class Clock:
    def __init__(self):
        self.now = 0.0

    def time(self):
        return self.now


def run_reference(location, msgs, mods=None):
    """-> list of dicts holding only what the reference computed for each message."""
    exc, alt, parse, cpr = mods or load_reference()
    clock = Clock()
    fake_time = types.SimpleNamespace(time=clock.time)
    cpr.time = fake_time                                  # the one patch (module attribute, file untouched)
    dec = cpr.cpr_decoder(list(location) if location is not None else None)
    out = []
    for hexs, ecc, secs, frac in msgs:
        clock.now = float(secs) + float(frac)
        r = {}
        try:
            data = parse.modes_reply(int(hexs, 16))
        except exc.NoHandlerError:
            out.append({"dropped": 1})
            continue
        df = data.get_type()
        r["df"] = df
        try:
            if df in (0, 16):
                r["vs"], r["ri"], r["sl"] = data["vs"], data["ri"], data["sl"]
                r["altitude"] = alt.decode_alt(data["ac"], True)
            elif df in (4, 20):
                r["fs"] = data["fs"]
                r["altitude"] = alt.decode_alt(data["ac"], True)
            elif df in (5, 21):
                r["fs"] = data["fs"]
                r["squawk"] = parse.decode_id(data["id"])
            elif df == 11:
                r["icao"], r["ca"] = data["aa"], data["ca"]
        except exc.MetricAltError:
            r["metric_alt"] = 1
        if df in (20, 21):
            bds1 = data["bds1"]
            r["bds"] = bds1
            if bds1 == 1:
                r["aux"] = [data["acs"], data["bcs"], data["ecs"], data["cfs"]]
            elif bds1 == 2:
                r["ident"] = parse.parseMB_id(data)
            elif bds1 == 3:
                tti = data["tti"]
                r["tti"] = tti
                r["ara"], r["rac"], r["rat"], r["mte"] = data["ara"], data["rac"], data["rat"], data["mte"]
                if tti == 1:
                    r["tid"] = parse.parseMB_TCAS_threatid(data)[4]
                elif tti == 2:
                    try:
                        t = parse.parseMB_TCAS_threatloc(data)
                        r["threat_alt"], r["tidr"], r["tidb"] = t[4], t[5], t[6]
                    except exc.MetricAltError:
                        r["threat_metric_alt"] = 1
        if df == 17:
            r["icao"], r["ca"] = data["aa"], data["ca"]
            bds = data["me"].get_type()
            r["bds"], r["ftc"] = bds, data["ftc"]
            try:
                if bds == 0x08:
                    r["cat"] = data["cat"]
                    r["ident"] = "".join(parse.charmap(data["ident"] >> (42 - 6 * i) & 0x3F) for i in range(8))
                elif bds == 0x06:
                    r["cpr"] = [data["cpr"], data["lat"], data["lon"]]
                    r["ground_track"] = data["gtk"] * 360. / 128
                    got = parse.parseBDS06(data, dec)
                    assert got[0] == r["ground_track"]
                    r["pos"] = got[1:]
                elif bds == 0x05:
                    r["cpr"] = [data["cpr"], data["lat"], data["lon"]]
                    got = parse.parseBDS05(data, dec)
                    r["altitude"] = got[0]
                    r["pos"] = got[1:]
                elif bds == 0x09:
                    sub = data["bds09"].get_type()
                    r["subtype"] = sub
                    if sub == 0:
                        r["val"] = [float(x) for x in parse.parseBDS09_0(data)]
                    elif sub == 1:
                        r["val"] = [float(x) for x in parse.parseBDS09_1(data)]
                    elif sub == 3:
                        v = parse.parseBDS09_3(data)
                        r["ast"] = 1 if v[1] == "TAS" else 0
                        r["val"] = [float(v[0]), float(v[2]), float(v[3]), float(v[4])]
                elif bds == 0x61:
                    r["eps"] = data["eps"]
            except exc.CPRBoundaryStraddleError:
                r["cpr_error"] = "straddle"
            except exc.CPRNoPositionError:
                r["cpr_error"] = "nopos"
        out.append(r)
    return out


class PubSub(dict):
    """Stand-in for gnuradio.gr.pubsub (a dict whose assignments call the subscribers), all msprint.py needs."""

    def __init__(self):
        dict.__init__(self)
        self._subs = {}

    def subscribe(self, key, fn):
        self._subs.setdefault(key, []).append(fn)

    def __setitem__(self, key, val):
        dict.__setitem__(self, key, val)
        for fn in self._subs.get(key, []):
            fn(val)


def run_reference_printer(location, msgs, mods=None):
    """The reference's own consumer chain: make_parser (parse.py:422-436) -> pubsub -> output_print (msprint.py),
    one fresh cpr_decoder. -> per message the printed line or None."""
    exc, alt, parse, cpr = mods or load_reference()
    pkg = sys.modules["air_modes"]
    for name in dir(parse):
        if not name.startswith("_"):
            setattr(pkg, name, getattr(parse, name))
    msprint = _load("air_modes.msprint", os.path.join(REF, "msprint.py"))
    clock = Clock()
    cpr.time = types.SimpleNamespace(time=clock.time)
    dec = cpr.cpr_decoder(list(location) if location is not None else None)
    pub = PubSub()
    got = []
    msprint.output_print(dec, pub, callback=got.append)
    publish = parse.make_parser(pub)
    lines = []
    import decode_cases
    for text, (hexs, ecc, secs, frac) in zip(decode_cases.message_strings(msgs), msgs):
        clock.now = float(secs) + float(frac)
        del got[:]
        try:
            publish(text)
        except IndexError:              # parseBDS08's category table has a short row (parse.py:264,268)
            pass
        assert len(got) <= 1
        lines.append(got[0] if got else None)
    return lines


def main():
    import decode_cases
    mods = load_reference()
    cases = []
    for kw in decode_cases.CASES:
        loc, msgs = decode_cases.make_case(**kw)
        ref = run_reference(loc, msgs, mods)
        stat = {}
        for r in ref:
            k = "dropped" if "dropped" in r else "df%d%s" % (r["df"], ("/%02x" % r["bds"]) if r.get("bds") is not None and r["df"] == 17 else "")
            stat[k] = stat.get(k, 0) + 1
        npos = sum(1 for r in ref if "pos" in r)
        nstr = sum(1 for r in ref if r.get("cpr_error") == "straddle")
        print("seed", kw["seed"], len(msgs), "msgs;", npos, "positions,", nstr, "straddles;", stat)
        lines = run_reference_printer(loc, msgs, mods)
        print("   printed lines:", sum(1 for x in lines if x is not None))
        cases.append({"args": {k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()},
                      "location": loc, "msgs": [list(m) for m in msgs], "ref": ref, "lines": lines})
    unload_reference()

    def clean(o):
        if isinstance(o, float) and (math.isnan(o) or math.isinf(o)):
            return None
        if isinstance(o, dict):
            return {k: clean(v) for k, v in o.items()}
        if isinstance(o, (list, tuple)):
            return [clean(v) for v in o]
        return o
    import gzip
    path = os.path.join(HERE, "decode_golden.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps(clean({"cases": cases}), separators=(",", ":")).encode())
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
