"""SURVEY.md 8 row f2: the message strings we emit are consumed by the reference's UNMODIFIED parser
(python/parse.py make_parser, :422-436). What the parser made of each message is recorded in
tests/golden/ref_python.json.gz (the `ref_py` fixture, tests/ref_golden.py); while recording, the reference files are
imported in place behind a stub `air_modes` package, never copied."""
import importlib.util
import math
import os
import sys
import types

from helpers import load_golden

REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _parse_with_reference(msgs):
    """-> per message None (no handler) or what the reference's make_parser published for it."""
    saved = {k: v for k, v in sys.modules.items() if k == "air_modes" or k.startswith("air_modes.")}
    pkg = types.ModuleType("air_modes")
    pkg.__path__ = []
    sys.modules["air_modes"] = pkg
    try:
        _load("air_modes.exceptions", os.path.join(REF, "exceptions.py"))
        _load("air_modes.altitude", os.path.join(REF, "altitude.py"))
        mt = _load("air_modes.modes_types", os.path.join(REF, "modes_types.py"))
        pkg.modes_report, pkg.stamp = mt.modes_report, mt.stamp
        parser = _load("air_modes.parse", os.path.join(REF, "parse.py"))
        out = []
        for m in msgs:
            pub = {}
            parser.make_parser(pub)(m)
            if "modes_dl" not in pub:       # the parser drops types it has no handler for (ADSBError)
                out.append(None)
                continue
            rep = pub["modes_dl"]
            df = rep.data.get_type()
            out.append({"ecc": rep.ecc, "rssi": rep.rssi, "secs": rep.timestamp.secs, "frac_secs": rep.timestamp.frac_secs,
                        "df": df, "typed": ("type%i_dl" % df) in pub,
                        "aa": rep.data["aa"] if df in (11, 17) else None})
        return out
    finally:
        for k in [k for k in sys.modules if k == "air_modes" or k.startswith("air_modes.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_reference_parser_accepts_our_messages(ref_py):
    meta, scenes = load_golden()
    seen = 0
    for s, _ in scenes:
        parsed = ref_py.get("make_parser/" + s["name"], s["msgs"], lambda: _parse_with_reference(s["msgs"]))
        assert len(parsed) == len(s["msgs"])
        for m, rep in zip(s["msgs"], parsed):
            data, ecc, ref, secs, frac = m.split()
            if rep is None:
                continue
            assert rep["ecc"] == int(ecc, 16)
            assert abs(rep["rssi"] - 10.0 * math.log10(max(1e-8, float(ref)))) < 1e-12
            assert rep["secs"] == int(secs) and rep["frac_secs"] == float(frac)
            df = int(data[:2], 16) >> 3
            assert rep["df"] == df and rep["typed"]
            if df in (11, 17) and data in s["sent"]:
                assert rep["aa"] == int(data[2:8], 16)      # ICAO address straight from our payload
                seen += 1
    assert seen >= 20
