"""SURVEY.md 8 row f4 (field decode: parse.py / altitude.py / cpr.py) - CPU side.

  * oracle/decode_oracle.py against the committed golden produced by the UNMODIFIED reference modules
    (tests/golden/make_decode_golden.py), bit-exact incl. every float;
  * the same against the reference's answers on fresh seeds and fuzzed bytes (tests/golden/ref_python.json.gz);
  * the product's per-message device code (gr_air_modes_b200/csrc/amb_decode_core.h, the `__host__ __device__`
    functions the CUDA kernels call) compiled for the host by tests/decode_host_shim.cc - a test-only harness, not a
    product path - against the golden, so the decode arithmetic is checked even where no GPU is present.
"""
import os
import sys

import pytest

from helpers import compare_decode, load_decode_golden

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def test_decode_oracle_matches_reference_golden():
    from oracle import decode_oracle as do
    n = 0
    for ci, case in enumerate(load_decode_golden()):
        recs = do.decode_batch([tuple(m) for m in case["msgs"]], case["location"])
        assert len(recs) == len(case["ref"])
        for k, (rec, ref) in enumerate(zip(recs, case["ref"])):
            compare_decode(rec, ref, 0.0, "case %d msg %d" % (ci, k))
            n += 1
    assert n > 5000


def _reference():
    """The unmodified reference modules (only called while recording, see tests/ref_golden.py)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_decode_golden as mg
    return mg


def test_decode_oracle_matches_live_reference_on_fresh_seeds(ref_py):
    import decode_cases
    from oracle import decode_oracle as do
    for seed in (101, 102, 103):
        loc, msgs = decode_cases.make_case(seed, location=(None if seed == 102 else (40.0 + seed % 7, -70.0)),
                                           seconds=30.0, surface_share=0.4)

        def live():
            mg = _reference()
            try:
                return mg.run_reference(loc, msgs, mg.load_reference())
            finally:
                mg.unload_reference()
        ref = ref_py.get("run_reference/seed%d" % seed, [loc, msgs], live)
        recs = do.decode_batch(msgs, loc)
        assert len(recs) == len(ref)
        for k, (rec, r) in enumerate(zip(recs, ref)):
            compare_decode(rec, r, 0.0, "seed %d msg %d" % (seed, k))


# ---- the product's decode arithmetic, compiled for the host by a test-only shim -------------------------------------
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    import ctypes as C
    import emul_build
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(emul_build.ROOT, "tests", "decode_host_shim.cc")))
    lib.shim_decode.restype = C.c_int
    lib.shim_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    lib.shim_nl.restype = C.c_int
    lib.shim_nl.argtypes = [C.c_double]
    return lib


def _shim_decode(lib, msgs, location):
    import ctypes as C
    import numpy as np
    from gr_air_modes_b200 import decode
    arr, n = decode.frames_from_messages(msgs)
    out = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    have, lat, lon = (0, 0.0, 0.0) if location is None else (1, location[0], location[1])
    assert lib.shim_decode(C.cast(arr, C.c_void_p), n, have, lat, lon, C.c_void_p(out.ctypes.data)) == 0
    return [decode.record_to_dict(r) for r in out]


def test_product_decode_core_on_host_matches_reference_golden(shim):
    assert shim.shim_sizeof_fields() == 144
    n = 0
    for ci, case in enumerate(load_decode_golden()):
        recs = _shim_decode(shim, [tuple(m) for m in case["msgs"]], case["location"])
        for k, (rec, ref) in enumerate(zip(recs, case["ref"])):
            # lat/lon bit-exact; hypot-based values to 1e-14 (CPython's math.hypot is its own routine, not libm's)
            compare_decode(rec, ref, 0.0, "case %d msg %d" % (ci, k), tol_libm=1e-14)
            n += 1
    assert n > 5000


def test_product_decode_core_equals_oracle_record_for_record(shim):
    """Every member of struct amb_fields, not only what the reference's consumers read."""
    import math
    import decode_cases
    from oracle import decode_oracle as do
    for seed in (201, 202):
        loc, msgs = decode_cases.make_case(seed, location=(None if seed == 202 else (-12.0, 130.9)), seconds=25.0,
                                           surface_share=0.5, n_random=500)
        want = do.decode_batch(msgs, loc)
        got = _shim_decode(shim, msgs, loc)
        for k, (g, w) in enumerate(zip(got, want)):
            for key, wv in w.items():
                gv = g[key]
                near = key in ("val", "range", "bearing")          # hypot & co: last-place differences allowed
                for a, b in (zip(gv, wv) if isinstance(wv, list) else [(gv, wv)]):
                    if isinstance(b, float) and math.isnan(b):
                        assert math.isnan(a), (seed, k, key, g, w)
                    elif near:
                        assert abs(a - b) <= 1e-14 * max(1.0, abs(b)), (seed, k, key, g, w)
                    else:
                        assert a == b, (seed, k, key, g, w)


def test_nl_table_equals_formula(shim):
    """amb_nl() (transition table built from the host libm) against cpr.py:46-51 evaluated directly."""
    import numpy as np
    from oracle import decode_oracle as do
    rng = np.random.default_rng(5)
    lats = np.concatenate([rng.uniform(-90, 90, 20000), [0.0, 86.999, 87.0, -87.0, 89.9, 10.4704713, -10.4704713]])
    # and a fine sweep across every transition
    for k in range(2, 60):
        lo, hi = 0.0, 87.0
        for _ in range(60):
            mid = (lo + hi) / 2
            if do.nl(mid) >= k:
                lo = mid
            else:
                hi = mid
        lats = np.concatenate([lats, lo + np.arange(-50, 51) * 1e-13, -(lo + np.arange(-50, 51) * 1e-13)])
    bad = [x for x in lats if shim.shim_nl(float(x)) != int(do.nl(float(x)))]
    # every latitude the decoder can reach, and the table's last bit: tests/test_decode_fp_edges_cpu.py
    assert not bad, bad[:10]


def test_report_lines_match_reference_printer(shim):
    """gr_air_modes_b200.report (the text apps/modes_rx prints by default) against the lines the UNMODIFIED
    python/msprint.py printed for the same messages (golden 'lines'); records from the host build of the product's
    decode arithmetic."""
    import decode_cases
    from gr_air_modes_b200 import report
    n = printed = 0
    for ci, case in enumerate(load_decode_golden()):
        msgs = [tuple(m) for m in case["msgs"]]
        recs = _shim_decode(shim, msgs, case["location"])
        for k, (text, rec, want) in enumerate(zip(decode_cases.message_strings(msgs), recs, case["lines"])):
            got = report.format_report(text, rec)
            assert got == want, (ci, k, text, got, want)
            n += 1
            printed += want is not None
    assert n > 5000 and printed > 4000


def test_fuzz_oracle_core_and_reports_against_live_reference(shim, ref_py):
    """Unconstrained message bytes (incl. what no slicer emits: long DFs in 56 bits, short DFs in 112 bits) through
    the UNMODIFIED parse.py / altitude.py / cpr.py / msprint.py, the oracle, the host build of the product's decode
    arithmetic, and report.py: all four agree message by message."""
    import numpy as np
    import decode_cases
    from gr_air_modes_b200 import report
    from oracle import decode_oracle as do
    rng = np.random.default_rng(77)
    msgs, t = [], 0.0
    for _ in range(12000):
        frame, ecc = decode_cases.raw_message(rng)
        t += float(rng.exponential(0.02)) + (12.0 if rng.random() < 0.001 else 0.0)
        msgs.append((frame.hex(), ecc, int(t), t - int(t)))
    texts = decode_cases.message_strings(msgs)
    locs = ([37.4, -122.1], None, [-45.0, 170.0])

    def live():
        """The first location's answers in full, the others' only where they differ from it (keeps the record small)."""
        mg = _reference()
        try:
            mods = mg.load_reference()
            runs = [(mg.run_reference(loc, msgs, mods), mg.run_reference_printer(loc, msgs, mods)) for loc in locs]
        finally:
            mg.unload_reference()
        (ref0, lines0), rest = runs[0], runs[1:]
        return {"ref": ref0, "lines": lines0,
                "delta": [{"ref": {str(k): r for k, r in enumerate(ref) if r != ref0[k]},
                           "lines": {str(k): x for k, x in enumerate(lines) if x != lines0[k]}} for ref, lines in rest]}
    rec = ref_py.get("fuzz77", [locs, msgs], live)
    for li, loc in enumerate(locs):
        ref, lines = list(rec["ref"]), list(rec["lines"])
        if li:
            for k, r in rec["delta"][li - 1]["ref"].items():
                ref[int(k)] = r
            for k, x in rec["delta"][li - 1]["lines"].items():
                lines[int(k)] = x
        want = do.decode_batch(msgs, loc)
        got = _shim_decode(shim, msgs, loc)
        assert len(ref) == len(lines) == len(msgs)
        for k, (w, g, r, text, line) in enumerate(zip(want, got, ref, texts, lines)):
            compare_decode(w, r, 0.0, "oracle %d %s" % (k, msgs[k][0]))
            compare_decode(g, r, 0.0, "core %d %s" % (k, msgs[k][0]), tol_libm=1e-13)
            assert report.format_report(text, g) == line, (k, text)
        assert sum("pos" in r for r in ref) > 300


class _ShimBackend:
    """Stands in for decode.batch_decoder in CPU tests: same decode()/set_location() surface, arithmetic from the host
    build of the product's decode core (tests/decode_host_shim.cc), state kept across calls like the device table."""

    def __init__(self, lib, location):
        import ctypes as C
        lib.shim_new.restype = C.c_void_p
        lib.shim_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
        self._lib, self._h, self._loc = lib, lib.shim_new(), location

    def set_location(self, loc):
        self._loc = loc

    def decode(self, frames, n):
        import ctypes as C
        import numpy as np
        from gr_air_modes_b200 import decode
        out = np.zeros(n, dtype=decode.FIELDS_DTYPE)
        have, lat, lon = (0, 0.0, 0.0) if self._loc is None else (1, self._loc[0], self._loc[1])
        self._lib.shim_step(self._h, C.cast(frames, C.c_void_p), n, have, lat, lon, C.c_void_p(out.ctypes.data))
        return out


def _cpr_sweep_events():
    """The reference's own self-test procedure (cpr.py:264-331: sweep of positions, even then odd report) plus surface
    reports, expiry and a moving receiver location, as a list of steps: ("new", location) starts a decoder,
    ("loc", location) moves the receiver, ("decode", now, icao, lat17, lon17, odd, surface) decodes one report."""
    import decode_cases as dc
    events, now = [], 0.0
    rounds = 1500
    for surface in (0, 1):
        loc = [35.0, -100.0]
        events.append(("new", list(loc)))
        for i in range(rounds):
            lat = i / (rounds / 170.) - 85 if not surface else 35.0 + (i % 50) * 1e-3
            if not surface and 100 <= i < 160:
                lat = 10.4704713 - 7e-4 + (i - 100) * 2.5e-5          # across an NL transition: boundary straddles
            lon = i / (rounds / 360.) - 180 if not surface else -100.0 + (i % 70) * 1e-3
            icao = (i * 7919) & 0xFFFFFF
            now = 1000.0 + i * 0.37 + (30.0 if i == 700 else 0.0)
            if i == 900:
                loc = [34.5, -99.5]
                events.append(("loc", list(loc)))
            for odd, dl in ((0, 0.0), (1, 1e-3)):
                la, lo = dc.cpr_encode(lat + dl, min(lon + dl, 180), odd, bool(surface))
                now += 0.01
                events.append(("decode", now, icao, la, lo, odd, surface))
    return rounds, events


def _run_cpr_events(events, new, exc_straddle, exc_nopos, clock):
    """Drive cpr_decoder-shaped objects through the steps; -> per decode step the result or "straddle" / "nopos"."""
    out, dec = [], None
    for ev in events:
        if ev[0] == "new":
            dec = new(list(ev[1]))
        elif ev[0] == "loc":
            dec.set_location(list(ev[1]))
        else:
            _, clock.now, icao, la, lo, odd, surface = ev
            try:
                out.append(dec.decode(icao, la, lo, odd, surface))
            except exc_straddle:
                out.append("straddle")
            except exc_nopos:
                out.append("nopos")
    return out


def test_cpr_decoder_dropin_class_against_the_reference_class(shim, ref_py):
    """decode.cpr_decoder (same methods, return list and exceptions as python/cpr.py:183-240) side by side with the
    UNMODIFIED reference class on the reference's own self-test procedure (_cpr_sweep_events); both run on one
    injected clock."""
    from gr_air_modes_b200 import decode
    from gr_air_modes_b200.errors import CPRBoundaryStraddleError, CPRNoPositionError
    rounds, events = _cpr_sweep_events()

    def live():
        mg = _reference()
        try:
            exc, alt, parse, cpr = mg.load_reference()
            clock = mg.Clock()
            cpr.time = type("T", (), {"time": staticmethod(clock.time)})
            return _run_cpr_events(events, cpr.cpr_decoder, exc.CPRBoundaryStraddleError, exc.CPRNoPositionError, clock)
        finally:
            mg.unload_reference()
    wants = ref_py.get("cpr_decoder_class", events, live)

    class Clock:
        now = 0.0

        def time(self):
            return self.now
    clock = Clock()
    gots = _run_cpr_events(events, lambda loc: decode.cpr_decoder(loc, clock=clock.time, _backend=_ShimBackend(shim, loc)),
                           CPRBoundaryStraddleError, CPRNoPositionError, clock)
    assert len(gots) == len(wants)
    ok = straddle = nopos = 0
    for k, (got, want) in enumerate(zip(gots, wants)):
        if isinstance(want, str):
            assert got == want, (k, got, want)
            straddle += want == "straddle"
            nopos += want == "nopos"
        else:
            assert got[0] == want[0] and got[1] == want[1], (k, got, want)     # lat/lon bit-exact
            assert abs(got[2] - want[2]) <= 1e-12 * max(1, want[2]) and abs(got[3] - want[3]) <= 1e-10
            ok += 1
    assert ok > 2500 and nopos >= 2 * rounds and straddle > 0
