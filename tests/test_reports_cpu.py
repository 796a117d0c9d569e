"""Decoder option "reports" without a GPU: the text-report formatting the kernels run
(gr_air_modes_b200/csrc/amb_report_format.h, compiled for the host by tests/reports_host_shim.cc) against Python's %,
float() and report.format_report:
  * "%.6g" / "%.10g" of float32 and "%.10g" of double, read back with float(): every power of ten and its +-3-ulp
    neighbours, exact decimal ties, the largest floats, and 10^6 random bit patterns per type over the domain the
    stage formats (float32 levels above 2^-27, fracs from 2^-61 to 2^64);
  * the rssi against report.prefix at every float32 nearest 10^(k/10) and its neighbours, subnormal, zero, negative,
    NaN and infinite levels, and the two facts its exactness rests on: log10 of every power of ten in the range is
    exact in CPython, and 10 log10 of every other level read back lies at least 1e-11 from an integer;
  * the stamp "%.8f" for secs in {0, 1.7e9, 2^53 +- 1, 2^63, 2^64 - 1} and fracs at k 1e-8 +- 1 ulp and exact ties;
  * "%.Nf" for N = 0 .. 8 at ties, signs and 2^66;
  * the whole line against report.format_report on the records of the decoder's host-compiled arithmetic for every
    golden scene, and the line bodies against the golden's reference-printer lines; and on the records of the emulated
    decoder for the Comm-B, op-status and local-CPR cases, with every kind of line those options add;
  * option validation."""
import ctypes as C
import decimal
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import reports_cases as rc  # noqa: E402
from helpers import load_decode_golden  # noqa: E402

ROOT = emul_build.ROOT
INT_MIN = -(1 << 31)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "reports_host_shim.cc")))
    lib.shim_roundtrip.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p]
    lib.shim_rssi.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_void_p]
    lib.shim_prefix.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p]
    lib.shim_fixed.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_void_p]
    lib.shim_line.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_char_p]
    return lib


@pytest.fixture(scope="module")
def dshim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "decode_host_shim.cc")))
    lib.shim_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    return lib


def _roundtrip(shim, x, N):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.zeros_like(x)
    p10 = np.zeros(len(x), dtype=np.int32)
    shim.shim_roundtrip(C.c_void_p(x.ctypes.data), len(x), N, C.c_void_p(out.ctypes.data), C.c_void_p(p10.ctypes.data))
    return out, p10


def _check_roundtrip(shim, x, N):
    got, p10 = _roundtrip(shim, x, N)
    for v, g, p in zip(x.tolist(), got.tolist(), p10.tolist()):
        text = "%.*g" % (N, v)
        want = float(text)
        assert g == want and math.copysign(1, g) == math.copysign(1, want), (v, N, text, g)
        m = text.lstrip("-").split("e")
        digits = m[0].replace(".", "").lstrip("0").rstrip("0")
        assert (p != INT_MIN) == (digits == "1"), (v, text, p)
        if p != INT_MIN:
            assert float("1e%d" % p) == abs(want)


def _f32_neighbours(base, k=3):
    b = np.asarray(base, dtype=np.float32).view(np.int32)
    out = np.concatenate([(b + i).view(np.float32) for i in range(-k, k + 1)])
    return out[np.isfinite(out) & (out > np.float32(2.0 ** -27))]


def test_roundtrip_of_float32_levels(shim):
    pows = _f32_neighbours([np.float32(10.0 ** e) for e in range(-8, 39)])
    ties = np.array([1234565, 7777775, 1000005, 9999995], dtype=np.float32) * np.float32(1.0)   # 7-digit ints ending in 5
    top = _f32_neighbours([np.finfo(np.float32).max], 6)
    rng = np.random.default_rng(1)
    bits = rng.integers(np.float32(2.0 ** -27).view(np.int32), 0x7F800000, 1_000_000, dtype=np.int64).astype(np.int32)
    rand = bits.view(np.float32)
    for x in (pows, ties, top):
        for N in (6, 10):
            _check_roundtrip(shim, x.astype(np.float64), N)
    for N in (6, 10):
        x = rand.astype(np.float64)
        got, _ = _roundtrip(shim, x, N)
        want = np.array([float("%.*g" % (N, v)) for v in x.tolist()])
        assert np.array_equal(got, want), N


def test_roundtrip_of_double_fracs(shim):
    pows = np.concatenate([[10.0 ** e * (1 + i * 2.0 ** -52) for i in range(-3, 4)] for e in range(-18, 20)])
    ties = np.array([k / 512 for k in range(1, 512, 2)] + [0.5, 0.25, 0.125, 2.0 ** -30 * 3])
    rng = np.random.default_rng(2)
    lo, hi = np.float64(2.0 ** -61).view(np.int64), np.float64(2.0 ** 64).view(np.int64)
    rand = rng.integers(lo, hi, 1_000_000, dtype=np.int64).view(np.float64)
    _check_roundtrip(shim, pows, 10)
    _check_roundtrip(shim, ties, 10)
    _check_roundtrip(shim, -ties, 10)
    got, _ = _roundtrip(shim, rand, 10)
    want = np.array([float("%.10g" % v) for v in rand.tolist()])
    assert np.array_equal(got, want)


def _rssi(shim, lev, first):
    lev = np.ascontiguousarray(lev, dtype=np.float32)
    out = np.zeros(len(lev), dtype=np.int32)
    shim.shim_rssi(C.c_void_p(lev.ctypes.data), len(lev), int(first), C.c_void_p(out.ctypes.data))
    return out


def _py_rssi(lev, first):
    text = "%.*g" % (6 if first else 10, float(lev))
    try:
        return int(10.0 * math.log10(max(1e-8, float(text))))
    except OverflowError:
        return INT_MIN


def test_rssi_at_every_boundary_and_special_level(shim):
    base = [np.float32(10.0 ** (k / 10.0)) for k in range(-80, 386)]
    b = np.asarray(base, dtype=np.float32).view(np.int32)
    lev = np.concatenate([(b + i).view(np.float32) for i in range(-3, 4)])
    special = np.array([0.0, -0.0, -1.0, np.nan, -np.inf, np.inf, 1e-45, 1e-38, 7.45e-9, 2.0 ** -27, 1e-8, 1.0000001e-8,
                        np.finfo(np.float32).max], dtype=np.float32)
    lev = np.concatenate([lev, special])
    for first in (True, False):
        got = _rssi(shim, lev, first)
        want = [_py_rssi(x, first) for x in lev.tolist()]
        assert got.tolist() == want


def test_log10_facts_the_rssi_rests_on():
    """Every power of ten a level can read back as has an exact log10 in CPython; and for k = -79 .. 385 the decimals of
    6 and 10 digits nearest 10^(k/10) on either side - the read-back levels closest to the boundary - lie at least
    1e-11 from it in 10 log10, far beyond what an ulp of log10 can move."""
    for e in range(-8, 39):
        assert math.log10(float("1e%d" % e)) == e
    ctx = decimal.Context(prec=60)
    worst = 1.0
    for k in range(-79, 386):
        if k % 10 == 0:
            continue
        b = ctx.power(decimal.Decimal(10), ctx.divide(decimal.Decimal(k), decimal.Decimal(10)))
        for N in (6, 10):
            e = b.adjusted()
            unit = decimal.Decimal(1).scaleb(e - N + 1)
            lo = b.quantize(unit, rounding=decimal.ROUND_FLOOR, context=ctx)
            for d in (lo, lo + unit):
                L = float(d)
                t = ctx.multiply(decimal.Decimal(10), ctx.log10(decimal.Decimal(L)))
                worst = min(worst, abs(float(t - k)))
    assert worst > 1e-11, worst


def _prefix(shim, lev, secs, frac, first):
    n = len(secs)
    lev = np.ascontiguousarray(np.broadcast_to(np.float32(lev), (n,)))
    secs = np.ascontiguousarray(secs, dtype=np.uint64)
    frac = np.ascontiguousarray(frac, dtype=np.float64)
    out = np.zeros(n * 64, dtype=np.uint8)
    shim.shim_prefix(C.c_void_p(lev.ctypes.data), C.c_void_p(secs.ctypes.data), C.c_void_p(frac.ctypes.data), n,
                     int(first), C.c_void_p(out.ctypes.data))
    return [bytes(out[i * 64:(i + 1) * 64]).split(b"\0")[0].decode() for i in range(n)]


def test_stamp_against_report_prefix(shim):
    from gr_air_modes_b200 import report
    rng = np.random.default_rng(4)
    fracs = []
    for k in rng.integers(0, 10 ** 8, 200).tolist() + [0, 1, 99999999]:
        x = k * 1e-8
        fracs += [x, np.nextafter(x, 1.0), np.nextafter(x, -1.0), x + 5e-9]
    fracs += [j / 512 for j in range(1, 512, 2)] + [0.0, -0.0, 1.5, -0.25, 2.0 ** -70, 3.0, 7.9999999999]
    for secs in (0, 1700000000, 2 ** 53 - 1, 2 ** 53 + 1, 2 ** 63, 2 ** 64 - 1):
        got = _prefix(shim, 0.5, [secs] * len(fracs), fracs, False)
        for f, g in zip(fracs, got):
            text = "%.10g" % f
            assert g == report.prefix(float("%.10g" % np.float32(0.5)), secs, float(text)), (secs, f, g)
    assert _prefix(shim, 0.5, [2 ** 64 - 1], [0.0], False)[0].endswith(" 18446744073709551616.00000000) ")
    assert _prefix(shim, 0.5, [1], [float("nan")], False) == [""]
    assert _prefix(shim, 0.5, [1], [2.0 ** 64], False) == [""]


def _fixed(shim, x, prec, lim=63):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.zeros(len(x) * 48, dtype=np.uint8)
    shim.shim_fixed(C.c_void_p(x.ctypes.data), len(x), prec, lim, C.c_void_p(out.ctypes.data))
    return [bytes(out[i * 48:(i + 1) * 48]).split(b"\0")[0].decode() for i in range(len(x))]


def test_fixed_for_every_precision(shim):
    rng = np.random.default_rng(6)
    x = np.concatenate([np.arange(-40, 41) / 16.0, np.arange(-40, 41) / 8.0 + 0.5, [0.0, -0.0, -0.4, 2.5, 3.5, -2.5],
                        rng.uniform(-400, 400, 20000), rng.uniform(-1, 1, 5000) * 1e-6])
    for prec in range(9):
        assert _fixed(shim, x, prec) == ["%.*f" % (prec, v) for v in x.tolist()], prec
    big = np.array([2.0 ** 64, 2.0 ** 65 + 2048.0, -(2.0 ** 65), 2.0 ** 63 - 1024.0])
    assert _fixed(shim, big, 8, 66) == ["%.8f" % v for v in big.tolist()]
    assert _fixed(shim, np.array([2.0 ** 66]), 8, 66) == [""]


def _scene_records(dshim, frames, n, loc):
    from gr_air_modes_b200 import decode
    out = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    have, lat, lon = (0, 0.0, 0.0) if loc is None else (1, loc[0], loc[1])
    assert dshim.shim_decode(C.c_void_p(frames.ctypes.data), n, have, lat, lon, C.c_void_p(out.ctypes.data)) == 0
    return out


def _line(shim, f, r, first):
    buf = C.create_string_buffer(600)
    shim.shim_line(C.c_void_p(f.ctypes.data), C.c_void_p(r.ctypes.data), int(first), buf)
    return buf.value.decode("latin-1")


def test_lines_of_every_golden_scene_and_the_reference_printers_bodies(shim, dshim):
    from gr_air_modes_b200 import decode, report
    import decode_cases
    n = printed = 0
    for ci, case in enumerate(load_decode_golden()):
        msgs = [tuple(m) for m in case["msgs"]]
        arr, k = decode.frames_from_messages(msgs)
        fr = rc.frames_with_levels(arr, k, ci)
        recs = _scene_records(dshim, fr, k, case["location"])
        for i in range(k):
            f, r = fr[i:i + 1], recs[i:i + 1]
            got = _line(shim, f, r, i == 0)
            want = report.format_report(rc.slicer_text(fr[i], i == 0), recs[i])
            assert got == ("" if want is None else want + "\n"), (ci, i)
            ref = case["lines"][i]
            assert (ref is None) == (want is None), (ci, i)
            if ref is not None:
                assert got.split(") ", 1)[1] == ref.split(") ", 1)[1] + "\n", (ci, i)
                printed += 1
            n += 1
        assert len(decode_cases.message_strings(msgs)) == k
    assert n > 5000 and printed > 4000


def test_lines_of_the_comm_b_op_status_and_local_cpr_cases(shim, tmp_path_factory):
    """The whole line through the host shim against report.format_report on records with option results: the records
    of the emulated decoder (tests/simt/decode_emul.cc, the decoder's own kernels) over every op-status and Comm-B scene
    with its option on, and over local-CPR scenes with local_cpr on (positions only a local fix gives). Together they
    hold every kind of line commb and opstatus add."""
    import local_cpr_cases as lc
    import track_cases as tc
    from gr_air_modes_b200 import decode, report
    e = emul_build.decode_emul(tmp_path_factory)
    msgs, _ = lc.trajectory_scene(3, n_aircraft=12, seconds=60.0, drop=0.3, small_addresses=True)
    scenes = list(rc.text_option_scenes(small=True))
    scenes += [("local_trajectory", tc.frames_of(msgs), dict(local_cpr=10, loc=(48.0, 11.0))),
               ("local_chain", tc.frames_of(lc.chain_scene()), dict(local_cpr=10))]
    kinds, local_lines = set(), 0
    for name, fr, stages in scenes:
        stages = dict(stages)
        h = e.emul_new(17)
        try:
            emul_build.opts(e, h, stages.pop("loc", None), **stages)
            recs = np.zeros(len(fr), dtype=decode.FIELDS_DTYPE)
            assert e.emul_decode(h, C.c_void_p(fr.ctypes.data), len(fr), C.c_void_p(recs.ctypes.data)) == 0
        finally:
            e.emul_free(h)
        text, first = [], True
        for i in range(len(fr)):
            if int(recs[i]["status"]) & decode.FS_NOT_QUEUED:
                continue
            got = _line(shim, fr[i:i + 1], recs[i:i + 1], first)
            want = report.format_report(rc.slicer_text(fr[i], first), recs[i])
            first = False
            assert got == ("" if want is None else want + "\n"), (name, i)
            text.append(got)
            local_lines += bool(got) and int(decode.local_outcome(recs[i])) == decode.LOCAL_DECODED
        kinds |= rc.line_kinds("".join(text).encode("latin-1"))
    assert kinds >= rc.OPTION_LINE_KINDS, rc.OPTION_LINE_KINDS - kinds
    assert local_lines > 20


def test_option_validation():
    from gr_air_modes_b200 import decode
    assert decode.check_reports(True) == 1 and decode.check_reports(0) == 0
    for bad in (2, -1, "1", 1.0, None):
        with pytest.raises(ValueError):
            decode.check_reports(bad)
