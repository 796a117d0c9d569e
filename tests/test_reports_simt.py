"""The text-report stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_reports.cuh, enqueued last by the decoder's
own amb_decode_launch) on the host under the SIMT emulator (tests/simt/simt_emul.h), through the decoder harness
tests/simt/decode_emul.cc with the accessors of tests/simt/decode_reports_emul.cc: the packed text of every call byte
for byte against report.format_report of the slicer's text of each frame and the decoder's own record, for single
messages, cuts at 31/32/33 and random splits, with the other stages on and off, the first-message flag across calls,
after a reset and with the option turned on mid-stream, a call of nothing but the longest lines, and every scene of
the op-status and Comm-B case generators with those options on, which hold every kind of line they add. The launch
count is three more with the option on and unchanged with it off (also with the coverage map on), and nothing is
allocated while it is off. Eight mutants must fail: %.Nf rounding half up, the raw frac in place of its "%.10g" round
trip, the first message's precision ignored, a scan that drops the last block, an op-status line with the wrong byte
for NICbaro, a target-state baro off by one step, target-state modes shown without their valid bit, and a Comm-B Mach
number with the wrong LSB."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import reports_cases as rc  # noqa: E402
from helpers import load_decode_golden  # noqa: E402

HARNESS = os.path.join("tests", "simt", "decode_reports_emul.cc")


def _bind(tmp_path_factory, src):
    e = emul_build.decode_emul(tmp_path_factory, src)
    e.emul_set_reports.argtypes = [C.c_void_p, C.c_int]
    e.emul_report_text.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    e.emul_reports_state.argtypes = [C.c_void_p]
    e.emul_set_coverage.argtypes = [C.c_void_p, C.c_int]
    e.simt_launch_count.restype = C.c_ulonglong
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(tmp_path_factory, os.path.join(emul_build.ROOT, HARNESS))


def _scenes():
    """The golden scenes' frames (levels spread over the receiver's range) and locations; the small pairing table of
    the harness needs the position squitters' addresses below 2^15."""
    from gr_air_modes_b200 import decode
    out = []
    for ci, case in enumerate(load_decode_golden()):
        arr, n = decode.frames_from_messages([tuple(m) for m in case["msgs"]])
        fr = rc.frames_with_levels(arr, n, ci)
        out.append((fr, case["location"]))
    return out


def _stamp_frames():
    """DF11 replies (always printed) with stamps at the edges of "%.8f": secs from 0 to 2^64 - 1, fracs at k 1e-8 +
    5e-9 -+ 1e-13 (where the "%.10g" round trip moves the 8th decimal), exact ties j / 512, and the first level just
    below 10, where precision 6 and 10 give different rssi."""
    from gr_air_modes_b200 import decode
    raw = bytes.fromhex("5d4840d6aaaaaa")
    msgs = []
    rng = np.random.default_rng(3)
    for secs in (0, 1700000000, 2 ** 53 + 1, 2 ** 63, 2 ** 64 - 1):
        for k in rng.integers(0, 10 ** 8, 12):
            for d in (-1e-13, 1e-13, 0.0):
                msgs.append((raw.hex(), 0, secs, float(k) * 1e-8 + 5e-9 + d))
    msgs += [(raw.hex(), 0, secs, j / 512) for secs in (0, 1700000000) for j in range(1, 512, 34)]
    arr, n = decode.frames_from_messages(msgs)
    fr = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=n).copy()
    fr["ref_level"] = np.float32(0.25)
    fr["ref_level"][0] = np.float32(9.999999)
    return fr


def _tcas_frames(n):
    """DF20 TCAS replies (bds1 = 3, tti = 2) with every resolution and complement bit set and a threat altitude: the
    longest line the stage writes."""
    from gr_air_modes_b200 import decode
    mb = (0x30 << 48) | (0x3FFF << 34) | (0xF << 30) | (1 << 29) | (1 << 28) | (2 << 26) | (0x0ABC << 13) | (0x7F << 6)
    body = bytes([20 << 3 | 0, 0x00, 0x0A, 0xB8]) + mb.to_bytes(7, "big")
    msgs = [((body + bytes([0x12, 0x34, k & 0xFF])).hex(), 0x123456, 100 + k, 0.5) for k in range(n)]
    arr, m = decode.frames_from_messages(msgs)
    return np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=m).copy()


def _run(e, h, frames, opts, reports=1):
    """One emulated decode; returns (records, the call's text or None when the option is off)."""
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    e.emul_set_reports(h, reports)
    assert e.emul_decode(h, C.c_void_p(frames.ctypes.data), len(frames), opts, C.c_void_p(recs.ctypes.data)) == 0
    if not reports:
        return recs, None
    n = C.c_size_t()
    buf = C.create_string_buffer(len(frames) * 480 + 1)
    assert e.emul_report_text(h, len(frames), buf, len(buf), C.byref(n)) == 0
    return recs, buf.raw[: n.value]


def _check_stream(e, frames, loc, cuts, opts=None, log2=17):
    """The stream cut at `cuts`, one call per piece: each call's text equals the expected text of its frames and
    records, the first call's first queued frame at precision 6."""
    h = e.emul_new(log2)
    try:
        o = opts if opts is not None else emul_build.opts(loc)
        first = True
        for a, b in zip([0] + list(cuts), list(cuts) + [len(frames)]):
            if a == b:
                continue
            part = np.ascontiguousarray(frames[a:b])
            recs, text = _run(e, h, part, o)
            want = rc.expected_text(part, recs, first)
            assert text == want, (a, b, text[:300], want[:300])
            first = first and not np.any((recs["status"] & 0x80) == 0)
    finally:
        e.emul_free(h)


def _small(frames):
    """The frames whose position squitters' addresses fit the harness's 2^17-slot pairing table."""
    from gr_air_modes_b200 import decode
    keep = []
    for k, f in enumerate(frames):
        icao = int.from_bytes(bytes(f["data"][1:4]), "big")
        keep.append(int(f["df"]) != 17 or icao < (1 << 15))
    return np.ascontiguousarray(frames[np.asarray(keep)])


def test_scenes_in_one_call_single_messages_and_cuts(emul):
    for fr, loc in _scenes()[:2]:
        fr = _small(fr)[:400]
        _check_stream(emul, fr, loc, [])
        _check_stream(emul, fr[:40], loc, list(range(1, 40)))
        _check_stream(emul, fr, loc, [31, 32, 33, 64, 65, 127, 128, 129])


def test_random_splits(emul):
    rng = np.random.default_rng(7)
    for fr, loc in _scenes()[2:4]:
        fr = _small(fr)[:600]
        _check_stream(emul, fr, loc, sorted(rng.integers(0, len(fr), 9).tolist()))


@pytest.mark.parametrize("stages", [dict(local_cpr=10), dict(commb=30, opstatus=60), dict(track=60, track_ext=60),
                                    dict(sbs1=1), dict(local_cpr=10, commb=30, opstatus=60, track=60, sbs1=1)])
def test_with_other_stages_on(emul, stages):
    fr, loc = _scenes()[0]
    fr = _small(fr)[:500]
    _check_stream(emul, fr, loc, [200], emul_build.opts(loc, **stages))


def test_stamps_and_first_level(emul):
    fr = _stamp_frames()
    _check_stream(emul, fr, None, [1, 50])


def test_first_message_across_calls_reset_and_mid_stream(emul):
    from gr_air_modes_b200 import decode
    fr = _stamp_frames()[:30]
    o = emul_build.opts(None)
    h = emul.emul_new(15)
    try:
        a, b, c = fr[:10].copy(), fr[10:20].copy(), fr[20:].copy()
        b["ref_level"][0] = c["ref_level"][0] = np.float32(9.999999)
        # unqueued frames before the first queued one leave the flag for it
        a["passed"][:3] = 0
        recs, text = _run(emul, h, a, o)
        assert text == rc.expected_text(a, recs, True)
        recs, text = _run(emul, h, b, o)
        assert text == rc.expected_text(b, recs, False) and text != rc.expected_text(b, recs, True)
        emul.emul_reset(h)
        assert emul.emul_reports_state(h) & 4
        recs, text = _run(emul, h, b, o)
        assert text == rc.expected_text(b, recs, True)
        # off and on again: the count goes on
        _run(emul, h, a, o, reports=0)
        recs, text = _run(emul, h, c, o)
        assert text == rc.expected_text(c, recs, False)
    finally:
        emul.emul_free(h)
    # turned on mid-stream: its first call's first queued frame is the first
    h = emul.emul_new(15)
    try:
        _run(emul, h, a, o, reports=0)
        assert emul.emul_reports_state(h) == 0                    # nothing allocated while off
        recs, text = _run(emul, h, c, o)
        assert text == rc.expected_text(c, recs, True)
        assert decode.FS_NOT_QUEUED == 0x80
    finally:
        emul.emul_free(h)


def test_a_call_of_the_longest_lines(emul):
    from gr_air_modes_b200 import report
    fr = _tcas_frames(300)
    h = emul.emul_new(15)
    try:
        recs, text = _run(emul, h, fr, emul_build.opts(None))
        assert text == rc.expected_text(fr, recs, True)
        lines = text.split(b"\n")[:-1]
        assert len(lines) == 300 and min(map(len, lines)) > 400, len(lines[0])
        assert " (multiple threats) (resolved) at " in report.format_report(rc.slicer_text(fr[1], False), recs[1])
    finally:
        emul.emul_free(h)


def test_launch_count_and_no_allocation_while_off(emul):
    fr = _small(_scenes()[0][0])[:300]
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(fr), dtype=decode.FIELDS_DTYPE)
    for stages, coverage in ((dict(), 0), (dict(local_cpr=10, commb=30), 1), (dict(sbs1=1, track=60, opstatus=30), 1)):
        o = emul_build.opts((37.4, -122.1), **stages)
        counts = []
        for on in (0, 1):
            h = emul.emul_new(17)
            try:
                emul.emul_set_reports(h, on)
                emul.emul_set_coverage(h, coverage)
                k0 = emul.simt_launch_count()
                assert emul.emul_decode(h, C.c_void_p(fr.ctypes.data), len(fr), o, C.c_void_p(recs.ctypes.data)) == 0
                counts.append(emul.simt_launch_count() - k0)
                assert (emul.emul_reports_state(h) != 0) == bool(on)
            finally:
                emul.emul_free(h)
        assert counts[1] == counts[0] + 3, (stages, coverage, counts)


def _check_option_scenes(e):
    """Every op-status and Comm-B scene with its option on, in one call and cut in three; returns the OPTION_LINE_KINDS
    their texts hold."""
    kinds = set()
    for name, fr, stages in rc.text_option_scenes(small=True):
        o = emul_build.opts(None, **stages)
        n = len(fr)
        for cuts in ([], sorted({n // 3, min(n, n // 3 + 33)} - {0, n})):
            h = e.emul_new(17)
            try:
                first = True
                for a, b in zip([0] + cuts, cuts + [n]):
                    part = np.ascontiguousarray(fr[a:b])
                    recs, text = _run(e, h, part, o)
                    assert text == rc.expected_text(part, recs, first), (name, a, b)
                    first = first and not np.any((recs["status"] & 0x80) == 0)
                    kinds |= rc.line_kinds(text)
            finally:
                e.emul_free(h)
    return kinds


def test_op_status_and_comm_b_lines(emul):
    """The lines options opstatus and commb add: every scene of their case generators, byte for byte, and every kind of
    line among them (BDS4,0 / 5,0 / 6,0; BDS6,5 airborne and surface, version 0 and later; BDS6,2 with and without each
    optional part)."""
    kinds = _check_option_scenes(emul)
    assert kinds >= rc.OPTION_LINE_KINDS, rc.OPTION_LINE_KINDS - kinds


MUTANTS = [
    ("gr_air_modes_b200/csrc/amb_sbs1_format.h", "if (rem > half || (rem == half && (q & 1))) q++;",
     "if (rem >= half) q++;"),
    ("gr_air_modes_b200/csrc/amb_report_format.h", ": amb_rep_roundtrip(frac, 10, &e10);", ": frac;"),
    ("gr_air_modes_b200/csrc/amb_report_format.h", "amb_rep_roundtrip((double)level, first ? 6 : 10, &e10)",
     "amb_rep_roundtrip((double)level, 10, &e10)"),
    ("gr_air_modes_b200/csrc/amb_decode_reports.cuh", "(amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb, b->boff);",
     "(amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb - 1, b->boff); b->boff[nb] = b->boff[nb - 1];"),
    ("gr_air_modes_b200/csrc/amb_report_format.h", 'p = amb_sbs1_str(p, " NICbaro "); p = amb_sbs1_u64(p, b[9]);',
     'p = amb_sbs1_str(p, " NICbaro "); p = amb_sbs1_u64(p, b[10]);'),
    ("gr_air_modes_b200/csrc/amb_report_format.h", "800.0 + ((int)w1 - 1) * 0.8", "800.0 + (int)w1 * 0.8"),
    ("gr_air_modes_b200/csrc/amb_report_format.h", "if (!(modes & mbit[i]) || (i < 5 && !(modes & 0x80))) continue;",
     "if (!(modes & mbit[i])) continue;"),
    ("gr_air_modes_b200/csrc/amb_report_format.h", "raw * (2.048 / 512) + 0.0, 3", "raw * (2.0 / 512) + 0.0, 3"),
]


@pytest.mark.parametrize("which", range(len(MUTANTS)))
def test_mutants_fail(tmp_path, tmp_path_factory, which):
    rel, old, new = MUTANTS[which]
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        import shutil
        shutil.copytree(os.path.join(emul_build.ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1, old
    p.write_text(src.replace(old, new))
    e = _bind(tmp_path_factory, tmp_path / HARNESS)
    fr, loc = _scenes()[0]
    with pytest.raises(AssertionError):
        _check_stream(e, _stamp_frames(), None, [])
        _check_stream(e, _small(fr)[:300], loc, [])
        _check_option_scenes(e)
