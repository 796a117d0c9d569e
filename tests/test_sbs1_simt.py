"""The SBS-1 stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_sbs1.cuh, enqueued by the decoder's own
amb_decode_launch after every other stage) on the host under the SIMT emulator (tests/simt/simt_emul.h), through
tests/simt/decode_sbs1_emul.cc - the track-extension harness plus this option - against the sequential checker
(tests/sbs1_oracle.py) fed with the same frames and the decoder's own records: the text byte for byte and every id,
across single messages, cuts at 31/32/33 and random splits, with local_cpr / commb / opstatus / track on and off; the
window crossed across calls, inside one call, in a cascade, and by one call of more than 10000 new addresses; a reset
followed by earlier timestamps. Four mutants must fail: a walk that reads the table instead of the earlier lane, a
plain scan that ignores expiry inside a call, round-half-up formatting and rounded milliseconds."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import sbs1_oracle as so  # noqa: E402
import track_cases as tc  # noqa: E402

ROOT = emul_build.ROOT
HARNESS = os.path.join(ROOT, "tests", "simt", "decode_sbs1_emul.cc")


def _bind(e):
    e.emul_decode_sbs1.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int,
                                   C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.POINTER(C.c_size_t)]
    e.emul_sbs1_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    e.emul_reset_sbs1.argtypes = [C.c_void_p]
    e.emul_free_sbs1.argtypes = [C.c_void_p]
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(emul_build.decode_emul(tmp_path_factory, HARNESS))


LOC = (47.9, 11.1)                                       # receiver location: surface positions need one


def _call(e, h, frames, opts, tz, chk):
    from gr_air_modes_b200 import decode
    n = len(frames)
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    buf = C.create_string_buffer(max(1, n * 192))
    nb = C.c_size_t()
    local_S, commb_S, opstatus_S, track_S = opts
    assert e.emul_decode_sbs1(h, C.c_void_p(frames.ctypes.data), n, 1, LOC[0], LOC[1], local_S, commb_S, opstatus_S, track_S,
                              20 if track_S else 0, 1, tz, C.c_void_p(recs.ctypes.data), buf, len(buf), C.byref(nb)) == 0
    want_ids = []
    want = chk.feed(frames, recs, want_ids)
    got = buf.raw[: nb.value]
    assert got == want, _first_diff(got, want)
    ids = np.zeros(max(1, n), dtype=np.uint64)
    m = e.emul_sbs1_ids(h, C.c_void_p(recs.ctypes.data), n, C.c_void_p(ids.ctypes.data))
    assert ids[:m].tolist() == want_ids
    return got


def _first_diff(got, want):
    g, w = got.split(b"\r\n"), want.split(b"\r\n")
    for i, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return "line %d: %r != %r" % (i, a, b)
    return "%d lines != %d lines" % (len(g), len(w))


def _run(e, calls, opts=(0, 0, 0, 0), tz=0, resets=()):
    """Decode the frame arrays `calls` one call each; text and ids equal to the checker's after every call."""
    h = e.emul_new(17)
    assert h
    chk = so.Sbs1Checker(tz)
    out = []
    for i, frames in enumerate(calls):
        if i in resets:
            e.emul_reset_sbs1(h)
            chk.reset()
        out.append(_call(e, h, frames, opts, tz, chk))
    e.emul_free_sbs1(h)
    return b"".join(out), chk


def _cut(frames, splits):
    out, pos = [], 0
    for c in list(splits) + [len(frames)]:
        c = min(c, len(frames) - pos)
        if c > 0:
            out.append(frames[pos:pos + c])
            pos += c
    return out


OPTS = [(0, 0, 0, 0), (10, 30, 30, 20)]
SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


@pytest.mark.parametrize("opts", OPTS, ids=["plain", "local_commb_opstatus_track"])
@pytest.mark.parametrize("name", [nm for nm, _ in sc.scenes()])
def test_scene_in_batch_splits(emul, name, opts):
    msgs = next(m for nm, m in sc.scenes() if nm == name)
    frames = tc.frames_of(msgs)
    texts = [_run(emul, _cut(frames, splits), opts)[0] for splits in SPLITS]
    assert texts[0] == texts[1]                          # the text does not depend on the cut


def test_mix_scene_has_every_line_kind_and_a_time_zone(emul):
    frames = tc.frames_of(sc.mix_scene())
    text, _ = _run(emul, [frames], tz=-330)
    kinds = {ln.split(b",")[1] for ln in text.split(b"\r\n") if ln}
    assert kinds == {b"1", b"2", b"3", b"4", b"5", b"6", b"7", b"8"}


def test_random_splits(emul):
    frames = tc.frames_of(sc.mix_scene(seed=8))
    rng = np.random.default_rng(5)
    for _ in range(3):
        splits = [int(x) for x in rng.integers(1, 200, 20)]
        _run(emul, _cut(frames, splits), OPTS[1])


def test_window_across_calls_inside_a_call_and_in_a_cascade(emul):
    calls = [tc.frames_of(m, unqueued_every=0) for m in sc.window_calls()]
    _, chk = _run(emul, calls)
    assert chk.n > 10000 + 3 * 60 + 50                   # every revisit of an expired address took a new id


def test_one_call_with_more_than_10000_new_addresses(emul):
    _, chk = _run(emul, [tc.frames_of(sc.big_call(), unqueued_every=0)])
    assert chk.n > 12000


def test_reset_then_earlier_stamps(emul):
    a = tc.frames_of(sc.mix_scene(seed=4))
    b = tc.frames_of(sc.mix_scene(seed=5))
    b["secs"] -= 3600 * 24 * 400
    text, chk = _run(emul, [a, b, a[:100]], OPTS[1], resets=(1,))
    assert text.count(b"MSG,") > 0


def _mutant(tmp_path, tmp_path_factory, rel, old, new):
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1
    p.write_text(src.replace(old, new))
    return _bind(emul_build.decode_emul(tmp_path_factory, tmp_path / "tests/simt/decode_sbs1_emul.cc"))


def test_a_walk_reading_the_table_instead_of_the_earlier_lane_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_sbs1.cuh",
                "src[k] = before ? (AMB_SBS1_MARK | pk) : slot;", "src[k] = slot; (void)pk;")
    with pytest.raises(AssertionError):
        _run(e, [tc.frames_of(sc.mix_scene())])


def test_a_plain_scan_ignoring_expiry_inside_a_call_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_sbs1.cuh",
                "amb_sbs1_live(g, G0, base) != amb_sbs1_live(g, G0 + AMB_SBS1_CHUNK, base)) s_amb = 1u;",
                "false) s_amb = 1u;")
    with pytest.raises(AssertionError):
        _run(e, [tc.frames_of(m, unqueued_every=0) for m in sc.window_calls()])


def test_round_half_up_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_sbs1_format.h",
                "if (rem > half || (rem == half && (q & 1))) q++;", "if (rem >= half) q++;")
    with pytest.raises(AssertionError):
        _run(e, [tc.frames_of(sc.mix_scene())])


def test_rounded_milliseconds_are_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_sbs1_format.h",
                "double msf = floor(f * 1000.0);", "double msf = rint(f * 1000.0);")
    with pytest.raises(AssertionError):
        _run(e, [tc.frames_of(sc.mix_scene())])
