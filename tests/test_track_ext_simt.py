"""The aircraft table extension's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_track_ext.cuh, enqueued by the
decoder's own amb_decode_launch after the track stage, and read out by amb_snap_count / amb_snap_scan /
amb_snap_gather_ext) on the host under the SIMT emulator (tests/simt/simt_emul.h), through
tests/simt/decode_track_ext_emul.cc - the op-status harness plus this option - against the sequential checker
(tests/track_ext_oracle.py) fed with the same frames and the decoder's own records: snapshots byte for byte after every
batch and at the end, in several batch splits (single messages, cuts at 31/32/33 inside a 32-record step, random sizes),
with the local CPR stage on and off. Three mutants must fail: a walk that keeps the first writer of a group instead of
the last, a snapshot without the first_seen test, and a reset that leaves groups visible."""
import ctypes as C
import math
import os
import shutil
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
import track_ext_oracle as xo  # noqa: E402

ROOT = emul_build.ROOT
HARNESS = os.path.join(ROOT, "tests", "simt", "decode_track_ext_emul.cc")
OPSTATUS_S, COMMB_S = 30, 30


def _bind(e):
    e.emul_decode_ext.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int,
                                  C.c_int, C.c_int, C.c_int, C.c_void_p]
    e.emul_snapshot_ext.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_int]
    e.emul_reset_ext.argtypes = [C.c_void_p]
    e.emul_free_ext.argtypes = [C.c_void_p]
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(emul_build.decode_emul(tmp_path_factory, HARNESS))


def _words(frames):
    """Bitmap words the snapshot scans: every DF17 address of the scene (a multiple of 1024 words)."""
    df17 = frames["data"][:, 0] >> 3 == 17
    a = frames["data"][df17][:, 1:4].astype(np.int64)
    top = int(((a[:, 0] << 16) | (a[:, 1] << 8) | a[:, 2]).max()) if len(a) else 0
    return (top // 32 // 1024 + 1) * 1024


def _snapshot(e, h, now, S, S2, words):
    from gr_air_modes_b200 import decode
    now = math.nan if now is None else now
    n = e.emul_snapshot_ext(h, now, S, S2, words, None, None, 0)
    assert n >= 0
    out = np.zeros(n, dtype=decode.AIRCRAFT_DTYPE)
    ext = np.zeros(n, dtype=decode.AIRCRAFT_EXT_DTYPE)
    if n:
        assert e.emul_snapshot_ext(h, now, S, S2, words, C.c_void_p(out.ctypes.data), C.c_void_p(ext.ctypes.data),
                                   n - 1) == -5
        assert not ext.view(np.uint8).any()
        assert e.emul_snapshot_ext(h, now, S, S2, words, C.c_void_p(out.ctypes.data), C.c_void_p(ext.ctypes.data),
                                   n) == n
    return out, ext


def _decode(e, h, frames, local_S, S, S2, recs):
    assert e.emul_decode_ext(h, C.c_void_p(frames.ctypes.data), len(frames), 0, 0.0, 0.0, local_S, COMMB_S, OPSTATUS_S,
                             S, S2, C.c_void_p(recs.ctypes.data)) == 0


def _run(e, msgs, S, S2, splits, local_S=0, each=False):
    """Decode in batches cut at `splits` with every option on; compare with the checker after every batch (each=True)
    and at the end (now = the latest record, the middle of the stream and just past the end). Returns the
    final snapshot."""
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(msgs)
    words = _words(frames)
    n = len(frames)
    h = e.emul_new(17)
    assert h
    chk = xo.ExtTracker(S, S2)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        recs = np.zeros(c, dtype=decode.FIELDS_DTYPE)
        _decode(e, h, frames[pos:pos + c], local_S, S, S2, recs)
        chk.feed(frames[pos:pos + c], recs)
        if each:
            xo.assert_snapshots_equal(_snapshot(e, h, None, S, S2, words), chk.snapshot_arrays(), ("batch at", pos))
        pos += c
    ts = [float(s) + float(f) for s, f in zip(frames["secs"], frames["frac"])]
    final = _snapshot(e, h, None, S, S2, words)
    xo.assert_snapshots_equal(final, chk.snapshot_arrays(), "end")
    for now in (ts[n // 2], ts[-1] + S2 / 2):
        xo.assert_snapshots_equal(_snapshot(e, h, now, S, S2, words), chk.snapshot_arrays(now), ("now", now))
    e.emul_free_ext(h)
    return final


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])
SCENES = [nm for nm, _, _, _ in xc.scenes()]


@pytest.mark.parametrize("local_S", [0, 10], ids=["", "local_cpr"])
@pytest.mark.parametrize("name", SCENES)
def test_scene_in_batch_splits(emul, name, local_S):
    """Every scene cut into single messages and at 31/32/33, checked after every batch; without local CPR also in one
    call, which must give the same final snapshot."""
    msgs, S, S2 = next((m, s, s2) for nm, m, s, s2 in xc.scenes() if nm == name)
    finals = [_run(emul, msgs, S, S2, splits, local_S, each=bool(splits)) for splits in SPLITS[1 if local_S else 0:]]
    for a, b in zip(finals[0], finals[-1]):
        assert a.tobytes() == b.tobytes()
    rows, ext = finals[0]
    assert len(rows)
    if name in ("absence", "bucket", "opstatus_table"):
        assert np.any(ext["shown"] & AXG_INTEG)
    if name in ("absence", "bucket", "burst"):
        assert np.any(ext["shown"] & AXG_COMMB)


AXG_INTEG, AXG_COMMB = 1 << xo.INTEG, (1 << xo.B40) | (1 << xo.B50) | (1 << xo.B60)


def test_random_batch_sizes(emul):
    rng = np.random.default_rng(5)
    _run(emul, xc.bucket_scene(), 30, 2, [int(x) for x in rng.integers(1, 70, 40)], each=True)
    _run(emul, xc.absence_scene(), 10, 60, [int(x) for x in rng.integers(1, 20, 30)], local_S=10, each=True)


def test_one_address_with_many_writers_in_a_step(emul):
    msgs = xc.burst_scene()
    rows, ext = _run(emul, msgs, 20, 600 // 10, [2, 31, 1, 32, 33], each=True)
    assert len(rows) == 1 and ext["shown"][0] == 0x3F


def test_groups_written_while_the_row_was_absent_stay_hidden(emul):
    msgs = xc.absence_scene(S=10)
    rows, ext = _run(emul, msgs, 10, 600, [])
    assert len(rows) == 3
    # the second aircraft got no Comm-B after its row was created again: its B40..B60 groups are hidden
    assert ext["shown"][1] & 0x38 == 0 and ext["shown"][0] & 0x38 != 0
    assert np.all(ext["t"][:, 0] >= rows["first_seen"])


def test_a_group_exactly_S2_old_is_shown_and_one_2_to_the_minus_40_older_is_not(emul):
    now = 100.5
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(xc.age_edge(S2=30, now=now), unqueued_every=0)
    h = emul.emul_new(17)
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    _decode(emul, h, frames, 0, 60, 30, recs)
    rows, ext = _snapshot(emul, h, now, 60, 30, 1024)
    emul.emul_free_ext(h)
    xo.assert_snapshots_equal((rows, ext), xo.replay(frames, recs, 60, 30, now), "age edge")
    assert len(rows) == 1
    assert ext["shown"][0] & 0x01 and ext["t"][0][0] == now - 30            # OPS: exactly S2 old
    assert not ext["shown"][0] & 0x02 and math.isnan(ext["t"][0][1])       # TS: 2^-40 s older
    assert ext["t"][0][xo.INTEG] == rows["pos_t"][0]


def _reset_run(e, S=60, S2=600):
    """Stream A, a reset, then stream B with earlier timestamps on the same addresses that writes fewer groups; the
    snapshots after the reset must equal those of a checker that starts over."""
    from gr_air_modes_b200 import decode
    rng = np.random.default_rng(11)
    a_ev, b_ev = [], []
    for j, aa in enumerate((0x1300, 0x1301)):
        e_, _ = xc.life(aa, 1000.0 + j, rng, n=18)
        a_ev += e_
        for k in range(6):                                  # B: positions only, earlier than all of A
            b_ev.append((990.0 + j + 0.1 * k, *tc.position(aa, 47.0, 8.0, k % 2, False)))
    fa, fb = tc.frames_of(xc._msgs(a_ev), unqueued_every=0), tc.frames_of(xc._msgs(b_ev), unqueued_every=0)
    h = e.emul_new(17)
    chk = xo.ExtTracker(S, S2)
    for fr, reset in ((fa, False), (fb, True)):
        if reset:
            e.emul_reset_ext(h)
            chk.reset()
            assert e.emul_snapshot_ext(h, math.nan, S, S2, 1024, None, None, 0) == 0
        recs = np.zeros(len(fr), dtype=decode.FIELDS_DTYPE)
        _decode(e, h, fr, 0, S, S2, recs)
        chk.feed(fr, recs)
    for now in (None, 1003.0, 1010.0):                      # at 1003 and 1010 stream A's groups would be in range
        got = _snapshot(e, h, now, S, S2, 1024)
        xo.assert_snapshots_equal(got, chk.snapshot_arrays(now), ("after reset", now))
        assert len(got[0]) == 2 and not np.any(got[1]["shown"].astype(int) & ~AXG_INTEG)
    e.emul_free_ext(h)


def test_reset_forgets_every_group(emul):
    _reset_run(emul)


def _mutant(tmp_path, tmp_path_factory, rel, old, new):
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1
    p.write_text(src.replace(old, new))
    return _bind(emul_build.decode_emul(tmp_path_factory, tmp_path / "tests/simt/decode_track_ext_emul.cc"))


def test_a_walk_keeping_the_first_writer_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_track_ext.cuh",
                "if (g == q && (int)lane == 31 - __clz(w)) last = true;",
                "if (g == q && (int)lane == __ffs(w) - 1) last = true;")
    with pytest.raises(AssertionError):
        _run(e, xc.burst_scene(), 20, 60, [])


def test_a_snapshot_without_the_first_seen_test_is_caught(tmp_path, tmp_path_factory):
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_track_ext.cuh",
                "if (t >= first && t <= now", "if (t == t && t <= now")
    with pytest.raises(AssertionError):
        _run(e, xc.absence_scene(S=10), 10, 600, [])


def test_a_reset_leaving_groups_visible_is_caught(tmp_path, tmp_path_factory):
    """Mutation: a row written for the first time since reset keeps the times of the groups this step does not
    write, so stream A's groups show after the reset."""
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_track_ext.cuh",
                "if (!((wrote >> q) & 1u)) row->t[q] = NAN;", "(void)wrote;")
    with pytest.raises(AssertionError):
        _reset_run(e)
