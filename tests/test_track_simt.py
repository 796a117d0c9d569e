"""The aircraft table's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_track.cuh, launched by its own launchers after the
fields, pairing, resolve and local CPR kernels) on the host under the SIMT emulator (tests/simt/simt_emul.h), against
the sequential checker (tests/track_oracle.py) fed with the same records: after every batch and at the end, in several
batch splits (single messages, cuts at 31/32/33 inside a 32-record step, random sizes), for aircraft that fall silent
and come back, a bucket of 32 aircraft and one address with far more than 32 records in a row. A copy of the walk that
skips the expiry test must fail."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas", "-shared", "-fPIC"]
WORDS = 1024                    # bitmap words the snapshot scans: addresses below 2^15, like the emulated tables

import local_cpr_cases as lc  # noqa: E402
import track_cases as tc  # noqa: E402
import track_oracle as to  # noqa: E402


def _bind(path):
    e = C.CDLL(path)
    e.emul_track_new.restype = C.c_void_p
    e.emul_track_new.argtypes = [C.c_int]
    e.emul_track_free.argtypes = [C.c_void_p]
    e.emul_track_reset.argtypes = [C.c_void_p]
    e.emul_decode_track.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int,
                                    C.c_void_p]
    e.emul_track_snapshot.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_uint, C.c_void_p, C.c_int]
    return e


def _build(src, out):
    subprocess.run(FLAGS + ["-o", out, src], check=True)
    return _bind(out)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    d = tmp_path_factory.mktemp("simt_track")
    return _build(os.path.join(ROOT, "tests", "simt", "decode_track_emul.cc"), str(d / "libdecode_track_emul.so"))


def _snapshot(e, h, now, S):
    from gr_air_modes_b200 import decode
    n = e.emul_track_snapshot(h, math.nan if now is None else now, S, WORDS, None, 0)
    assert n >= 0
    out = np.zeros(n, dtype=decode.AIRCRAFT_DTYPE)
    if n:
        assert e.emul_track_snapshot(h, math.nan if now is None else now, S, WORDS, C.c_void_p(out.ctypes.data), n - 1) == -5
        assert e.emul_track_snapshot(h, math.nan if now is None else now, S, WORDS, C.c_void_p(out.ctypes.data), n) == n
    return out


def _run(e, msgs, loc, S, splits, local_S=0, each=False):
    """Decode in batches cut at `splits` with the table on; compare with the checker after every batch (each=True) and
    at the end (now = the latest record, the middle of the stream, and just past the end). Returns the final snapshot."""
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(msgs)
    n = len(frames)
    have, lat, lon = (0, 0.0, 0.0) if loc is None else (1, loc[0], loc[1])
    h = e.emul_track_new(17)
    assert h
    tr = to.Tracker(S)
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        assert e.emul_decode_track(h, C.c_void_p(frames.ctypes.data + 80 * pos), c, have, lat, lon, local_S, S,
                                   C.c_void_p(recs.ctypes.data + 144 * pos)) == 0
        tr.feed(frames[pos:pos + c], recs[pos:pos + c])
        if each:
            to.assert_rows_equal(_snapshot(e, h, None, S), tr.snapshot_array(), ("batch at", pos))
        pos += c
    ts = to.t_of(frames)
    final = _snapshot(e, h, None, S)
    to.assert_rows_equal(final, tr.snapshot_array(), "end")
    for now in (ts[n // 2], ts[-1] + S / 2):
        to.assert_rows_equal(_snapshot(e, h, now, S), tr.snapshot_array(now), ("now", now))
    e.emul_track_reset(h)
    assert e.emul_track_snapshot(h, math.nan, S, WORDS, None, 0) == 0
    assert e.emul_track_snapshot(h, ts[-1], S, WORDS, None, 0) == 0
    e.emul_track_free(h)
    return final, recs


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


@pytest.mark.parametrize("seed", [1, 2])
def test_life_scene_in_batch_splits(emul, seed):
    msgs = tc.life_scene(seed=seed)
    loc = [51.5, -0.2] if seed == 1 else None
    finals = []
    for splits in SPLITS:
        final, _ = _run(emul, msgs, loc, 20, splits, each=bool(splits))
        finals.append(final)
    to.assert_rows_equal(finals[0], finals[1], "splits")
    assert len(finals[0]) >= 4
    fl = finals[0]["flags"]
    for f in (to.AC_HAS_ALT, to.AC_HAS_SQUAWK, to.AC_HAS_IDENT, to.AC_HAS_POS, to.AC_HAS_VELOCITY, to.AC_HAS_HEADING):
        assert np.any(fl & f), f


def test_silence_and_a_reply_do_not_revive(emul):
    """The checker's own account of the scene: rows recreated after a silence start over; replies to unknown addresses
    never make a row."""
    msgs = tc.life_scene(seed=1)
    frames = tc.frames_of(msgs)
    _, recs = _run(emul, msgs, None, 20, [])
    tr = to.Tracker(20)
    tr.feed(frames, recs)
    assert not any(0x6000 <= a < 0x6008 for a in tr.rows)
    ts = to.t_of(frames)
    firsts = {a: r["first_seen"] for a, r in tr.rows.items()}
    assert any(firsts[a] > ts[0] + 20 for a in firsts)         # a row created anew after a silence


def test_random_batch_sizes(emul):
    msgs, _ = lc.trajectory_scene(3, n_aircraft=12, seconds=120.0, drop=0.5, small_addresses=True)
    rng = np.random.default_rng(5)
    splits = [int(x) for x in rng.integers(1, 200, 40)]
    for local_S in (0, 30):
        _run(emul, msgs, [48.0, 11.0], 10, splits, local_S=local_S, each=True)


def test_a_bucket_of_32_aircraft(emul):
    msgs = tc.bucket_scene()
    for splits in ([], [33, 1, 31, 32, 700]):
        final, _ = _run(emul, msgs, [10.0, 20.0], 30, splits)
    assert len(final) == 32


def test_one_address_with_long_runs_in_a_step(emul):
    msgs = tc.burst_scene()
    for splits in ([], [2, 31, 1, 32, 33]):
        _run(emul, msgs, None, 3, splits, each=True)


def test_a_walk_without_the_expiry_test_is_caught(tmp_path):
    """Mutation: a row never expires, so a record after a silence keeps the old row instead of starting a new one (or
    of being ignored)."""
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / "gr_air_modes_b200/csrc/amb_decode_track.cuh"
    src = p.read_text()
    a = "const bool alive = live && !(t - seen > (double)max_age);"
    assert src.count(a) == 1
    p.write_text(src.replace(a, "const bool alive = live;"))
    e = _build(str(tmp_path / "tests/simt/decode_track_emul.cc"), str(tmp_path / "libbroken.so"))
    with pytest.raises(AssertionError):
        _run(e, tc.burst_scene(), None, 3, [])
