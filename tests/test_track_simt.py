"""The aircraft table's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_track.cuh, enqueued by the decoder's own
amb_decode_launch after the fields, pairing, resolve, local CPR and Comm-B kernels, and read out by its snapshot
launchers) on the host under the SIMT emulator (tests/simt/simt_emul.h), against the sequential checker
(tests/track_oracle.py) fed with the same records: after every batch and at the end, in several batch splits (single
messages, cuts at 31/32/33 inside a 32-record step, random sizes), for aircraft that fall silent and come back, a bucket
of 32 aircraft and one address with far more than 32 records in a row. A copy of the walk that skips the expiry test
must fail."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
WORDS = 1024                    # bitmap words the snapshot scans: addresses below 2^15, like the emulated tables

import emul_build  # noqa: E402
import local_cpr_cases as lc  # noqa: E402
import track_cases as tc  # noqa: E402
import track_oracle as to  # noqa: E402


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return emul_build.decode_emul(tmp_path_factory)


def _snapshot(e, h, now):
    from gr_air_modes_b200 import decode
    n = e.emul_snapshot(h, math.nan if now is None else now, WORDS, None, None, 0)
    assert n >= 0
    out = np.zeros(n, dtype=decode.AIRCRAFT_DTYPE)
    if n:
        assert e.emul_snapshot(h, math.nan if now is None else now, WORDS, C.c_void_p(out.ctypes.data), None,
                               n - 1) == -5
        assert e.emul_snapshot(h, math.nan if now is None else now, WORDS, C.c_void_p(out.ctypes.data), None, n) == n
    return out


def _run(e, msgs, loc, S, splits, local_S=0, each=False, commb_S=0):
    """Decode in batches cut at `splits` with the table on; compare with the checker after every batch (each=True) and
    at the end (now = the latest record, the middle of the stream, and just past the end). Returns the final snapshot."""
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(msgs)
    n = len(frames)
    h = e.emul_new(17)
    assert h
    emul_build.opts(e, h, loc, local_cpr=local_S, commb=commb_S, track=S)
    tr = to.Tracker(S)
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        assert e.emul_decode(h, C.c_void_p(frames.ctypes.data + 80 * pos), c,
                             C.c_void_p(recs.ctypes.data + 144 * pos)) == 0
        tr.feed(frames[pos:pos + c], recs[pos:pos + c])
        if each:
            to.assert_rows_equal(_snapshot(e, h, None), tr.snapshot_array(), ("batch at", pos))
        pos += c
    ts = to.t_of(frames)
    final = _snapshot(e, h, None)
    to.assert_rows_equal(final, tr.snapshot_array(), "end")
    for now in (ts[n // 2], ts[-1] + S / 2):
        to.assert_rows_equal(_snapshot(e, h, now), tr.snapshot_array(now), ("now", now))
    e.emul_reset(h)
    assert e.emul_snapshot(h, math.nan, WORDS, None, None, 0) == 0
    assert e.emul_snapshot(h, ts[-1], WORDS, None, None, 0) == 0
    e.emul_free(h)
    return final, recs


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


@pytest.mark.parametrize("seed,commb_S", [(1, 0), (2, 0), (1, 30), (2, 30)], ids=["1", "2", "1+commb", "2+commb"])
def test_life_scene_in_batch_splits(emul, seed, commb_S):
    """Alone, and with the Comm-B stage also on (+commb), as amb_decode_frames runs them."""
    msgs = tc.life_scene(seed=seed)
    loc = [51.5, -0.2] if seed == 1 else None
    finals = []
    for splits in SPLITS:
        final, _ = _run(emul, msgs, loc, 20, splits, each=bool(splits), commb_S=commb_S)
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


def test_a_walk_without_the_expiry_test_is_caught(tmp_path, tmp_path_factory):
    """Mutation: a row never expires, so a record after a silence keeps the old row instead of starting a new one (or
    of being ignored)."""
    e = emul_build.mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_track.cuh",
                          "const bool alive = live && !(t - seen > (double)max_age);", "const bool alive = live;")
    with pytest.raises(AssertionError):
        _run(e, tc.burst_scene(), None, 3, [])
