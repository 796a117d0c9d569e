"""The Comm-B stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_commb.cuh, enqueued by the decoder's own
amb_decode_launch after the fields, pairing, resolve and local CPR kernels) on the host under the SIMT emulator
(tests/simt/simt_emul.h), against the sequential checker (tests/commb_oracle.py) fed with the same frames and the
option-off records: byte for byte, in several batch splits (single messages, cuts at 31/32/33 inside a 32-record step,
random sizes), alone and with the local CPR and track stages also on. Two mutants must fail: a walk whose lanes read
the table instead of an earlier same-address lane, and an age test with < for <=."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import commb_cases as cc  # noqa: E402
import commb_oracle as co  # noqa: E402
import emul_build  # noqa: E402
import track_cases as tc  # noqa: E402


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return emul_build.decode_emul(tmp_path_factory)


def _decode(e, frames, S, splits, local_S=0, track_S=0):
    """Records of the emulated decode cut at `splits` (S = 0: the option off)."""
    from gr_air_modes_b200 import decode
    n = len(frames)
    h = e.emul_new(17)
    assert h
    emul_build.opts(e, h, local_cpr=local_S, commb=S, track=track_S)
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        assert e.emul_decode(h, C.c_void_p(frames.ctypes.data + 80 * pos), c,
                             C.c_void_p(recs.ctypes.data + 144 * pos)) == 0
        pos += c
    e.emul_free(h)
    return recs


def _check(e, msgs, S, splits, local_S=0, track_S=0):
    frames = tc.frames_of(msgs)
    off = _decode(e, frames, 0, [], local_S, track_S)
    got = _decode(e, frames, S, splits, local_S, track_S)
    co.assert_records_equal(got, co.replay(frames, off, S), ("splits", len(splits)))
    return got


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


SCENES = ["unique", "reference", "limits", "burst"]


@pytest.mark.parametrize("name", SCENES + [nm + "+local_cpr+track" for nm in SCENES])
def test_scene_in_batch_splits(emul, name):
    """Alone, and with every other stage of the decoder on (name + "+local_cpr+track"), as amb_decode_frames runs it."""
    name, _, others = name.partition("+")
    local_S, track_S = (10, 20) if others else (0, 0)
    msgs, S = next((m, s) for nm, m, s in cc.scenes() if nm == name)
    outs = [_check(emul, msgs, S, splits, local_S, track_S) for splits in SPLITS]
    assert outs[0].tobytes() == outs[1].tobytes()
    o = co.outcome_of(outs[0])
    assert np.any(o != co.NOT_TRIED)
    if name == "reference":
        assert np.any(o == co.RESOLVED) and np.any(o == co.AMBIGUOUS)
    if name == "unique":
        assert np.any(o == co.DECODED) and np.any(o == co.NONE)


def test_random_batch_sizes(emul):
    msgs = cc.reference_scene(S=30) + []
    rng = np.random.default_rng(5)
    splits = [int(x) for x in rng.integers(1, 40, 40)]
    _check(emul, msgs, 30, splits)
    _check(emul, cc.burst_scene(), 3, [int(x) for x in rng.integers(1, 70, 10)], local_S=10)


def test_a_bucket_of_32_aircraft(emul):
    msgs = cc.bucket_scene()
    for splits in ([], [33, 1, 31, 32, 700]):
        got = _check(emul, msgs, 30, splits)
    assert np.sum(co.outcome_of(got) == co.RESOLVED) > 100


def test_a_walk_reading_the_table_instead_of_an_earlier_lane_is_caught(tmp_path, tmp_path_factory):
    """Mutation: a record whose velocity came earlier in the same 32-record step reads the table, which holds the
    velocity of an earlier step (or none)."""
    e = emul_build.mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_commb.cuh",
                          "            if (!before) {", "            if (true) {")
    with pytest.raises(AssertionError):
        _check(e, cc.burst_scene(), 3, [])


def test_an_age_test_with_less_than_is_caught(tmp_path, tmp_path_factory):
    """Mutation: a reference exactly S seconds old no longer counts."""
    e = emul_build.mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_core.h",
                          "t - ref->t <= (double)max_age", "t - ref->t < (double)max_age")
    with pytest.raises(AssertionError):
        _check(e, cc.reference_scene(S=30), 30, [])
