"""The op-status stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_opstatus.cuh, enqueued by the decoder's own
amb_decode_launch after the Comm-B stage and before the track stage) on the host under the SIMT emulator
(tests/simt/simt_emul.h), through tests/simt/decode_opstatus_emul.cc - the shared decoder harness plus this option -
against the sequential checker (tests/opstatus_oracle.py) fed with the same frames and the option-off records: byte
for byte, in several batch splits (single messages, cuts at 31/32/33 inside a 32-record step, random sizes), alone and with the local CPR, Comm-B and track stages also on. Three mutants must fail: a walk whose
positions read the table instead of an earlier same-address lane, an age test with < for <=, and NIC-C taken from an
airborne writer."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import opstatus_cases as oc  # noqa: E402
import opstatus_oracle as oo  # noqa: E402
import track_cases as tc  # noqa: E402

ROOT = emul_build.ROOT
HARNESS = os.path.join(ROOT, "tests", "simt", "decode_opstatus_emul.cc")


def _bind(e):
    e.emul_decode_all.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int,
                                  C.c_int, C.c_int, C.c_void_p]
    e.emul_free_all.argtypes = [C.c_void_p]
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(emul_build.decode_emul(tmp_path_factory, HARNESS))


def _decode(e, frames, S, splits, others=(0, 0, 0)):
    """Records of the emulated decode cut at `splits` (S = 0: the option off); others = local_cpr, commb, track S."""
    from gr_air_modes_b200 import decode
    local_S, commb_S, track_S = others
    n = len(frames)
    h = e.emul_new(17)
    assert h
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        assert e.emul_decode_all(h, C.c_void_p(frames.ctypes.data + 80 * pos), c, 0, 0.0, 0.0, local_S, commb_S, S,
                                 track_S, C.c_void_p(recs.ctypes.data + 144 * pos)) == 0
        pos += c
    e.emul_free_all(h)
    return recs


def _check(e, msgs, S, splits, others=(0, 0, 0)):
    frames = tc.frames_of(msgs)
    off = _decode(e, frames, 0, [], others)
    got = _decode(e, frames, S, splits, others)
    oo.assert_records_equal(got, oo.replay(frames, off, S), ("splits", len(splits)))
    return got


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])
SCENES = ["table", "fields", "age", "burst"]


@pytest.mark.parametrize("name", SCENES + [nm + "+others" for nm in SCENES])
def test_scene_in_batch_splits(emul, name):
    """Alone, and with every other stage of the decoder on (name + "+others"), as amb_decode_frames runs it."""
    name, _, others = name.partition("+")
    other_S = (10, 30, 20) if others else (0, 0, 0)
    msgs, S = next((m, s) for nm, m, s in oc.scenes() if nm == name)
    outs = [_check(emul, msgs, S, splits, other_S) for splits in SPLITS]
    assert outs[0].tobytes() == outs[1].tobytes()
    o = oo.outcome_of(outs[0])
    if name == "table":
        assert all(np.any(o == v) for v in (oo.OPSTATUS, oo.NIC, oo.NUC))
    if name == "fields":
        assert all(np.any(o == v) for v in (oo.OPSTATUS, oo.TARGET_STATE, oo.UNSUPPORTED))


def test_random_batch_sizes(emul):
    rng = np.random.default_rng(5)
    _check(emul, oc.age_scene(S=30), 30, [int(x) for x in rng.integers(1, 10, 20)])
    _check(emul, oc.burst_scene(), 3, [int(x) for x in rng.integers(1, 70, 10)], (10, 0, 0))


def test_a_bucket_of_32_aircraft(emul):
    msgs = oc.bucket_scene()
    for splits in ([], [33, 1, 31, 32, 700]):
        got = _check(emul, msgs, 5, splits)
    assert np.sum(oo.outcome_of(got) == oo.NIC) > 300


def _mutant(tmp_path, tmp_path_factory, rel, old, new):
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1
    p.write_text(src.replace(old, new))
    return _bind(emul_build.decode_emul(tmp_path_factory, tmp_path / "tests/simt/decode_opstatus_emul.cc"))


def test_a_walk_reading_the_table_instead_of_an_earlier_lane_is_caught(tmp_path, tmp_path_factory):
    """Mutation: a position whose op status came earlier in the same 32-record step reads the table, which holds the
    op status of an earlier step (or none)."""
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_opstatus.cuh", "if (!before) {",
                "if (true) {")
    with pytest.raises(AssertionError):
        _check(e, oc.burst_scene(), 3, [])


def test_an_age_test_with_less_than_is_caught(tmp_path, tmp_path_factory):
    """Mutation: an op status exactly S seconds old no longer counts."""
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_core.h",
                "t - ref->t_any <= (double)max_age", "t - ref->t_any < (double)max_age")
    with pytest.raises(AssertionError):
        _check(e, oc.age_scene(S=30), 30, [])


def test_nic_c_from_an_airborne_writer_is_caught(tmp_path, tmp_path_factory):
    """Mutation: every op-status writer counts as a surface one, so a surface position takes its NIC-C (0) and age from
    an airborne writer later than the surface one."""
    e = _mutant(tmp_path, tmp_path_factory, "gr_air_modes_b200/csrc/amb_decode_opstatus.cuh",
                "__ballot_sync(0xffffffffu, kind == AMB_ES_KIND_SURF)",
                "__ballot_sync(0xffffffffu, kind == AMB_ES_KIND_SURF || kind == AMB_ES_KIND_AIR)")
    with pytest.raises(AssertionError):
        _check(e, oc.table_scene(), 30, [])
