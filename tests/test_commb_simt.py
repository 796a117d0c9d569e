"""The Comm-B stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_commb.cuh, launched by its own launcher after the
fields, pairing, resolve and local CPR kernels) on the host under the SIMT emulator (tests/simt/simt_emul.h), against
the sequential checker (tests/commb_oracle.py) fed with the same frames and the option-off records: byte for byte,
in several batch splits (single messages, cuts at 31/32/33 inside a 32-record step, random sizes). Two mutants must
fail: a walk whose lanes read the table instead of an earlier same-address lane, and an age test with < for <=."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas", "-shared", "-fPIC"]

import commb_cases as cc  # noqa: E402
import commb_oracle as co  # noqa: E402
import track_cases as tc  # noqa: E402


def _bind(path):
    e = C.CDLL(path)
    e.emul_commb_new.restype = C.c_void_p
    e.emul_commb_new.argtypes = [C.c_int]
    e.emul_commb_free.argtypes = [C.c_void_p]
    e.emul_commb_reset.argtypes = [C.c_void_p]
    e.emul_decode_commb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int,
                                    C.c_void_p]
    return e


def _build(src, out):
    subprocess.run(FLAGS + ["-o", out, src], check=True)
    return _bind(out)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    d = tmp_path_factory.mktemp("simt_commb")
    return _build(os.path.join(ROOT, "tests", "simt", "decode_commb_emul.cc"), str(d / "libdecode_commb_emul.so"))


def _decode(e, frames, S, splits, local_S=0):
    """Records of the emulated decode cut at `splits` (S = 0: the option off)."""
    from gr_air_modes_b200 import decode
    n = len(frames)
    h = e.emul_commb_new(17)
    assert h
    recs = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    pos = 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        assert e.emul_decode_commb(h, C.c_void_p(frames.ctypes.data + 80 * pos), c, 0, 0.0, 0.0, local_S, S,
                                   C.c_void_p(recs.ctypes.data + 144 * pos)) == 0
        pos += c
    e.emul_commb_free(h)
    return recs


def _check(e, msgs, S, splits, local_S=0):
    frames = tc.frames_of(msgs)
    off = _decode(e, frames, 0, [], local_S)
    got = _decode(e, frames, S, splits, local_S)
    co.assert_records_equal(got, co.replay(frames, off, S), ("splits", len(splits)))
    return got


SPLITS = ([], [1] * 40 + [31, 32, 33, 31, 65])


@pytest.mark.parametrize("name", ["unique", "reference", "limits", "burst"])
def test_scene_in_batch_splits(emul, name):
    msgs, S = next((m, s) for nm, m, s in cc.scenes() if nm == name)
    outs = [_check(emul, msgs, S, splits) for splits in SPLITS]
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


def _mutant(tmp_path, rel, old, new):
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    assert src.count(old) == 1
    p.write_text(src.replace(old, new))
    return _build(str(tmp_path / "tests/simt/decode_commb_emul.cc"), str(tmp_path / "libbroken.so"))


def test_a_walk_reading_the_table_instead_of_an_earlier_lane_is_caught(tmp_path):
    """Mutation: a record whose velocity came earlier in the same 32-record step reads the table, which holds the
    velocity of an earlier step (or none)."""
    e = _mutant(tmp_path, "gr_air_modes_b200/csrc/amb_decode_commb.cuh", "            if (!before) {",
                "            if (true) {")
    with pytest.raises(AssertionError):
        _check(e, cc.burst_scene(), 3, [])


def test_an_age_test_with_less_than_is_caught(tmp_path):
    """Mutation: a reference exactly S seconds old no longer counts."""
    e = _mutant(tmp_path, "gr_air_modes_b200/csrc/amb_decode_core.h", "t - ref->t <= (double)max_age",
                "t - ref->t < (double)max_age")
    with pytest.raises(AssertionError):
        _check(e, cc.reference_scene(S=30), 30, [])
