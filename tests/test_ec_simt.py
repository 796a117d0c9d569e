"""Error correction (option "ec") through the real C ABI of the EMULATED library (tests/simt/library_emul.cc, the same
recipe as tests/test_library_simt.py): the split-form slicer on constructed packets and the fused chain on a small IQ
scene, against the oracle plus the brute-force checker of tests/ec_oracle.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_cases as ecc  # noqa: E402
import ec_oracle as eo  # noqa: E402
from test_ec_cpu import low_weight_codeword  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("libsimt_ec") / "libairmodes_b200_emulated.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-psabi", "-shared", "-fPIC",
                    "-o", out, os.path.join(ROOT, "tests", "simt", "library_emul.cc")], check=True)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


@pytest.fixture(scope="module")
def codewords():
    return {n: low_weight_codeword(n) for n in (56, 112)}


def test_split_form_slicer_every_outcome(port, codewords):
    statuses = ecc.run_slicer_packets(port, codewords)
    for s in (eo.EC_FIXED, eo.EC_TOO_MANY, eo.EC_NO_SOLUTION, eo.EC_AMBIGUOUS, eo.EC_NOT_TRIED):
        assert s in statuses, (s, statuses)
    assert statuses.count(eo.EC_FIXED) >= 7


RATE, N, NB = 4e6, 48_000, 9


@pytest.fixture(scope="module")
def scene():
    return ecc.ec_scene(RATE, N, NB, seed=5)


def test_fused_chain_one_shot_and_chunked(port, scene):
    iq, _ = scene
    msgs, frames, st = ecc.run_chain(iq, RATE, ecc.K)
    _, statuses = ecc.check_chain(port, iq, RATE, frames, msgs, ecc.K)
    fixed = statuses.count(eo.EC_FIXED)
    assert fixed >= 4 and st.ec_fixed == fixed
    assert st.frames_passed == sum(f.passed for f in frames)
    rng = np.random.default_rng(3)
    for resolver in (0, 1):
        chunks = [int(x) for x in rng.integers(1, N // 3, 3)] + [1, 511, 513]
        msgs2, frames2, _ = ecc.run_chain(iq, RATE, ecc.K, chunks=chunks, resolver=resolver)
        assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def test_off_is_byte_identical_to_never_set(scene):
    iq, _ = scene
    msgs0, frames0, st0 = ecc.run_chain(iq, RATE, 0)
    msgs1, frames1, st1 = ecc.run_chain(iq, RATE, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert all(f.ec == 0 and f.ec_flips == 0 for f in frames0) and st0.ec_fixed == 0
    assert st1.kernel_launches == st0.kernel_launches
    _, _, st_on = ecc.run_chain(iq, RATE, ecc.K)
    assert st_on.kernel_launches == st0.kernel_launches + 1          # one call: one more launch


def test_option_range_and_persistence(port, scene):
    iq, _ = scene
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True)
    for bad in (-1, 24, 1000):
        with pytest.raises(RuntimeError):
            rx.set_ec(bad)
    assert rx.get_ec() == 0
    rx.set_ec(ecc.K)
    rx.reset()
    rx.set_rate(RATE)                                                 # a new stream; the option stays
    rx.process(iq, flush=True)
    ecc.check_chain(port, iq, RATE, rx.frames, q.strings(), ecc.K)
    assert rx.get_ec() == ecc.K
    rx.close()
