"""DF17 correction by at most M bits anywhere (option "ec_any") through the real C ABI of the EMULATED library
(tests/simt/library_emul.cc, the same recipe as tests/test_ec_simt.py): the split-form slicer on constructed packets and
the fused chain on a small IQ scene, against the oracle plus the brute-force checkers."""
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import ec_any_cases as eac  # noqa: E402
import ec_any_oracle as ea  # noqa: E402
import ec_cases as ecc  # noqa: E402
import ec_oracle as eo  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library(tmp_path_factory):
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


@pytest.mark.parametrize("k,m", [(0, 1), (0, 2), (ecc.K, 2)])
def test_split_form_slicer(port, k, m):
    statuses = eac.run_slicer_packets(port, k, m)
    anys = [s[1] for s in statuses]
    assert anys.count(ea.EC_FIXED) >= (5 if m == 1 else 14), statuses
    assert ea.EC_NO_SOLUTION in anys and ea.EC_NOT_TRIED in anys
    if k:
        for s in (eo.EC_FIXED, eo.EC_TOO_MANY, eo.EC_NO_SOLUTION):
            assert s in [s[0] for s in statuses]


RATE, N, NB = 4e6, 60_000, 12


@pytest.fixture(scope="module")
def scene():
    return eac.any_scene(RATE, N, NB, seed=11)


def test_fused_chain_one_shot_and_chunked(port, scene):
    iq, _ = scene
    msgs, frames, st = eac.run_chain(iq, RATE, 0, eac.M)
    _, statuses = eac.check_chain(port, iq, RATE, frames, msgs, 0, eac.M)
    fixed = eac.n_fixed(statuses)
    assert fixed >= 6 and st.ec_fixed == fixed
    assert st.frames_passed == sum(f.passed for f in frames)
    assert [f for f in frames if f.passed][0].ec_any == ea.EC_FIXED
    rng = np.random.default_rng(5)
    for resolver in (0, 1):
        chunks = [int(x) for x in rng.integers(1, N // 3, 3)] + [1, 511, 513]
        msgs2, frames2, _ = eac.run_chain(iq, RATE, 0, eac.M, chunks=chunks, resolver=resolver)
        assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def test_both_options_on(port):
    iq, _ = eac.any_scene(RATE, N, NB, seed=12, wrong_max=2)
    msgs, frames, st = eac.run_chain(iq, RATE, ecc.K, eac.M)
    _, statuses = eac.check_chain(port, iq, RATE, frames, msgs, ecc.K, eac.M)
    assert st.ec_fixed == eac.n_fixed(statuses)
    assert any(s[0] == eo.EC_FIXED for s in statuses) and any(s[1] == ea.EC_FIXED for s in statuses)


def test_off_is_byte_identical_to_never_set(scene):
    iq, _ = scene
    msgs0, frames0, st0 = eac.run_chain(iq, RATE, 0, 0)
    msgs1, frames1, st1 = eac.run_chain(iq, RATE, 0, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert all(bytes(f.pad_) == b"\0" * 6 for f in frames0) and st0.ec_fixed == 0
    assert st1.kernel_launches == st0.kernel_launches
    _, _, st_on = eac.run_chain(iq, RATE, 0, 1)
    assert st_on.kernel_launches == st0.kernel_launches + 1          # one call: one more launch
    _, _, st_both = eac.run_chain(iq, RATE, ecc.K, 2)
    assert st_both.kernel_launches == st0.kernel_launches + 1        # both passes share it


def test_option_range_and_persistence(port, scene):
    iq, _ = scene
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True)
    for bad in (-1, 3, 24):
        with pytest.raises(RuntimeError):
            rx.set_ec_any(bad)
    with pytest.raises(RuntimeError):
        rx.set_option("ec_any", 3)
    assert rx.get_ec_any() == 0
    rx.set_option("ec_any", eac.M)
    rx.reset()
    rx.set_rate(RATE)                                                 # a new stream; the option stays
    rx.process(iq, flush=True)
    eac.check_chain(port, iq, RATE, rx.frames, q.strings(), 0, eac.M)
    assert rx.get_ec_any() == eac.M
    rx.close()
