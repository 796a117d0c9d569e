"""Address/parity check (option "ap_filter") through the real C ABI of the EMULATED library (tests/simt/library_emul.cc,
the same recipe as tests/test_ec_simt.py): the fused chain on small fleet scenes, against the oracle plus the checkers
of tests/ec_oracle.py, tests/ec_any_oracle.py and tests/ap_oracle.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ap_cases as apc  # noqa: E402
import ap_oracle as apo  # noqa: E402
import ec_cases as ecc  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("libsimt_ap") / "libairmodes_b200_emulated.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-psabi", "-shared", "-fPIC",
                    "-o", out, os.path.join(ROOT, "tests", "simt", "library_emul.cc")], check=True)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


RATE, N, S = 4e6, 120_000, 1


@pytest.fixture(scope="module")
def scene():
    return apc.fleet_scene(RATE, N, 6, 60, seed=21, snr_db=(8.0, 30.0))


def test_fused_chain_one_shot_and_chunked(port, scene):
    iq, _ = scene
    msgs, frames, st = apc.run_chain(iq, RATE, S)
    _, statuses = apc.check_chain(port, iq, RATE, frames, msgs, S)
    assert apc.count(statuses, apo.AP_KNOWN) >= 10 and apc.count(statuses, apo.AP_UNKNOWN) >= 3
    assert any(f.ap == apo.AP_KNOWN and f.df == 11 and f.crc for f in frames)          # an accepted II/SI reply
    assert st.frames_passed == sum(f.passed for f in frames)
    # cuts between each known subject and the frame before it
    idx = [int(f.sample_index) for f in frames]
    cuts = sorted({(idx[i - 1] + idx[i]) // 2 for i, f in enumerate(frames) if i and f.ap == apo.AP_KNOWN})[:4]
    chunks = list(np.diff([0] + cuts))
    rng = np.random.default_rng(5)
    for resolver in (0, 1):
        for ch in (chunks, [int(x) for x in rng.integers(1, N // 3, 3)] + [1, 511, 513]):
            msgs2, frames2, _ = apc.run_chain(iq, RATE, S, chunks=[int(c) for c in ch], resolver=resolver)
            assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def test_with_both_corrections(port):
    iq, _ = apc.fleet_scene(RATE, N, 5, 60, seed=22, snr_db=(5.0, 30.0), garble_frac=0.3)
    msgs, frames, _ = apc.run_chain(iq, RATE, S, k=ecc.K, m=2)
    apc.check_chain(port, iq, RATE, frames, msgs, S, k=ecc.K, m=2)


def test_one_address_beyond_the_tile(port):
    """One aircraft, more of its frames in one call than the shared-memory tile holds: the in-place global path."""
    iq, _ = apc.fleet_scene(RATE, 240_000, 1, 440, seed=23, snr_db=(10.0, 30.0))
    msgs, frames, _ = apc.run_chain(iq, RATE, S)
    _, statuses = apc.check_chain(port, iq, RATE, frames, msgs, S)
    assert sum(x[2] != apo.AP_NOT_CHECKED or x[3] == apo.CONF for x in statuses) > 256
    assert apc.count(statuses, apo.AP_KNOWN) > 100


def test_reset_and_set_rate_clear_the_table(port):
    rng = np.random.default_rng(24)
    addrs = [0x4840D6, 0xA1B2C3]
    a = apc.place_scene(RATE, 40_000, [(4000 + 9000 * i, apc.one_frame(17, x, rng)) for i, x in enumerate(addrs)], 1)
    b = apc.place_scene(RATE, 40_000, [(4000 + 9000 * i, apc.one_frame(df, x, rng, code=5 if df == 11 else 0))
                                       for i, (df, x) in enumerate([(4, addrs[0]), (11, addrs[1]), (20, addrs[1])])], 2)
    # one stream: b's replies are known from a's squitters
    msgs, frames, _ = apc.run_chain(np.concatenate([a, b]), RATE, S)
    apc.check_chain(port, np.concatenate([a, b]), RATE, frames, msgs, S)
    assert [f.ap for f in frames] == [0, 0, 1, 1, 1] and sum(f.passed for f in frames) == 5
    for how in ("reset", "set_rate"):
        q = am.msg_queue()
        rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ap_filter=S)
        apc.run_chain(a, RATE, S, rx=rx, q=q, close=False)
        rx.reset() if how == "reset" else rx.set_rate(RATE)
        q2 = am.msg_queue()
        rx._queue = rx._slicer._queue = q2
        rx._slicer._first = True                                       # the message precision rule restarts too
        msgs, frames, _ = apc.run_chain(b, RATE, S, rx=rx, q=q2)
        apc.check_chain(port, b, RATE, frames, msgs, S)
        assert [f.ap for f in frames] == [2, 2, 2] and msgs == [], how
        assert rx.get_ap_filter() == S


def test_off_is_byte_identical_and_launch_count(scene):
    iq, _ = scene
    msgs0, frames0, st0 = apc.run_chain(iq, RATE, 0)
    msgs1, frames1, st1 = apc.run_chain(iq, RATE, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert all(bytes(f.pad_) == b"\0" * 6 for f in frames0)
    assert st1.kernel_launches == st0.kernel_launches
    _, _, st_on = apc.run_chain(iq, RATE, S)
    assert st_on.kernel_launches == st0.kernel_launches + 4            # one call: four more launches


def test_option_range_and_refusals(scene):
    iq, _ = scene
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True)
    for bad in (-1, 3601):
        with pytest.raises(RuntimeError):
            rx.set_ap_filter(bad)
    with pytest.raises(RuntimeError):
        rx.set_option("ap_filter", 3601)
    assert rx.get_ap_filter() == 0
    rx.set_option("ap_filter", 3600)
    with pytest.raises(RuntimeError):
        rx.seek(0, 0)
    with pytest.raises(RuntimeError):
        rx.defer_resolve(True)
    rx.set_ap_filter(0)
    rx.defer_resolve(True)
    with pytest.raises(RuntimeError):
        rx.set_ap_filter(60)
    rx.defer_resolve(False)
    rx.seek(0, 0)
    with pytest.raises(RuntimeError):
        rx.set_ap_filter(60)
    rx.reset()
    rx.set_ap_filter(60)
    assert rx.get_ap_filter() == 60
    rx.close()


def test_split_form_slicer_leaves_ap_unset(port):
    rng = np.random.default_rng(25)
    addr = 0x3C6586
    chips = np.zeros((3, 240), np.float32)
    for i, (df, code) in enumerate([(17, 0), (11, 9), (4, 0)]):
        c = synth.frame_chips(apc.one_frame(df, addr, rng, code))
        chips[i, :c.size] = c
    q = am.msg_queue()
    sl = am.slicer(q)
    sl._ctx.call("amb_set_option", b"ap_filter", 60)
    frames = sl.process(chips, [(0, 0.0)] * 3)
    assert [f.ap for f in frames] == [0, 0, 0] and [f.passed for f in frames] == [1, 0, 1]
    want = port.run_slicer(chips, np.zeros(3, np.uint64), np.zeros(3))
    assert q.strings() == want.msgs
