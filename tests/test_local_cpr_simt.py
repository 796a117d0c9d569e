"""The local CPR stage's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_local.cuh, launched by its own launcher after
the fields, pairing and resolve kernels) on the host under the SIMT emulator (tests/simt/simt_emul.h), against the
sequential replay of the same arithmetic (tests/local_cpr_host_shim.cc) byte for byte and against the brute-force checker
(tests/local_cpr_oracle.py) record for record: decode_cases scenes in several batch splits (single messages, cuts at
31/32/33 inside a 32-message step), a bucket holding many aircraft, and one aircraft with far more than 32 consecutive
local fixes. A copy of the kernel whose lanes read the table instead of their predecessor's fix must fail."""
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

import local_cpr_cases as lc  # noqa: E402
import local_cpr_oracle as lo  # noqa: E402


def _bind_emul(path):
    e = C.CDLL(path)
    e.emul_local_new.restype = C.c_void_p
    e.emul_local_new.argtypes = [C.c_int]
    e.emul_local_free.argtypes = [C.c_void_p]
    e.emul_decode_local.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p]
    return e


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = tmp_path_factory.mktemp("simt_local")
    emul, shim = str(d / "libdecode_emul.so"), str(d / "libdecode_shim.so")
    subprocess.run(FLAGS + ["-o", emul, os.path.join(ROOT, "tests", "simt", "decode_local_emul.cc")], check=True)
    subprocess.run(FLAGS + ["-o", shim, os.path.join(ROOT, "tests", "local_cpr_host_shim.cc")], check=True)
    s = C.CDLL(shim)
    s.shim_local_new.restype = C.c_void_p
    s.shim_local_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p]
    return _bind_emul(emul), s


def _run(e, s, msgs, loc, S, splits):
    """Decode msgs in batches cut at `splits` (batch sizes; the rest in one) by the emulated kernels and by the shim."""
    from gr_air_modes_b200 import decode
    arr, n = decode.frames_from_messages(msgs)
    have, lat, lon = (0, 0.0, 0.0) if loc is None else (1, loc[0], loc[1])
    he = e.emul_local_new(17)
    hs = s.shim_local_new() if s is not None else None
    got = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    want = np.zeros(n, dtype=decode.FIELDS_DTYPE)
    base, pos = C.addressof(arr), 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c <= 0:
            break
        fr = C.c_void_p(base + 80 * pos)
        assert e.emul_decode_local(he, fr, c, have, lat, lon, S, C.c_void_p(got.ctypes.data + 144 * pos)) == 0
        if hs is not None:
            s.shim_local_step(hs, fr, c, have, lat, lon, S, C.c_void_p(want.ctypes.data + 144 * pos))
        pos += c
    e.emul_local_free(he)
    return got, want


def _check(e, s, msgs, loc, S, splits, where):
    got, want = _run(e, s, msgs, loc, S, splits)
    assert got.tobytes() == want.tobytes(), where                    # every byte of every record
    chk = lo.decode_local(msgs, loc, S)
    lc.assert_records_match(got, chk, where)
    return chk


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_decode_case_scenes_in_batch_splits(libs, case):
    import decode_cases as dc
    e, s = libs
    loc, msgs = dc.make_case(**dc.CASES[case])
    msgs = lc.remap_addresses(msgs)
    S = (10, 60, 600, 60)[case]
    for splits in ([], [1] * 40 + [31, 32, 33, 31, 65]):
        chk = _check(e, s, msgs, loc, S, splits, (case, len(splits)))
    outcomes = [r["local"] for r in chk]
    assert outcomes.count(lo.LOCAL_NO_REF) >= 1
    if case == 3:
        assert outcomes.count(lo.LOCAL_DECODED) >= 1 and outcomes.count(lo.LOCAL_REJECTED) >= 1


def test_weak_signal_trajectories(libs):
    """Tracks with 90 % of the messages lost, and fades: many positions only the local decode gives."""
    e, s = libs
    msgs, _ = lc.trajectory_scene(3, n_aircraft=12, seconds=120.0, drop=0.9, small_addresses=True)
    for splits, loc in (([], None), ([1] * 20 + [31, 32, 33, 500], (48.0, 11.0))):
        chk = _check(e, s, msgs, loc, 30, splits, splits)
    outcomes = [r["local"] for r in chk]
    assert outcomes.count(lo.LOCAL_DECODED) >= 40


def test_off_leaves_the_plain_decode(libs):
    import decode_cases as dc
    e, s = libs
    loc, msgs = dc.make_case(**dc.CASES[0])
    msgs = lc.remap_addresses(msgs)[:600]
    got, want = _run(e, s, msgs, loc, 0, [])
    assert got.tobytes() == want.tobytes()
    from oracle import decode_oracle as do
    assert [r["status"] for r in do.decode_batch(msgs, loc)] == got["status"].tolist()
    assert not np.any(got["pad_"])


def test_many_aircraft_in_one_bucket(libs):
    e, s = libs
    msgs = lc.bucket_scene()
    for splits, loc in (([], None), ([33, 1, 31, 32, 700], (10.0, 20.0))):
        chk = _check(e, s, msgs, loc, 30, splits, splits)
    outcomes = [r["local"] for r in chk]
    assert outcomes.count(lo.LOCAL_DECODED) >= 200 and outcomes.count(lo.LOCAL_STALE) + outcomes.count(lo.LOCAL_NO_REF) >= 1


def test_one_aircraft_with_a_long_local_chain(libs):
    e, s = libs
    msgs = lc.chain_scene(n_local=100)
    for splits in ([], [2, 31, 1, 32, 33]):
        chk = _check(e, s, msgs, None, 5, splits, splits)
    run, best = 0, 0
    for r in chk:
        if r["icao"] == 0x1234 and r["surface"]:
            run = run + 1 if r["local"] == lo.LOCAL_DECODED else 0
            best = max(best, run)
    assert best > 64


def test_a_chain_that_reads_the_table_instead_of_its_predecessor_is_caught(libs, tmp_path):
    """Mutation: every lane takes its reference from the table, none from the previous member of its group."""
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / "gr_air_modes_b200/csrc/amb_decode_local.cuh"
    src = p.read_text()
    a, b = "if (mine && rank == 0) {", "if (mine && (rank == 0 || (fields[k].status & AMB_FS_HAS_POS))) {"
    assert src.count(a) == 1 and src.count(b) == 1
    p.write_text(src.replace(a, "if (mine) {").replace(b, "if (mine) {"))
    lib = str(tmp_path / "libbroken.so")
    subprocess.run(FLAGS + ["-o", lib, str(tmp_path / "tests/simt/decode_local_emul.cc")], check=True)
    e = _bind_emul(lib)
    msgs = lc.chain_scene(n_local=100)
    got, _ = _run(e, None, msgs, None, 5, [])
    with pytest.raises(AssertionError):
        lc.assert_records_match(got, lo.decode_local(msgs, None, 5), "mutant")
