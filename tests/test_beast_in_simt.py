"""Beast binary input's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_beast_in.cuh) and C ABI on the host, through the
emulated library (tests/simt/library_emul.cc) and gr_air_modes_b200.beast.beast_reader: the frames equal
tests/beast_in_oracle.py's field for field (the bits of frac and ref_level included), and the counters counter for
counter, for the writer's bytes of the golden scenes' frames and the adversarial frames, garbage dense in 0x1a, 0x1a
runs of 1 to 70 before every type byte, and messages of nothing but 0x1a; under every cut of a short stream into two
calls, random cuts of a long one and cuts inside 0x1a runs. Also: five launches per call whatever the size, the C ABI's
AMB_ERR_STATE / AMB_ERR_OVERFLOW / AMB_ERR_INVALID, and the decoder's records, SBS-1 lines and text reports of the
reader's frames equal those of the oracle's. Four mutants must fail: the run parity taken from the wrong end, the odd
trailing 0x1a dropped from the carry, a body cut by a sync token still emitted, and the level computed in float."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_in_oracle as bi  # noqa: E402
import beast_oracle as bo  # noqa: E402
import emul_build  # noqa: E402
from test_beast_simt import _scene_frames  # noqa: E402

ESC = 0x1A


def _use(path):
    from gr_air_modes_b200 import _lib
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = path, None
    return saved


def _restore(saved):
    from gr_air_modes_b200 import _lib
    _lib.LIB_PATH, _lib._lib = saved


@pytest.fixture(scope="module")
def emulated_library(tmp_path_factory):
    saved = _use(emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL))
    try:
        yield
    finally:
        _restore(saved)


def _written():
    """The writer's bytes of the golden scenes' frames and of the adversarial frames."""
    fr = np.ascontiguousarray(np.concatenate([_scene_frames()[:400], bo.adversarial_frames()]))
    return bo.beast(fr)


def _runs():
    """0x1a runs of length 1 to 70 before every type byte, each followed by a whole message."""
    m = bi.message(0x33, 0x1A1A1A1A1A1A, ESC, bytes.fromhex("8D1A1A1A201A1A1A1A1A1A1A1A1A"))
    out = bytearray()
    for r in range(1, 71):
        for ty in (0x31, 0x32, 0x33, 0x34, 0x00, ESC + 1):
            out += b"\x1a" * r + bytes([ty]) + m
    return bytes(out)


def _all_escapes():
    """Messages whose every byte is 0x1a: T = 0x1a1a1a1a1a1a, S = 0x1a, a payload of 0x1a bytes."""
    return b"".join(bi.message(ty, 0x1A1A1A1A1A1A, ESC, b"\x1a" * n) for ty, n in ((0x33, 14), (0x32, 7), (0x31, 2))) * 5


def _streams():
    rng = np.random.default_rng(5)
    return {"written": _written(), "garbage": bi.garbage(rng, 9000, 0.5) + _written()[:3000] + bi.garbage(rng, 5000, 0.8),
            "runs": _runs(), "escapes": _all_escapes()}


def _read(data, cuts, reader=None):
    """Frames (concatenated) and counters of the reader over `data` cut at `cuts`, flush on the last call."""
    from gr_air_modes_b200 import beast
    r = reader or beast.beast_reader()
    try:
        r.reset()
        parts = []
        bounds = [0] + list(cuts) + [len(data)]
        for k in range(len(bounds) - 1):
            parts.append(r.process(data[bounds[k]: bounds[k + 1]], flush=k == len(bounds) - 2))
        st = r.stats()
        return np.concatenate(parts), st
    finally:
        if reader is None:
            r.close()


def _check(data, cuts, reader=None):
    want, cnt, _ = bi.parse(data)
    got, st = _read(data, cuts, reader)
    assert got.dtype == want.dtype and len(got) == len(want)
    for name in want.dtype.names:
        assert want[name].tobytes() == got[name].tobytes(), name
    assert {k: st[k] for k in cnt} == cnt and st["bytes_in"] == len(data) and st["carried"] == 0


@pytest.mark.parametrize("which", ["written", "garbage", "runs", "escapes"])
def test_one_call_equals_the_oracle(emulated_library, which):
    data = _streams()[which]
    _check(data, [])
    if which == "written":
        fr, _, _ = bi.parse(data)
        assert (fr["passed"] == 0).any()                     # DF11 payloads with a syndrome among them (rule 4)
        fr["passed"] = 1
        assert bo.beast(fr) == data                          # frames -> Beast -> frames -> Beast: the same bytes


def test_every_cut_of_a_short_stream(emulated_library):
    from gr_air_modes_b200 import beast
    data = b"q\x1a" + _all_escapes()[:60] + bi.message(0x32, 7, 9, bytes.fromhex("5D4840D6AAAAAA")) + b"\x1a\x1a\x1a"
    r = beast.beast_reader()
    try:
        for c in range(len(data) + 1):
            _check(data, [c], r)
    finally:
        r.close()


def test_random_cuts_and_cuts_inside_runs(emulated_library):
    from gr_air_modes_b200 import beast
    rng = np.random.default_rng(17)
    r = beast.beast_reader()
    try:
        for which, data in _streams().items():
            _check(data, sorted(set(rng.integers(0, len(data), 12).tolist())), r)
            runs = [i for i in range(1, len(data)) if data[i - 1] == ESC and data[i] == ESC]
            _check(data, sorted(set(rng.choice(runs, min(len(runs), 25), replace=False).tolist())), r)
    finally:
        r.close()


def test_carry_between_calls(emulated_library):
    from gr_air_modes_b200 import beast
    m = bi.message(0x33, 1, 2, bytes.fromhex("8D4840D6202CC371C32CE0576098"))
    r = beast.beast_reader()
    try:
        for k in range(len(m)):
            r.reset()
            assert len(r.process(b"xx" + m[:k])) == 0
            p = bi.Parser()
            p.feed(b"xx" + m[:k])
            assert r.stats()["carried"] == p.carry() <= 43, k
        r.reset()
        assert len(r.process(b"\x1a" * 43)) == 0 and r.stats()["carried"] == 1
    finally:
        r.close()


def test_launches_per_call_do_not_depend_on_size(emulated_library):
    from gr_air_modes_b200 import beast
    r = beast.beast_reader()
    try:
        data = _written()
        for n in (0, 1, 100, len(data)):
            k0 = r.stats()["kernel_launches"]
            r.process(data[:n])
            assert r.stats()["kernel_launches"] - k0 == 5, n
    finally:
        r.close()


def test_c_abi_errors(emulated_library):
    from gr_air_modes_b200 import _lib, beast
    r = beast.beast_reader()
    lib, h = r._lib, r._h
    try:
        data = _written()[:2000]
        n = r._push(data, False)
        assert n > 3
        buf = (C.c_uint8 * (80 * n))(*([0xEE] * (80 * n)))
        assert lib.amb_beast_reader_frames(h, None, 0) == n
        assert lib.amb_beast_reader_frames(h, buf, n - 1) == _lib.ERR_OVERFLOW
        assert bytes(buf) == b"\xee" * (80 * n)                         # nothing written
        assert lib.amb_beast_reader_last_error(h).decode() == "amb_beast_reader_frames: output buffer too small"
        assert lib.amb_beast_reader_frames(h, buf, n) == n
        assert lib.amb_beast_reader_push(h, None, 5, _lib.MEM_HOST, 0) == _lib.ERR_INVALID
        assert lib.amb_beast_reader_push(h, data, 5, 7, 0) == _lib.ERR_INVALID
        assert lib.amb_beast_reader_push(h, data, _lib.BEAST_PUSH_MAX + 1, _lib.MEM_HOST, 0) == _lib.ERR_INVALID
        assert "AMB_BEAST_PUSH_MAX" in lib.amb_beast_reader_last_error(h).decode()
        with pytest.raises(ValueError):
            r.process(np.zeros(4, np.float32))
        r.process(b"", flush=True)
        assert lib.amb_beast_reader_push(h, data, 5, _lib.MEM_HOST, 0) == _lib.ERR_STATE
        with pytest.raises(RuntimeError, match="flushed"):
            r.process(data)
        r.reset()
        assert len(r.process(data, flush=True)) == n
    finally:
        r.close()


def test_decoder_of_reader_frames_equals_decoder_of_oracle_frames(emulated_library):
    from gr_air_modes_b200 import beast, decode
    data = _written() + bi.garbage(np.random.default_rng(3), 3000, 0.5)
    want, _, _ = bi.parse(data)
    r = beast.beast_reader()
    try:
        got = r.process(data, flush=True)
    finally:
        r.close()
    out = []
    for fr in (got, want):
        d = decode.batch_decoder(None, sbs1=True, reports=True)
        try:
            out.append((d.decode(fr).tobytes(), d.sbs1_text(), d.report_text()))
        finally:
            d.close()
    assert out[0] == out[1] and len(out[0][2]) > 1000


MUTANTS = [
    # the run parity from the first byte of a tile that is not 0x1a, not the last
    ("if (t0 + k < L && amb_bin_at(s, in, t0 + k) != AMB_BIN_ESC) m = t0 + k;",
     "if (t0 + k < L && amb_bin_at(s, in, t0 + k) != AMB_BIN_ESC && m < 0) m = t0 + k;"),
    # the odd trailing 0x1a dropped from the carry
    ("            if (!flush) atomicMin(&dv->cs, (unsigned)i);", "            if (false) atomicMin(&dv->cs, (unsigned)i);"),
    # a body cut by a sync token read on as data, and emitted
    ("if (b[p + 1] != AMB_BIN_ESC) { *got = k; return AMB_BIN_TRUNCATED; }", "if (false) { *got = k; return AMB_BIN_TRUNCATED; }"),
    # the level in float arithmetic ((float)(S * S) / 65025.0f would be exact-equivalent: both are one correctly rounded
    # quotient of exact operands)
    ("f->ref_level = (float)((double)(S * S) / 65025.0);", "f->ref_level = (S / 255.0f) * (S / 255.0f);"),
]


@pytest.mark.parametrize("which", range(len(MUTANTS)))
def test_mutants_fail(tmp_path, tmp_path_factory, which):
    old, new = MUTANTS[which]
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(emul_build.ROOT, sub), str(tmp_path / sub))
    p = tmp_path / "gr_air_modes_b200/csrc/amb_beast_in.cuh"
    src = p.read_text()
    assert src.count(old) == 1
    p.write_text(src.replace(old, new))
    saved = _use(emul_build.build(tmp_path_factory, tmp_path / "tests/simt/library_emul.cc"))
    try:
        rng = np.random.default_rng(23)
        failed = 0
        for which_stream, data in _streams().items():
            for cuts in ([], sorted(rng.integers(0, len(data), 12).tolist())):
                try:
                    _check(data, cuts)
                except AssertionError:
                    failed += 1
        assert failed
    finally:
        _restore(saved)
