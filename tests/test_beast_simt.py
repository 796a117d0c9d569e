"""The Beast and AVR feeds' KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_beast.cuh, enqueued by the decoder's own
amb_decode_launch) on the host under the SIMT emulator (tests/simt/simt_emul.h), through the decoder harness
tests/simt/decode_emul.cc (tests/simt/beast_emul.cc adds the read-out of every kind): the bytes of every call equal
tests/beast_oracle.py's, byte for byte, for option beast and both AVR forms, over the frames of the golden scenes and
the adversarial frames (escapes everywhere, the 2^48 wrap, secs near 2^64, ties, fracs that are not finite, every edge
of the signal byte, unqueued and error-corrected frames); arbitrary cuts into calls concatenate to the one-call bytes.
With the options off the records, the SBS-1 and report text and the launch count equal a decoder's that never had
them; each option on adds exactly three launches. Through the emulated library (tests/simt/library_emul.cc), the C ABI
and batch_decoder: AMB_ERR_STATE while an option is off, AMB_ERR_OVERFLOW with nothing written and the size due, and
the feed of rx_path's own frames. Two mutants must fail: ties rounded away from zero, and a payload byte 0x1a written
once."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_oracle as bo  # noqa: E402
import emul_build  # noqa: E402
from helpers import load_decode_golden  # noqa: E402

BEAST_EMUL = os.path.join(emul_build.ROOT, "tests", "simt", "beast_emul.cc")
TEXT_SBS1, TEXT_REPORTS, TEXT_BEAST, TEXT_AVR = 0, 1, 2, 3
AMB_ERR_STATE = -8
# (beast, avr) settings checked: every format and form
SETTINGS = [(1, 0), (0, 1), (0, 2), (1, 2)]


def _bind(e):
    e.emul_feed.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    e.emul_feed_poison.argtypes = [C.c_void_p]
    e.emul_feed_state.argtypes = [C.c_void_p]
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(emul_build.decode_emul(tmp_path_factory, BEAST_EMUL))


def _scene_frames():
    """The frames of the golden scenes (tests/golden/golden.json: the reference's messages of scenes.npz) and of the
    decode golden cases, parsed back from their messages; DF17 positions kept below the harness's 2^15 addresses."""
    from gr_air_modes_b200 import decode
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden.json")) as f:
        msgs = [m for s in json.load(f)["scenes"] for m in s["msgs"]]
    msgs += [m for case in load_decode_golden()[:3] for m in (tuple(x) for x in case["msgs"])]
    arr, n = decode.frames_from_messages(msgs)
    fr = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=n).copy()
    icao = (fr["data"][:, 1].astype(np.int64) << 16) | (fr["data"][:, 2].astype(np.int64) << 8) | fr["data"][:, 3]
    return np.ascontiguousarray(fr[(fr["df"] != 17) | (icao < (1 << 15))])


def _inputs():
    return np.ascontiguousarray(np.concatenate([_scene_frames()[:700], bo.adversarial_frames()]))


def _feed(e, h, kind, cap):
    n = C.c_size_t()
    buf = C.create_string_buffer(max(cap, 1))
    assert e.emul_feed(h, kind, buf, len(buf), C.byref(n)) == 0
    return buf.raw[: n.value]


def _run(e, h, frames, beast, avr, **stages):
    """One emulated decode with options beast / avr (and `stages`); returns (records, Beast bytes, AVR bytes), the
    bytes None for an option that is off."""
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    emul_build.opts(e, h, None, beast=beast, avr=avr, **stages)
    e.emul_feed_poison(h)
    assert e.emul_decode(h, C.c_void_p(frames.ctypes.data), len(frames), C.c_void_p(recs.ctypes.data)) == 0
    b = _feed(e, h, TEXT_BEAST, 44 * len(frames)) if beast else None
    a = _feed(e, h, TEXT_AVR, 43 * len(frames)) if avr else None
    return recs, b, a


def _stream(e, frames, cuts, beast, avr):
    h = e.emul_new(17)
    try:
        got_b, got_a = [], []
        for lo, hi in zip([0] + list(cuts), list(cuts) + [len(frames)]):
            if lo == hi:
                continue
            part = np.ascontiguousarray(frames[lo:hi])
            recs, b, a = _run(e, h, part, beast, avr)
            if beast:
                assert b == bo.beast(part, recs), (lo, hi)
                got_b.append(b)
            if avr:
                assert a == bo.avr(part, avr, recs), (lo, hi)
                got_a.append(a)
        return b"".join(got_b), b"".join(got_a)
    finally:
        e.emul_free(h)


@pytest.mark.parametrize("beast,avr", SETTINGS)
def test_bytes_equal_the_oracle_in_one_call(emul, beast, avr):
    fr = _inputs()
    assert (fr["passed"] == 0).any() and (fr["pad_"][:, 0] == 1).any()
    b, a = _stream(emul, fr, [], beast, avr)
    if beast:
        assert b == bo.beast(fr) and len(bo.parse_beast(b)) == int((fr["passed"] != 0).sum())
        assert b"\x1a\x33" + b"\x1a" * 14 in b                   # the worked vector of 0x1a everywhere
    if avr:
        assert a == bo.avr(fr, avr)


@pytest.mark.parametrize("beast,avr", SETTINGS[:3])
def test_cuts_concatenate_to_the_one_call_bytes(emul, beast, avr):
    fr = _inputs()
    rng = np.random.default_rng(11 + 3 * beast + avr)
    one = _stream(emul, fr, [], beast, avr)
    for cuts in ([1, 31, 32, 33, 127, 128, 129], sorted(rng.integers(0, len(fr), 8).tolist()),
                 list(range(len(fr) - 20, len(fr)))):
        assert _stream(emul, fr, cuts, beast, avr) == one, cuts


def test_off_changes_nothing_and_on_adds_three_launches_per_option(emul):
    """Decoder X runs call 1 with the feeds on and call 2 with them off; decoder Y never has them. Records, SBS-1 lines
    and text reports of both calls are equal, and so are the launches of call 2; call 1 has three more per option."""
    fr = _inputs()
    first, second = np.ascontiguousarray(fr[: len(fr) // 2]), np.ascontiguousarray(fr[len(fr) // 2:])
    for beast, avr in SETTINGS:
        out = {}
        for name, on in (("X", (beast, avr)), ("Y", (0, 0))):
            h = emul.emul_new(17)
            try:
                rows = []
                for part, (b, a) in ((first, on), (second, (0, 0))):
                    k0 = emul.simt_launch_count()
                    recs, _, _ = _run(emul, h, part, b, a, sbs1=1, reports=1, commb=30)
                    k = emul.simt_launch_count() - k0
                    rows.append((recs.tobytes(), _feed(emul, h, TEXT_SBS1, 200 * len(part)),
                                 _feed(emul, h, TEXT_REPORTS, 480 * len(part)), k))
                out[name] = (rows, emul.emul_feed_state(h))
            finally:
                emul.emul_free(h)
        (x1, x2), sx = out["X"]
        (y1, y2), sy = out["Y"]
        assert x1[:3] == y1[:3] and x2 == y2
        assert x1[3] == y1[3] + 3 * (beast + (avr > 0))
        assert sy == 0 and sx == (1 if beast else 0) | (2 if avr else 0)   # nothing allocated for an option never on


MUTANTS = [
    ("gr_air_modes_b200/csrc/amb_decode_beast.cuh", "(uint64_t)(int64_t)rint(x)", "(uint64_t)(int64_t)round(x)"),
    ("gr_air_modes_b200/csrc/amb_decode_beast.cuh", "i == 6 ? S : f.data[i - 7];",
     "i == 6 ? S : f.data[i - 7]; if (i > 6 && b == 0x1a) { if (out) out[L] = (char)b; L++; continue; }"),
]


@pytest.mark.parametrize("which", range(len(MUTANTS)))
def test_mutants_fail(tmp_path, tmp_path_factory, which):
    import shutil
    rel, old, new = MUTANTS[which]
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(emul_build.ROOT, sub), str(tmp_path / sub))
    src = (tmp_path / rel).read_text()
    assert src.count(old) == 1
    (tmp_path / rel).write_text(src.replace(old, new))
    e = _bind(emul_build.decode_emul(tmp_path_factory, tmp_path / "tests/simt/beast_emul.cc"))
    with pytest.raises(AssertionError):
        _stream(e, bo.adversarial_frames(), [], 1, 2)


# ---- the C ABI and batch_decoder, through the emulated library -----------------------------------------------------
@pytest.fixture(scope="module")
def emulated_library(tmp_path_factory):
    from gr_air_modes_b200 import _lib
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def test_c_abi_state_and_overflow(emulated_library):
    from gr_air_modes_b200 import _lib, decode
    fr = bo.adversarial_frames()
    d = decode.batch_decoder(None)
    try:
        lib, h = d._lib, d._h
        n = C.c_size_t(7)
        for fetch, name in ((lib.amb_decoder_beast, b"beast"), (lib.amb_decoder_beast_device, b"beast"),
                            (lib.amb_decoder_avr, b"avr"), (lib.amb_decoder_avr_device, b"avr")):
            assert fetch(h, None, 0, C.byref(n)) == AMB_ERR_STATE and n.value == 0
            assert lib.amb_decoder_last_error(h).decode().endswith("option %s is off" % name.decode())
        assert lib.amb_decoder_last_error(h).decode() == "amb_decoder_avr_device: option avr is off"
        with pytest.raises(RuntimeError):
            d.beast_bytes()
        with pytest.raises(ValueError):
            d.set_avr(3)
        with pytest.raises(ValueError):
            d.set_avr(True)
        assert lib.amb_decoder_set_option(h, b"avr", 3) == _lib.ERR_INVALID
        assert lib.amb_decoder_last_error(h).decode() == "avr: 0 (off), 1 (* lines) or 2 (@ lines with the timestamp)"
        assert lib.amb_decoder_set_option(h, b"beast", 2) == _lib.ERR_INVALID
        assert lib.amb_decoder_last_error(h).decode() == "beast: 0 (off) or 1 (on)"
        d.set_beast(True)
        d.set_avr(2)
        assert d.get_beast() and d.get_avr() == 2
        recs = d.decode(fr)
        want_b, want_a = bo.beast(fr, recs), bo.avr(fr, 2, recs)
        for fetch, want in ((lib.amb_decoder_beast, want_b), (lib.amb_decoder_avr, want_a)):
            buf = C.create_string_buffer(b"\xee" * len(want))
            assert fetch(h, buf, len(want) - 1, C.byref(n)) == _lib.ERR_OVERFLOW and n.value == len(want)
            assert buf.raw[: len(want)] == b"\xee" * len(want)           # nothing written
            assert fetch(h, None, 0, C.byref(n)) == _lib.ERR_OVERFLOW and n.value == len(want)
            assert fetch(h, buf, len(want), C.byref(n)) == 0 and buf.raw[: len(want)] == want
        assert d.beast_bytes() == want_b and d.avr_text() == want_a
        d.set_avr(1)
        d.decode(fr[:3])
        assert d.avr_text() == bo.avr(fr[:3], 1)
        assert lib.amb_decode_frames(h, None, 0, _lib.MEM_HOST, None) == 0   # a call of nothing writes nothing
        assert d.beast_bytes() == b"" and d.avr_text() == b""
        d.set_beast(False)
        with pytest.raises(RuntimeError, match="option beast is off"):
            d.beast_bytes()
    finally:
        d.close()


def test_batch_decoder_feeds_rx_path_frames(emulated_library):
    """rx_path's own frames (a synthetic 4 Msps scene, unqueued detections among them) through batch_decoder with both
    options: the bytes equal the oracle's over the same frames, and the parsed stream is every queued frame."""
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, synth
    sc = synth.make_scene(4e6, 1 << 17, 14, seed=23)
    rx = am.rx_path(4e6, 7.0, am.msg_queue(), use_pmf=True)
    frames = []
    for lo in range(0, sc.iq.size, 1 << 16):
        rx.process(sc.iq[lo: lo + (1 << 16)], flush=lo + (1 << 16) >= sc.iq.size)
        frames += rx.frames
    rx.close()
    arr = (decode.Frame * len(frames))(*frames)
    fr = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE).copy()
    assert (fr["passed"] != 0).sum() >= 5
    d = decode.batch_decoder(None, beast=True, avr=2)
    try:
        recs = d.decode(fr)
        assert d.beast_bytes() == bo.beast(fr, recs) == bo.beast(fr)
        assert d.avr_text() == bo.avr(fr, 2)
        got = bo.parse_beast(d.beast_bytes())
        q = fr[fr["passed"] != 0]
        assert [p for _, _, p in got] == [bo.payload(f) for f in q]
        assert [t for t, _, _ in got] == [(int(f["sample_index"]) * 3) % (1 << 48) for f in q]   # 12 MHz / 4 Msps
    finally:
        d.close()
