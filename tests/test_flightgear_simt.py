"""The FlightGear feed's KERNEL SOURCE (gr_air_modes_b200/csrc/amb_decode_flightgear.cuh, enqueued by the decoder's own
amb_decode_launch) on the host under the SIMT emulator (tests/simt/simt_emul.h), through the decoder harness with the
read-out of every kind (tests/simt/beast_emul.cc): the packets of every call equal tests/flightgear_oracle.py's, byte
for byte, over the FlightGear scenes of the golden, in one call and cut into calls at 31 / 32 / 33 and at random
points, with the state carried from call to call and forgotten at a reset, and with every other option on. With the
option off the records and every other output equal a decoder's that never had it, and it adds exactly nine launches
when on. Four mutants must fail: a packet on a velocity record, state not carried across calls, >= 0 in the sign
rule, and an out-of-range category kept as a santa callsign."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402
import flightgear_cases as fc  # noqa: E402
import flightgear_oracle as fo  # noqa: E402
import track_cases as tc  # noqa: E402

BEAST_EMUL = os.path.join(emul_build.ROOT, "tests", "simt", "beast_emul.cc")
TEXT_SBS1, TEXT_REPORTS, TEXT_BEAST, TEXT_AVR, TEXT_FLIGHTGEAR = 0, 1, 2, 3, 4
LAUNCHES = 9
OTHERS = dict(local_cpr=30, commb=30, opstatus=30, track=60, track_ext=60, sbs1=1, coverage=1, reports=1, beast=1, avr=2)


def _bind(e):
    e.emul_feed.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    return e


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _bind(emul_build.decode_emul(tmp_path_factory, BEAST_EMUL))


def _frames(names=("categories", "late", "fleet", "pole")):
    """The frames of the golden's FlightGear scenes (every 97th not queued), one scene after another."""
    msgs = []
    t = 0
    for name, _, m in fc.scenes():
        if name in names:
            msgs += [(h, e, s + t, f) for h, e, s, f in m]
            t += 100000
    return tc.frames_of(msgs)


def _feed(e, h, kind, cap):
    n = C.c_size_t()
    buf = C.create_string_buffer(max(cap, 1))
    assert e.emul_feed(h, kind, buf, len(buf), C.byref(n)) == 0
    return buf.raw[: n.value]


def _run(e, h, frames, flightgear=1, **stages):
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    emul_build.opts(e, h, fc.LOCATION, flightgear=flightgear, **stages)
    k0 = e.simt_launch_count()
    assert e.emul_decode(h, C.c_void_p(frames.ctypes.data), len(frames), C.c_void_p(recs.ctypes.data)) == 0
    k = e.simt_launch_count() - k0
    return recs, (_feed(e, h, TEXT_FLIGHTGEAR, fo.PACKET_BYTES * len(frames)) if flightgear else None), k


def _stream(e, frames, cuts, reset_at=(), **stages):
    """Decode frames cut at `cuts`, reset before the calls whose start is in reset_at; every call's packets must equal
    the checker's. Returns the packets of all calls."""
    h = e.emul_new(17)
    chk = fo.FgChecker()
    try:
        got = []
        for lo, hi in zip([0] + list(cuts), list(cuts) + [len(frames)]):
            if lo == hi:
                continue
            if lo in reset_at:
                e.emul_reset(h)
                chk.reset()
            part = np.ascontiguousarray(frames[lo:hi])
            recs, p, _ = _run(e, h, part, **stages)
            assert p == chk.feed(part, recs), (lo, hi)
            got.append(p)
        return b"".join(got)
    finally:
        e.emul_free(h)


def test_packets_equal_the_checker_in_one_call(emul):
    fr = _frames()
    p = _stream(emul, fr, [])
    assert len(p) % fo.PACKET_BYTES == 0 and len(p) // fo.PACKET_BYTES > 1000


def test_cuts_and_random_splits_give_the_one_call_packets(emul):
    fr = _frames(("categories", "fleet"))
    one = _stream(emul, fr, [])
    rng = np.random.default_rng(31)
    for cuts in ([31, 32, 33], list(range(31, len(fr), 32)), list(range(33, len(fr), 33)),
                 sorted(set(rng.integers(1, len(fr), 12).tolist()))):
        assert _stream(emul, fr, cuts) == one


def test_reset_forgets_callsigns_and_velocities(emul):
    fr = _frames(("categories", "late"))
    mid = len(fr) // 2
    two = _stream(emul, fr, [mid], reset_at=(mid,))
    assert two[: len(_stream(emul, fr[:mid], []))] == _stream(emul, fr[:mid], [])
    assert two[len(_stream(emul, fr[:mid], [])):] == _stream(emul, np.ascontiguousarray(fr[mid:]), [])


def test_every_other_option_on(emul):
    fr = _frames(("late", "pole", "categories"))
    _stream(emul, fr, [len(fr) // 3], **OTHERS)


def test_off_changes_nothing_and_on_adds_nine_launches(emul):
    """Decoder X runs call 1 with the feed on and call 2 with it off; decoder Y never has it. Records and every other
    output of both calls are equal, and so are the launches of call 2; call 1 has nine more. Nothing is allocated for
    an option never on."""
    fr = _frames(("late", "categories"))
    first, second = np.ascontiguousarray(fr[: len(fr) // 2]), np.ascontiguousarray(fr[len(fr) // 2:])
    out = {}
    for name, on in (("X", 1), ("Y", 0)):
        h = emul.emul_new(17)
        try:
            rows = []
            for part, fg in ((first, on), (second, 0)):
                recs, _, k = _run(emul, h, part, flightgear=fg, sbs1=1, reports=1, beast=1, avr=2, local_cpr=30)
                rows.append((recs.tobytes(), [_feed(emul, h, kind, 500 * len(part)) for kind in range(4)], k))
            out[name] = rows
        finally:
            emul.emul_free(h)
    (x1, x2), (y1, y2) = out["X"], out["Y"]
    assert x1[:2] == y1[:2] and x2 == y2
    assert x1[2] == y1[2] + LAUNCHES


def test_launch_count_is_fixed_whatever_the_data(emul):
    fr = _frames(("late",))
    h = emul.emul_new(17)
    try:
        ks = {_run(emul, h, np.ascontiguousarray(fr[lo:lo + n]))[2] - _run(emul, h, np.ascontiguousarray(fr[lo:lo + n]),
                                                                          flightgear=0)[2]
              for lo, n in ((0, 1), (5, 40), (0, len(fr)))}
    finally:
        emul.emul_free(h)
    assert ks == {LAUNCHES}


MUTANTS = [
    # a packet on a velocity record
    [("gr_air_modes_b200/csrc/amb_decode_flightgear.cuh", "if (kind == AMB_FG_POSITION) st[k] = slot;",
      "if (kind >= AMB_FG_VELOCITY) st[k] = slot;"),
     ("gr_air_modes_b200/csrc/amb_decode_flightgear.cuh", "if (amb_fg_kind(r) != AMB_FG_POSITION) return 0u;",
      "if (amb_fg_kind(r) < AMB_FG_VELOCITY) return 0u;")],
    # state not carried across calls
    [("gr_air_modes_b200/csrc/amb_decode_flightgear.cuh", "    AMB_LAUNCH((amb_fg_keys), nb,",
      "    cudaMemsetAsync(table, 0, (size_t)AMB_FG_SLOTS * sizeof(AmbFgSlot), s);\n    AMB_LAUNCH((amb_fg_keys), nb,")],
    # >= 0 in the sign rule
    [("gr_air_modes_b200/csrc/amb_fg_format.h", "if (!(q[3] > 0))", "if (!(q[3] >= 0))")],
    # an IndexError category stored as a santa callsign
    [("gr_air_modes_b200/csrc/amb_fg_format.h", "amb_fg_model(r->ftc, r->cat) >= 0 ? AMB_FG_CALLSIGN : AMB_FG_NONE",
      "AMB_FG_CALLSIGN"),
     ("gr_air_modes_b200/csrc/amb_decode_flightgear.cuh", "model = amb_fg_model(r->ftc, r->cat);",
      "model = amb_fg_model(r->ftc, r->cat) < 0 ? AMB_FG_SANTA : amb_fg_model(r->ftc, r->cat);")],
]


@pytest.mark.parametrize("which", range(len(MUTANTS)))
def test_mutants_fail(tmp_path, tmp_path_factory, which):
    import shutil
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(emul_build.ROOT, sub), str(tmp_path / sub))
    for rel, old, new in MUTANTS[which]:
        src = (tmp_path / rel).read_text()
        assert src.count(old) == 1, old
        (tmp_path / rel).write_text(src.replace(old, new))
    e = _bind(emul_build.decode_emul(tmp_path_factory, tmp_path / "tests/simt/beast_emul.cc"))
    fr = _frames(("categories", "pole"))
    with pytest.raises(AssertionError):
        _stream(e, fr, [len(fr) // 2])
