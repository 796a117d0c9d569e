"""The rules of the Beast binary and AVR raw feeds (include/airmodes_b200.h; DESIGN.md §8 "Beast and AVR feeds") on
the independent checker tests/beast_oracle.py, CPU only: the worked vectors as literals, the escape of 0x1a in every
position, the timestamp at the 2^48 wrap, at secs near 2^64, at half-tick ties and for fracs that are not finite or too
large, the signal byte at its edges, parse(encode(frames)) for every queued frame, and a timestamp that never
decreases over a stream of rx_path's stamps."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_oracle as bo  # noqa: E402

DF17 = "8D4840D6202CC371C32CE0576098"


def _frame(hexstr=DF17, secs=1, frac=0.5, level=0.25, passed=1):
    from gr_air_modes_b200 import decode
    fr = np.zeros(1, dtype=decode.FRAME_DTYPE)
    raw = bytes.fromhex(hexstr)
    fr["data"][0][: len(raw)] = np.frombuffer(raw, np.uint8)
    fr["nbits"], fr["df"] = 8 * len(raw), raw[0] >> 3
    fr["secs"], fr["frac"], fr["ref_level"], fr["passed"] = secs, frac, np.float32(level), passed
    return fr


def test_worked_vectors():
    fr = _frame()
    assert bo.beast(fr) == bytes.fromhex("1A 33 00 00 01 12 A8 80 80 8D 48 40 D6 20 2C C3 71 C3 2C E0 57 60 98")
    assert bo.avr(fr, 2) == b"@00000112A8808D4840D6202CC371C32CE0576098;\n"
    assert bo.avr(fr, 1) == b"*8D4840D6202CC371C32CE0576098;\n"
    t = 0x1A1A1A1A1A1A
    fr = _frame(secs=t // 12_000_000, frac=(t % 12_000_000) / 12e6, level=float(np.float32((26 / 255) ** 2)))
    assert bo.timestamp(fr["secs"][0], fr["frac"][0]) == t and bo.signal(fr["ref_level"][0]) == 0x1A
    assert bo.beast(fr) == b"\x1a\x33" + b"\x1a" * 14 + bytes.fromhex(DF17)


def test_escape_in_every_position():
    for i in range(14):                                  # each payload byte on its own
        raw = bytearray(bytes.fromhex(DF17))
        raw[i] = 0x1A
        fr = _frame(raw.hex(), secs=0, frac=0.0, level=0.0)
        want = b"\x1a\x33" + bytes(7) + bytes(raw).replace(b"\x1a", b"\x1a\x1a")
        assert bo.beast(fr) == want and len(want) == 2 + 7 + 15
    for i in range(6):                                   # each timestamp byte on its own
        t = 0x1A << (40 - 8 * i)
        fr = _frame("5D4840D6AAAAAA", secs=t // 12_000_000, frac=(t % 12_000_000) / 12e6, level=0.0)
        assert bo.timestamp(fr["secs"][0], fr["frac"][0]) == t
        msg = bo.beast(fr)
        assert msg[:2] == b"\x1a\x32" and msg[2:2 + 7] == t.to_bytes(6, "big")[: i + 1] + b"\x1a" + \
            t.to_bytes(6, "big")[i + 1:] and len(msg) == 2 + 1 + 7 + 7
    fr = _frame(level=float(np.float32((26 / 255) ** 2)), secs=0, frac=0.0)   # the signal byte
    assert bo.beast(fr)[8:10] == b"\x1a\x1a"
    # the longest message: every byte after the type byte is 0x1a
    t = 0x1A1A1A1A1A1A
    fr = _frame("1A" * 14, secs=t // 12_000_000, frac=(t % 12_000_000) / 12e6, level=float(np.float32((26 / 255) ** 2)))
    assert bo.beast(fr) == b"\x1a\x33" + b"\x1a" * 42 and len(bo.beast(fr)) == 44
    assert bo.parse_beast(bo.beast(fr)) == [(t, 0x1A, b"\x1a" * 14)]


def test_timestamp_wrap_and_secs_near_2_64():
    wrap = (1 << 48) // 12_000_000
    assert bo.timestamp(wrap, 0.0) == wrap * 12_000_000 < 1 << 48
    assert bo.timestamp(wrap + 1, 0.0) == (wrap + 1) * 12_000_000 - (1 << 48)
    left = (1 << 48) - wrap * 12_000_000                 # ticks to the wrap from secs = wrap
    assert bo.timestamp(wrap, (left - 1) / 12e6) == (1 << 48) - 1
    assert bo.timestamp(wrap, left / 12e6) == 0
    for secs in (2 ** 64 - 1, 2 ** 64 - 2, 2 ** 63):
        assert bo.timestamp(secs, 0.25) == ((secs * 12_000_000) % 2 ** 64 + 3_000_000) % 2 ** 48
    assert bo.timestamp(0, -0.25) == (1 << 48) - 3_000_000         # (uint64)(int64) of a negative count
    fr = _frame(secs=2 ** 64 - 1, frac=0.999)
    assert bo.parse_avr(bo.avr(fr, 2))[0][0] == bo.timestamp(2 ** 64 - 1, 0.999)


def test_half_tick_ties_round_to_even():
    assert 2.0 ** -9 * 12e6 == 23437.5 and bo.timestamp(0, 2.0 ** -9) == 23438
    assert 3 * 2.0 ** -9 * 12e6 == 70312.5 and bo.timestamp(0, 3 * 2.0 ** -9) == 70312
    assert bo.timestamp(0, 5 * 2.0 ** -9) == 117188                   # 117187.5
    assert bo.timestamp(0, -(2.0 ** -9)) == (1 << 48) - 23438


@pytest.mark.parametrize("frac", [float("nan"), float("inf"), float("-inf"), 1e300, 2.0 ** 62 / 12e6,
                                  -2.0 ** 62 / 12e6])
def test_frac_not_finite_or_too_large_gives_zero(frac):
    assert bo.timestamp(12345, frac) == 0
    assert bo.beast(_frame(secs=12345, frac=frac))[2:8] == bytes(6)
    assert bo.timestamp(12345, float(np.nextafter(2.0 ** 62 / 12e6, 0))) != 0


def test_signal_byte():
    assert bo.signal(float("nan")) == 0 and bo.signal(-1.0) == 0 and bo.signal(-0.0) == 0 and bo.signal(0.0) == 0
    assert bo.signal(1e-45) == 1 and bo.signal(1e-10) == 1             # tiny positive: at least 1
    assert bo.signal(1.0) == 255 and bo.signal(2.0) == 255 and bo.signal(float("inf")) == 255
    assert bo.signal(0.25) == 128                                        # 127.5, half to even
    assert bo.signal(float(np.float32((26 / 255) ** 2))) == 26
    assert bo.signal(float(np.float32(0.999))) == 255                   # 254.87
    for s in range(1, 256):                                              # (S / 255)^2 reads back as S
        assert bo.signal(float(np.float32((s / 255) ** 2))) == s


def test_parse_of_encode_returns_every_queued_frame():
    fr = bo.adversarial_frames()
    q = fr["passed"] != 0
    assert 0 < q.sum() < len(fr)
    want = [(bo.timestamp(f["secs"], f["frac"]), bo.signal(f["ref_level"]), bo.payload(f)) for f in fr[q]]
    assert bo.parse_beast(bo.beast(fr)) == want
    assert bo.parse_avr(bo.avr(fr, 2)) == [(t, p) for t, _, p in want]
    assert bo.parse_avr(bo.avr(fr, 1)) == [(None, p) for _, _, p in want]
    lines = bo.avr(fr, 2).split(b"\n")[:-1]
    assert {len(x) + 1 for x in lines} == {29, 43} and {len(x) + 1 for x in bo.avr(fr, 1).split(b"\n")[:-1]} == {17, 31}
    # records decide, not passed: a record marked not queued is left out
    from gr_air_modes_b200 import decode
    recs = np.zeros(len(fr), dtype=decode.FIELDS_DTYPE)
    recs["status"] = np.where(q, 0, bo.FS_NOT_QUEUED)
    assert bo.beast(fr, recs) == bo.beast(fr)
    with pytest.raises(ValueError):
        bo.parse_beast(bo.beast(fr)[:-1])
    with pytest.raises(ValueError):
        bo.parse_beast(b"\x1a\x33\x1a\x00" + bytes(20))


@pytest.mark.parametrize("rate", [4_000_000, 10_000_000, 20_000_000])
def test_timestamp_never_decreases_over_rx_path_stamps(rate):
    """rx_path's stamp without a start time (secs = count // rate, frac = (count % rate) / rate, amb_api.cu stamp):
    T follows the sample count, also across second boundaries."""
    rng = np.random.default_rng(rate // 1000)
    counts = np.unique(np.concatenate([np.sort(rng.integers(0, 50 * rate, 20000)),
                                       np.arange(rate - 40, rate + 40), np.arange(7 * rate - 40, 7 * rate + 40)]))
    ts = [bo.timestamp(int(c) // rate, float(np.float64(int(c) % rate) / np.float64(rate))) for c in counts]
    assert all(b >= a for a, b in zip(ts, ts[1:]))
    assert all(abs(t - int(c) * 12_000_000 / rate) <= 0.5 for t, c in zip(ts, counts))
