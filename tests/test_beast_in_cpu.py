"""Beast binary input rules (include/airmodes_b200.h "Beast binary input") on the oracle alone, tests/beast_in_oracle.py:
agreement with the writer's own parser over every stream tests/beast_oracle.py encodes, worked vectors, a 0x1a in
every body position, timestamp edges, the two identities (stamp -> T -> stamp and S -> level -> S), each passed rule at
its edge, and the accounting of truncated, skipped, Mode A/C and other messages."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_in_oracle as bi  # noqa: E402
import beast_oracle as bo  # noqa: E402

DF17 = bytes.fromhex("8D4840D6202CC371C32CE0576098")       # a valid DF17 (syndrome 0)
DF11 = bytes.fromhex("5D4840D6") + bi.crc24(bytes.fromhex("5D4840D6")).to_bytes(3, "big")   # all-call reply, syndrome 0


def _frames_as_written(frames):
    """(T, S, payload) of each frame the writer writes, in order."""
    q = frames[bo.queued(frames)]
    return [(bo.timestamp(f["secs"], f["frac"]), bo.signal(f["ref_level"]), bo.payload(f)) for f in q]


def test_agrees_with_the_writers_parser():
    fr = bo.adversarial_frames()
    data = bo.beast(fr)
    got, cnt, carry = bi.parse(data)
    assert [(bo.timestamp(f["secs"], f["frac"]), bo.signal(f["ref_level"]), bo.payload(f)) for f in got] \
        == bo.parse_beast(data) == _frames_as_written(fr)
    assert cnt["modes"] == len(got) and cnt["truncated"] == cnt["skipped"] == cnt["other"] == cnt["modeac"] == 0
    assert carry == 0


def test_worked_vector():
    data = b"\x1a\x33" + bytes.fromhex("000000BB8001") + b"\x80" + DF17
    fr, cnt, _ = bi.parse(data)
    assert len(fr) == 1 and cnt["modes"] == 1 and cnt["passed"] == 1
    f = fr[0]
    T = 0xBB8001                                            # 12,288,001 ticks: 1 s and 288,001 / 12e6
    assert f["secs"] == 1 and f["frac"] == 288001 / 12e6 and f["sample_index"] == 0
    assert f["ref_level"] == np.float32(128 * 128 / 65025.0)
    assert f["nbits"] == 112 and f["df"] == 17 and f["crc"] == 0 and bytes(f["data"]) == DF17
    assert bo.timestamp(f["secs"], f["frac"]) == T and bo.signal(f["ref_level"]) == 128
    short = b"\x1a\x32" + bytes(6) + b"\x01" + DF11
    fr, _, _ = bi.parse(b"xy" + short)
    assert fr[0]["sample_index"] == 2 and fr[0]["nbits"] == 56 and bytes(fr[0]["data"]) == DF11 + bytes(7)
    assert fr[0]["crc"] == bi.crc24(DF11[:4]) ^ int.from_bytes(DF11[4:], "big")


@pytest.mark.parametrize("ty,nb", [(0x32, 7), (0x33, 14)])
def test_escape_at_every_body_position(ty, nb):
    base = (bytes(6) + b"\x40" + (DF17 if nb == 14 else DF11))
    for k in range(7 + nb):
        raw = bytearray(base)
        raw[k] = 0x1A
        data = bytes([0x1A, ty]) + bi.escape(bytes(raw))
        fr, cnt, _ = bi.parse(data + data)
        assert cnt["modes"] == 2 and cnt["skipped"] == 0, k
        for f in fr:
            body = int(f["secs"] * 12000000 + round(f["frac"] * 12e6)).to_bytes(6, "big")
            assert body + bytes([bo.signal(f["ref_level"])]) + bytes(f["data"][:nb]) == bytes(raw), k


@pytest.mark.parametrize("T", [0, (1 << 48) - 1, 12_000_000, 12_000_000 - 1, 12_000_001, 7 * 12_000_000 - 1,
                               7 * 12_000_000 + 1, 0x1A1A1A1A1A1A])
def test_timestamp_edges(T):
    fr, _, _ = bi.parse(bi.message(0x33, T, 1, DF17))
    f = fr[0]
    assert f["secs"] == T // 12_000_000 and 0.0 <= f["frac"] < 1.0
    assert bo.timestamp(f["secs"], f["frac"]) == T


def test_identity_every_signal_byte():
    for S in range(256):
        assert bo.signal(bi.level(S)) == S, S


def test_identity_stamps():
    for secs, frac in bo.STAMPS:
        T = bo.timestamp(secs, frac)
        s2, f2 = bi.stamp(T)
        assert bo.timestamp(s2, f2) == T, (secs, frac)


def test_passed_rules_at_their_edges():
    def one(payload, ty=None):
        ty = ty or (0x33 if len(payload) == 14 else 0x32)
        fr, _, _ = bi.parse(bi.message(ty, 5, 9, payload))
        return fr[0]

    assert one(bytes(14))["passed"] == 0 and one(bytes(7))["passed"] == 0
    for df in (16, 17, 20, 21):                              # long DFs sent short
        assert one(bytes([df << 3]) + bytes(5) + b"\x01")["passed"] == 0, df
    for df in (0, 4, 11):                                    # short DFs sent long
        assert one(bytes([df << 3]) + bytes(12) + b"\x01")["passed"] == 0, df
    df11 = bytearray(DF11)
    df11[-1] ^= 1                                            # syndrome 1
    assert one(bytes(df11))["crc"] == 1 and one(bytes(df11))["passed"] == 0
    df17 = bytearray(DF17)
    df17[-1] ^= 1
    assert one(bytes(df17))["crc"] == 1 and one(bytes(df17))["passed"] == 0
    df4 = bytes.fromhex("20001838CA3804")                    # an altitude reply: the syndrome is the address
    assert one(df4)["crc"] != 0 and one(df4)["passed"] == 1
    assert one(DF11)["passed"] == 1 and one(DF17)["passed"] == 1


def test_accounting():
    m = bi.message(0x33, 1, 2, DF17)
    ac = bi.message(0x31, 1, 2, b"\x12\x34")
    status = b"\x1a\x34" + b"abc" + b"\x1a\x1a"              # type '4': its 4 data tokens skipped
    data = b"pre" + m[:20] + ac + b"zz" + m + status + m[:5]
    fr, cnt, carry = bi.parse(data, flush=False)
    assert cnt == {"modes": 1, "modeac": 1, "other": 1, "truncated": 1, "skipped": 3 + 2 + 4, "passed": 1}
    assert len(fr) == 1 and fr[0]["sample_index"] == 3 + 20 + len(ac) + 2 and carry == 5
    p = bi.Parser()
    p.feed(data)
    p.feed(b"", flush=True)
    assert p.counts["truncated"] == 2
    assert bi.parse(b"ab\x1a", flush=False)[2] == 1 and bi.parse(b"ab\x1a\x1a", flush=False)[2] == 0
    _, cnt, _ = bi.parse(b"ab\x1a", flush=True)
    assert cnt["skipped"] == 2                               # the lone final 0x1a is dropped uncounted
