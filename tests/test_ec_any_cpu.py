"""DF17 correction by at most M bits anywhere (option "ec_any", DESIGN.md section 0), CPU only: the code-distance facts
it rests on, checked exhaustively, and the brute-force checker of tests/ec_any_oracle.py on constructed frames."""
import ctypes as C
import os
import re
import sys
from itertools import combinations

import numpy as np
import pytest

from gr_air_modes_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_any_oracle as ea  # noqa: E402
import ec_oracle as eo  # noqa: E402
from test_ec_cpu import SYN, dropped_frame, flip, low_weight_codeword  # noqa: E402

POS = np.arange(5, 112)                       # the search set of a DF17 frame
S1 = SYN[112][5:].astype(np.int64)            # one-bit syndromes s_i, i = 5..111


def pair_syndromes():
    i, j = np.triu_indices(POS.size, 1)
    return S1[i] ^ S1[j]


def test_kernel_bit_syndromes_are_the_crc_of_one_bit():
    """amb_ec_kernel's s_i = i < 88 ? crc_rem[87 - i] : 1 << (111 - i), with crc_rem[t] = x^(t+24) mod 0xFFF409 as
    amb_upload_tables builds it, equals the bytewise syndrome of a packet that is zero but bit i."""
    rem, r = [], 0xFFF409
    for _ in range(96):
        rem.append(r)
        r = (((r << 1) ^ 0xFFF409) if r & 0x800000 else (r << 1)) & 0xFFFFFF
    got = [rem[87 - i] if i < 88 else 1 << (111 - i) for i in range(112)]
    assert got == [int(x) for x in SYN[112]]


def test_one_and_two_bit_syndromes_are_nonzero_and_distinct():
    s2 = pair_syndromes()
    assert S1.size == 107 and s2.size == 5671
    both = np.concatenate([S1, s2])
    assert np.all(both != 0)
    assert np.unique(both).size == 107 + 5671


def test_no_three_bit_pattern_aliases_to_two_bits_or_fewer():
    s2 = pair_syndromes()
    small = np.concatenate([S1, s2])
    i, j = np.triu_indices(POS.size, 1)
    s3 = np.concatenate([s2[j < k] ^ S1[k] for k in range(POS.size)])      # i < j < k
    assert s3.size == 198_485
    assert not np.isin(s3, small).any()
    assert np.all(s3 != 0)


def test_four_bit_aliases():
    """Of the 5,160,610 four-bit patterns, 2,325 have a two-bit pattern's syndrome (a false two-bit fix) and none a
    one-bit pattern's."""
    i, j = np.triu_indices(POS.size, 1)
    s2 = pair_syndromes()
    order = np.argsort(i, kind="stable")                  # pairs (c, d) by c, to take those with c > b as a suffix
    ci, s2c = i[order], s2[order]
    start = np.searchsorted(ci, np.arange(POS.size + 1))
    s4 = np.concatenate([s2[p] ^ s2c[start[j[p] + 1]:] for p in range(s2.size)])   # a < b < c < d
    assert s4.size == 5_160_610
    assert not np.isin(s4, S1).any()
    assert int(np.isin(s4, s2).sum()) == 2_325


def _df17(seed):
    return synth.make_frame(17, np.random.default_rng(seed))


@pytest.mark.parametrize("m", [1, 2])
def test_every_single_position(m):
    sent = _df17(1)
    for p in range(5, 112):
        f = dropped_frame(flip(sent, [p]), [])
        st, bits, g = ea.correct_any(f, m)
        assert (st, bits) == (ea.EC_FIXED, (p,)), p
        assert bytes(g.data)[:14] == sent and g.crc == 0 and g.passed == 1


def test_every_pair():
    sent = _df17(2)
    for pr in combinations(range(5, 112), 2):
        f = dropped_frame(flip(sent, pr), [])
        st, bits, g = ea.correct_any(f, 2)
        assert (st, bits) == (ea.EC_FIXED, pr), pr
        assert bytes(g.data)[:14] == sent and g.crc == 0 and g.passed == 1
    for pr in [(5, 6), (5, 111), (87, 88), (110, 111), (30, 64)]:
        assert ea.correct_any(dropped_frame(flip(sent, pr), []), 1)[0] == ea.EC_NO_SOLUTION, pr


def test_table_equals_brute_force_on_random_frames():
    rng = np.random.default_rng(4)
    tables = {m: ea.SyndromeTable(m) for m in (1, 2)}
    seen = {}
    for trial in range(240):
        sent = synth.make_frame(17, rng)
        w = int(rng.integers(1, 6))
        pos = sorted(int(p) for p in rng.choice(np.arange(5, 112), w, replace=False))
        payload = flip(sent, pos)
        if trial % 7 == 0:                                 # random parity: a syndrome unrelated to any small pattern
            payload = payload[:11] + bytes(int(x) for x in rng.integers(0, 256, 3))
        f = dropped_frame(payload, [])
        for m in (1, 2):
            a, b = ea.correct_any(f, m), tables[m].correct(f)
            assert (a[0], a[1], bytes(a[2])) == (b[0], b[1], bytes(b[2])), (trial, pos, m)
            seen[(m, a[0])] = seen.get((m, a[0]), 0) + 1
    assert seen.get((1, ea.EC_FIXED), 0) >= 20 and seen.get((2, ea.EC_FIXED), 0) >= 40
    assert seen.get((2, ea.EC_NO_SOLUTION), 0) >= 60


def test_three_bit_errors_have_no_solution():
    rng = np.random.default_rng(5)
    table = ea.SyndromeTable(2)
    triples = [(5, 6, 7), (5, 87, 88), (86, 87, 88), (109, 110, 111), (5, 58, 111)]
    triples += [tuple(sorted(int(p) for p in rng.choice(np.arange(5, 112), 3, replace=False))) for _ in range(40)]
    for t in triples:
        sent = synth.make_frame(17, rng)
        f = dropped_frame(flip(sent, t), [])
        assert ea.correct_any(f, 2)[0] == ea.EC_NO_SOLUTION, t
        assert table.correct(f)[0] == ea.EC_NO_SOLUTION, t


def test_df11_is_never_tried():
    rng = np.random.default_rng(6)
    for p in (5, 20, 31, 32, 55):
        sent = synth.make_frame(11, rng)
        f = dropped_frame(flip(sent, [p]), [])
        assert f.df == 11 and f.crc != 0
        st, bits, g = ea.correct_any(f, 2)
        assert (st, bits, bytes(g)) == (ea.EC_NOT_TRIED, (), bytes(f))


def test_a_flipped_df_field_is_not_a_candidate():
    sent = _df17(7)
    for p in range(5):
        f = dropped_frame(flip(sent, [p]), [])
        assert f.df != 17
        assert ea.correct_any(f, 2)[0] == ea.EC_NOT_TRIED
        f = dropped_frame(flip(sent, [p, 40]), [])
        assert ea.correct_any(f, 2)[0] == ea.EC_NOT_TRIED


def test_passed_and_zero_syndrome_frames_are_not_tried():
    sent = _df17(8)
    f = dropped_frame(sent, [])
    assert f.crc == 0
    assert ea.correct_any(f, 2)[0] == ea.EC_NOT_TRIED
    f = dropped_frame(flip(sent, [40]), [])
    assert ea.correct_any(f, 0)[0] == ea.EC_NOT_TRIED


def test_every_ec_outcome_followed_by_ec_any():
    rng = np.random.default_rng(9)
    sent = synth.make_frame(17, rng)
    cw = low_weight_codeword(112)
    k = 9
    cases = [
        # (errors, low-confidence set, ec status, ec_any status at M = 2)
        ([60], [30, 60, 100], eo.EC_FIXED, ea.EC_NOT_TRIED),                     # ec fixes it: not tried again
        ([25], list(range(20, 30)), eo.EC_TOO_MANY, ea.EC_FIXED),                # 10 > K
        ([25, 90], list(range(20, 44)), eo.EC_TOO_MANY, ea.EC_FIXED),            # saturated count of 24: still a candidate
        ([40], [12, 20, 33], eo.EC_NO_SOLUTION, ea.EC_FIXED),                    # error outside L
        ([20, 40], [12, 20, 33], eo.EC_NO_SOLUTION, ea.EC_FIXED),
        ([20, 40, 70], [12, 20, 33], eo.EC_NO_SOLUTION, ea.EC_NO_SOLUTION),      # three bits: dropped
        (cw[:2], sorted(cw + [min(set(range(5, 112)) - set(cw))]), eo.EC_AMBIGUOUS, ea.EC_FIXED),
        ([77], [], eo.EC_NO_SOLUTION, ea.EC_FIXED),                              # no low-confidence bits at all
    ]
    for err, L, want_ec, want_any in cases:
        f = dropped_frame(flip(sent, err), L)
        (st, flips), (st2, bits), g = ea.correct_both(f, k, 2)
        assert (st, st2) == (want_ec, want_any), (err, L, st, st2)
        if st == eo.EC_FIXED:
            assert tuple(flips) == tuple(err) and bits == ()
        if st2 == ea.EC_FIXED:
            assert bits == tuple(err) and flips == ()
        if eo.EC_FIXED in (st, st2):
            assert bytes(g.data)[:14] == sent and g.passed == 1 and g.crc == 0
        else:
            assert bytes(g) == bytes(f)
        assert g.numlowconf == f.numlowconf and bytes(g.lowconfbits) == bytes(f.lowconfbits)
        # ec off: ec_any alone sees the frame as the slicer left it
        (st, _), (st2, bits), _ = ea.correct_both(f, 0, 2)
        assert st == eo.EC_NOT_TRIED and st2 == (ea.EC_FIXED if len(err) <= 2 else ea.EC_NO_SOLUTION)
        assert ea.correct_both(f, k, 0)[1] == (ea.EC_NOT_TRIED, ())


def test_frame_binding_reads_the_ec_any_bytes():
    """include/airmodes_b200.h keeps amb_frame's declared tail (ec, ec_flips, pad_[4]) and puts the "ec_any" outcome and
    bits in pad_[0] and pad_[1..2] (AMB_FRAME_EC_ANY / AMB_FRAME_EC_ANY_BIT); _lib.Frame reads them as bytes 76 and 77-78
    through .ec_any / .ec_any_bits, and its numpy record layout is unchanged."""
    from gr_air_modes_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "airmodes_b200.h")).read()
    body = re.search(r"typedef struct amb_frame \{(.*?)\} amb_frame;", hdr, re.S).group(1)
    decl = [ln.split("/*")[0].strip() for ln in body.splitlines() if ln.split("/*")[0].strip()]
    assert decl[-4:] == ["uint8_t data[14];", "uint8_t ec;", "uint8_t ec_flips;", "uint8_t pad_[4];"]
    macros = dict(re.findall(r"#define (AMB_FRAME_EC_ANY\w*\([^)]*\))\s+(\S+)", hdr))
    assert macros == {"AMB_FRAME_EC_ANY(f)": "((f)->pad_[0])", "AMB_FRAME_EC_ANY_BIT(f, i)": "((f)->pad_[1"}, macros
    assert C.sizeof(_lib.Frame) == 80 and _lib.Frame.pad_.offset == 74
    names = np.dtype(_lib.Frame).names
    assert not {"ec", "ec_flips", "ec_any", "ec_any_bits"} & set(names) and names[-1] == "pad_"
    raw = bytearray(80)
    raw[74:79] = bytes([eo.EC_TOO_MANY, 0, ea.EC_FIXED, 20, 111])
    f = _lib.Frame.from_buffer_copy(bytes(raw))
    assert (f.ec, f.ec_flips, f.ec_any, f.ec_any_bits) == (eo.EC_TOO_MANY, 0, ea.EC_FIXED, (20, 111))
