"""Error correction (option "ec", DESIGN.md section 0), CPU only: the brute-force checker of tests/ec_oracle.py on
constructed packets - every outcome - and a numpy restatement of the device's GF(2) elimination against brute force."""
import os
import sys

import numpy as np
import pytest

from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_oracle as eo  # noqa: E402


def bit_syndromes(nbits):
    """Syndrome of a packet that is all zero but bit p, for every p (the CRC is linear: syndromes add by XOR)."""
    rows = np.zeros((nbits, nbits // 8), np.uint8)
    for p in range(nbits):
        rows[p, p // 8] = 0x80 >> (p % 8)
    return eo.syndromes(rows, nbits).astype(np.uint32)


SYN = {56: bit_syndromes(56), 112: bit_syndromes(112)}


def flip(data: bytes, positions) -> bytes:
    d = bytearray(data)
    for p in positions:
        d[p // 8] ^= 0x80 >> (p % 8)
    return bytes(d)


def dropped_frame(payload: bytes, lowconf, numlowconf=None):
    """The frame the slicer makes of `payload` when it fails its CRC: passed 0, crc = syndrome (slicer_impl.cc:173-182)."""
    f = co.Frame()
    nbits = 8 * len(payload)
    f.nbits, f.df = nbits, payload[0] >> 3
    f.data[:len(payload)] = list(payload)
    f.crc = int(eo.syndromes(np.frombuffer(payload, np.uint8)[None, :], nbits)[0])
    f.passed = 0
    lc = sorted(lowconf)[:24]
    f.lowconfbits[:len(lc)] = lc
    f.numlowconf = len(lowconf) if numlowconf is None else numlowconf
    return f


def low_weight_codeword(nbits, lo=5):
    """Support of a lowest-weight codeword among positions >= lo: meet in the middle over the syndromes of all sets of
    up to 3 positions (4 for the short code, whose lightest codewords in 51 positions weigh more than 6): two disjoint
    sets with one syndrome form a codeword."""
    from itertools import combinations
    s = [int(x) for x in SYN[nbits]]
    seen, best = {}, None
    for r in range(1, 4 if nbits == 112 else 5):
        for sub in combinations(range(lo, nbits), r):
            x = 0
            for p in sub:
                x ^= s[p]
            for other in seen.get(x, ()):
                if not set(other) & set(sub) and (best is None or len(other) + r < len(best)):
                    best = sorted(other + sub)
            if len(seen.setdefault(x, [])) < 4:
                seen[x].append(sub)
    assert best is not None, "no light codeword"
    assert not int(np.bitwise_xor.reduce(SYN[nbits][best]))
    return best


@pytest.mark.parametrize("df", [11, 17])
def test_checker_finds_the_flipped_bits(df):
    rng = np.random.default_rng(100 + df)
    for trial in range(60):
        sent = synth.make_frame(df, rng)
        nbits = 8 * len(sent)
        size = int(rng.integers(1, 10 if df == 11 else 13))
        L = sorted(int(p) for p in rng.choice(np.arange(5, nbits), size, replace=False))
        S = sorted(int(p) for p in rng.choice(L, int(rng.integers(1, size + 1)), replace=False))
        f = dropped_frame(flip(sent, S), L)
        st, flips, g = eo.correct(f, 23)
        assert (st, list(flips)) == (eo.EC_FIXED, S), (trial, L, S)
        assert bytes(g.data)[:nbits // 8] == sent and g.crc == 0 and g.passed == 1
        assert g.numlowconf == f.numlowconf and bytes(g.lowconfbits) == bytes(f.lowconfbits)
        assert eo.correct(f, 0)[0] == eo.EC_NOT_TRIED


def test_too_many_low_confidence_bits():
    rng = np.random.default_rng(7)
    sent = synth.make_frame(17, rng)
    for k in (1, 4, 8, 12, 23):
        L = list(range(10, 10 + k + 1))
        f = dropped_frame(flip(sent, L[:1]), L)
        assert eo.correct(f, k)[0] == eo.EC_TOO_MANY
        assert eo.correct(f, k + 1 if k < 23 else k)[0] == (eo.EC_FIXED if k < 23 else eo.EC_TOO_MANY)
    f = dropped_frame(flip(sent, [30]), list(range(20, 44)), numlowconf=24)   # saturated: positions unknown past 24
    assert eo.correct(f, 23)[0] == eo.EC_TOO_MANY


def test_no_solution_when_the_error_is_outside_the_search_set():
    rng = np.random.default_rng(8)
    for df in (11, 17):
        for _ in range(20):
            sent = synth.make_frame(df, rng)
            nbits = 8 * len(sent)
            L = sorted(int(p) for p in rng.choice(np.arange(5, nbits - 1), 6, replace=False))
            outside = int(rng.choice([p for p in range(5, nbits) if p not in L]))
            f = dropped_frame(flip(sent, [L[0], outside]), L)
            assert eo.correct(f, 8)[0] == eo.EC_NO_SOLUTION


@pytest.mark.parametrize("nbits", [56, 112])
def test_ambiguous_when_the_search_set_holds_a_codeword(nbits):
    cw = low_weight_codeword(nbits)
    rng = np.random.default_rng(nbits)
    sent = synth.make_frame(17 if nbits == 112 else 11, rng)
    # flipping cw[:2] or the rest of cw gives the same syndrome: two solutions
    f = dropped_frame(flip(sent, cw[:2]), cw + [min(set(range(5, nbits)) - set(cw))])
    assert eo.correct(f, 9)[0] == eo.EC_AMBIGUOUS


def test_df_bits_are_never_flipped():
    rng = np.random.default_rng(9)
    sent = synth.make_frame(17, rng)
    for p in range(5):
        f = dropped_frame(flip(sent, [p]), [p, 40, 77])        # flipping p back would fix it, but p is in the DF field
        assert eo.correct(f, 8)[0] == eo.EC_NO_SOLUTION
        f = dropped_frame(flip(sent, [40]), [p, 40, 77])
        st, flips, g = eo.correct(f, 8)
        assert st == eo.EC_FIXED and flips == (40,) and bytes(g.data)[:14] == sent


def test_frame_binding_reads_the_outcome_bytes():
    """_lib.Frame keeps the six tail bytes as one pad_ field (its numpy record layout is unchanged); .ec / .ec_flips
    read bytes 74 / 75, where include/airmodes_b200.h puts them right behind data[14]."""
    import ctypes as C
    import re
    from gr_air_modes_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "airmodes_b200.h")).read()
    body = re.search(r"typedef struct amb_frame \{(.*?)\} amb_frame;", hdr, re.S).group(1)
    decl = [ln.split("/*")[0].strip() for ln in body.splitlines() if ln.split("/*")[0].strip()]
    assert decl[-4:] == ["uint8_t data[14];", "uint8_t ec;", "uint8_t ec_flips;", "uint8_t pad_[4];"]
    assert C.sizeof(_lib.Frame) == 80 and _lib.Frame.pad_.offset == 74
    assert "ec" not in np.dtype(_lib.Frame).names and "ec_flips" not in np.dtype(_lib.Frame).names
    raw = bytearray(80)
    raw[74], raw[75] = eo.EC_FIXED, 3
    f = _lib.Frame.from_buffer_copy(bytes(raw))
    assert (f.ec, f.ec_flips) == (eo.EC_FIXED, 3)


def eliminate(vectors, syn):
    """The device's algorithm (amb_ec_kernel) in numpy: row i = (syndrome vector of L[i], subset mask); for bit 23..0 the
    lowest non-pivot row with the bit set becomes the pivot, is XORed into every other row with the bit and, when the
    target has it, into the target. Returns (status, solution mask)."""
    v = np.array(vectors, np.uint32)
    m = (np.uint32(1) << np.arange(v.size, dtype=np.uint32)).astype(np.uint32)
    pivot = np.zeros(v.size, bool)
    sol, rank = 0, 0
    for b in range(23, -1, -1):
        has = ((v >> b) & 1).astype(bool)
        rows = np.nonzero(has & ~pivot)[0]
        if rows.size == 0:
            continue
        p = rows[0]
        pv, pm = int(v[p]), int(m[p])
        pivot[p] = True
        other = has.copy()
        other[p] = False
        v[other] ^= np.uint32(pv)
        m[other] ^= np.uint32(pm)
        if (syn >> b) & 1:
            syn ^= pv
            sol ^= pm
        rank += 1
    if syn:
        return eo.EC_NO_SOLUTION, 0
    return (eo.EC_AMBIGUOUS, 0) if rank < v.size else (eo.EC_FIXED, sol)


def enumerate_subsets(vectors, syn):
    """Every non-empty subset's syndrome (by doubling) against the target."""
    acc = np.zeros(1, np.uint32)
    for x in vectors:
        acc = np.concatenate([acc, acc ^ np.uint32(x)])
    hits = np.nonzero(acc[1:] == syn)[0] + 1
    if hits.size == 0:
        return eo.EC_NO_SOLUTION, 0
    return (eo.EC_AMBIGUOUS, 0) if hits.size > 1 else (eo.EC_FIXED, int(hits[0]))


def test_elimination_equals_brute_force_on_random_systems():
    rng = np.random.default_rng(12)
    seen = {eo.EC_FIXED: 0, eo.EC_NO_SOLUTION: 0, eo.EC_AMBIGUOUS: 0}
    cws = {n: low_weight_codeword(n) for n in (56, 112)}
    for trial in range(10_000):
        nbits = 112 if trial % 3 else 56
        size = int(rng.integers(0, 15))
        L = [int(p) for p in rng.choice(np.arange(5, nbits), size, replace=False)]
        if trial % 5 == 0 and size >= 6:                     # plant a codeword: rank deficient
            L = list(dict.fromkeys(cws[nbits] + L))[:14]
        vec = [int(SYN[nbits][p]) for p in L]
        if trial % 2 and L:                                  # syndrome of a random non-empty subset: solvable
            pick = rng.random(len(L)) < 0.5
            pick[int(rng.integers(0, len(L)))] = True
            syn = int(np.bitwise_xor.reduce(np.array(vec, np.uint32)[pick]))
        else:
            syn = int(rng.integers(1, 1 << 24))
        if syn == 0:
            continue
        got, want = eliminate(vec, syn), enumerate_subsets(vec, syn)
        assert got == want, (trial, L, syn)
        seen[got[0]] += 1
    assert min(seen.values()) >= 100, seen
