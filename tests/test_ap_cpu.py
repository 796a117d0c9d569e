"""Address/parity check (option "ap_filter"): the checker of tests/ap_oracle.py on constructed frame sequences, and a
restatement of the device algorithm (amb_ap_* in amb_kernels.cu: buckets by address hash, per-bucket sort, a chunked
max-scan over confirmer positions with a carry, a table of the latest confirmer across calls) against that brute-force
checker on random sequences. No GPU needed."""
import os
import sys

import numpy as np

from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ap_oracle as apo  # noqa: E402
import ec_oracle as eo  # noqa: E402

RATE_INT = 4_000_000


def frame(si, df, addr=0, passed=1, crc=0):
    f = co.Frame()
    f.index, f.df, f.passed, f.crc = si, df, passed, crc
    f.nbits = 112 if df in (16, 17, 20, 21) else 56
    f.data[0] = df << 3
    f.data[1], f.data[2], f.data[3] = (addr >> 16) & 0xFF, (addr >> 8) & 0xFF, addr & 0xFF
    return f


def outcome(frames, s=1, k=0):
    return [(ap, g.passed) for _, _, ap, g in apo.apply(frames, k, 0, s, RATE_INT)]


A, B = 0x4840D6, 0x3C6586


def test_window_edges():
    w = 1 * RATE_INT
    fs = [frame(1000, 17, A), frame(1000 + w, 4, passed=1, crc=A), frame(1001 + w, 20, passed=1, crc=A)]
    assert outcome(fs) == [(0, 1), (apo.AP_KNOWN, 1), (apo.AP_UNKNOWN, 0)]
    # a confirmer after its subject does not count
    fs = [frame(500, 5, crc=B), frame(900, 11, B)]
    assert outcome(fs) == [(apo.AP_UNKNOWN, 0), (0, 1)]
    assert outcome([frame(10, 17, A), frame(20, 0, crc=A)], s=0) == [(0, 1), (0, 1)]        # off: nothing checked


def test_fixed_frames_do_not_confirm():
    f = frame(100, 17, A)
    g = frame(200, 21, crc=A)
    assert outcome([f, g]) == [(0, 1), (apo.AP_KNOWN, 1)]
    items = [(100, *apo.classify(f, eo.EC_FIXED)), (200, *apo.classify(g))]
    assert apo.check(items, 1, RATE_INT) == [apo.AP_NOT_CHECKED, apo.AP_UNKNOWN]
    items = [(100, *apo.classify(f, eo.EC_NOT_TRIED, eo.EC_FIXED)), (200, *apo.classify(g))]
    assert apo.check(items, 1, RATE_INT) == [apo.AP_NOT_CHECKED, apo.AP_UNKNOWN]


def test_iisi_subjects():
    conf = frame(100, 11, A)
    assert outcome([conf, frame(200, 11, A, passed=0, crc=0x7F)]) == [(0, 1), (apo.AP_KNOWN, 1)]
    assert outcome([conf, frame(200, 11, A, passed=0, crc=0x80)]) == [(0, 1), (0, 0)]          # not an II/SI code
    assert outcome([frame(200, 11, A, passed=0, crc=0x05)]) == [(apo.AP_UNKNOWN, 0)]           # unknown: stays dropped
    assert outcome([frame(200, 17, A, passed=0, crc=0x05)]) == [(0, 0)]                        # DF17: never a subject
    # an accepted II/SI reply does not confirm its address for later subjects
    fs = [frame(100, 17, A), frame(200, 11, B, passed=0, crc=3), frame(300, 4, crc=B)]
    assert outcome(fs) == [(0, 1), (apo.AP_UNKNOWN, 0), (apo.AP_UNKNOWN, 0)]
    fs = [frame(100, 17, B), frame(200, 11, B, passed=0, crc=3), frame(300, 4, crc=B)]
    assert outcome(fs) == [(0, 1), (apo.AP_KNOWN, 1), (apo.AP_KNOWN, 1)]


def test_undefined_dfs_are_ap_subjects():
    for df in (1, 2, 3, 6, 7, 8, 9, 10, 12, 15, 18, 19, 22, 24, 31):
        assert outcome([frame(100, 17, A), frame(200, df, crc=A), frame(300, df, crc=B)]) == \
            [(0, 1), (apo.AP_KNOWN, 1), (apo.AP_UNKNOWN, 0)], df


# ---- the device algorithm, restated ----------------------------------------------------------------------------------
def bucketed(calls, window, n_buckets, tile):
    """calls: per call a list of (si, kind, addr) in work-list order (any order inside a call; calls ascending). Returns
    {si: AP_*} for every subject, the way amb_ap_resolve_kernel decides."""
    last = {}
    out = {}
    for items in calls:
        buckets = [[] for _ in range(n_buckets)]
        for si, kind, addr in items:
            if kind != apo.NONE:
                buckets[(addr * 0x9E3779B1 & 0xFFFFFFFF) % n_buckets].append((addr, si, kind))
        for e in buckets:
            e.sort()
            carry = -1
            for c0 in range(0, len(e), tile):
                chunk = e[c0: c0 + tile]
                conf = np.array([c0 + i if x[2] == apo.CONF else -1 for i, x in enumerate(chunk)])
                incl = np.maximum.accumulate(np.maximum(conf, carry))
                for i, (addr, si, kind) in enumerate(chunk):
                    if kind == apo.CONF:
                        continue
                    p = incl[i]
                    g1 = e[p][1] + 1 if p >= 0 and e[p][0] == addr else last.get(addr, 0)
                    out[si] = apo.AP_KNOWN if g1 and si + 1 - g1 <= window else apo.AP_UNKNOWN
                for i, (addr, si, kind) in enumerate(chunk):
                    q = c0 + i
                    run_end = q + 1 == len(e) or e[q + 1][0] != addr
                    p = incl[i]
                    if run_end and p >= 0 and e[p][0] == addr:
                        last[addr] = e[p][1] + 1
                carry = int(incl[-1])
    return out


def test_bucketed_algorithm_equals_brute_force():
    rng = np.random.default_rng(7)
    for t in range(10_000):
        n = int(rng.integers(1, 60))
        n_addr = int(rng.integers(1, 6)) if t % 3 else int(rng.integers(1, 40))
        pool = rng.integers(0, 1 << 24, n_addr)
        p = rng.dirichlet(np.full(n_addr, 0.3 if t % 2 else 3.0))      # skewed and even address mixes
        si = np.sort(rng.choice(10_000, n, replace=False)).astype(np.int64) + 1
        kind = rng.choice([apo.NONE, apo.CONF, apo.SUBJECT, apo.IISI], n, p=[0.1, 0.4, 0.35, 0.15])
        addr = pool[rng.choice(n_addr, n, p=p)]
        items = [(int(a), int(k), int(b)) for a, k, b in zip(si, kind, addr)]
        window = int(rng.integers(1, 3000))
        cuts = np.sort(rng.choice(np.arange(1, n + 1), min(n, int(rng.integers(0, 4))), replace=False))
        calls = [list(c) for c in np.split(np.array(items, dtype=object), cuts) if len(c)]
        for c in calls:
            rng.shuffle(c)
        got = bucketed([[tuple(x) for x in c] for c in calls], window, int(rng.choice([1, 2, 2048])),
                       int(rng.choice([2, 4, 256])))
        want = apo.check(items, 1, window)
        for (s, k, _), w in zip(items, want):
            assert (got.get(s, apo.AP_NOT_CHECKED) if k not in (apo.NONE, apo.CONF) else apo.AP_NOT_CHECKED) == w, t
