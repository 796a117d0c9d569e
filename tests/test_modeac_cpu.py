"""The Mode A/C reply rules (include/airmodes_b200.h, option "modeac") pinned on their checker, tests/modeac_oracle.py:
planted replies of every code found at every supported rate, none in noise or in Mode S scenes, every comparison of the
rules at its boundary, the squawk and altitude against the reference's own decode_id / decode_alt, and the checker's
independence of how the stream is cut."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

from gr_air_modes_b200 import blocks, synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import modeac_oracle as mo  # noqa: E402
from helpers import load_golden  # noqa: E402

REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")
ALL = [(code, spi) for code in range(1 << 13) if not code & 0x40 for spi in (False, True)]   # 4096 codes x SPI


def oracle(port, iq, rate, **kw):
    return mo.run_iq(port, iq, rate, 7.0, **kw)


@pytest.mark.parametrize("rate,found_share,exact_share", [(4e6, 0.999, 0.985), (5e6, 0.999, 0.985), (8e6, 1.0, 1.0),
                                                           (10e6, 1.0, 1.0), (20e6, 1.0, 1.0)])
def test_every_code_with_and_without_spi_is_found(port, rate, found_share, exact_share):
    """8192 replies at 15-30 dB SNR, F1 at a fractional sample, 30 us apart. The F1 index lies within -1 .. +spc
    samples of the planted leading edge: the PMF peak of a 0.45 us pulse is the first sample whose spc-sample window
    covers it, at most 0.9 spc - 1 + 1 samples after the edge, and noise may move the rising-edge test by one sample
    either way. No reply gives more than one record, and no record lies elsewhere. At 8 Msps and above every reply is
    found with its exact code and SPI. At 4-5 Msps, with 2-2.5 samples per 0.45 us pulse, the fixed rounded offsets
    can sample a pulse on its flank: a framing pulse there loses the reply (1 in 8192 at 5 Msps, where o(20.3) is a
    tie rounded up), a code pulse there loses that bit (about 1 %, all at the low end of the SNR range)."""
    codes = np.array([c for c, _ in ALL])
    spis = np.array([s for _, s in ALL])
    rng = np.random.default_rng(int(rate))
    order = rng.permutation(len(ALL))
    n = int(len(ALL) * 57 * rate / 1e6) + 4096
    sc, planted = synth.make_modeac_scene(rate, n, len(ALL), 500 + int(rate / 1e6), codes=codes[order], spis=spis[order])
    got = oracle(port, sc.iq, rate)
    h = blocks.query_geometry(rate, 7.0, True).history - 1
    idx = np.array([r["sample_index"] - h for r in got])
    spc = rate / 2e6
    once = exact = 0
    for p in planted:
        k = np.flatnonzero((idx >= p.start - 1) & (idx <= p.start + spc))
        assert k.size <= 1, (p, idx[k])
        if k.size:
            r = got[int(k[0])]
            once += 1
            exact += r["code"] == p.code and r["spi"] == int(p.spi)
    assert len(got) == once >= found_share * len(planted)
    assert exact >= exact_share * len(planted)


@pytest.mark.parametrize("rate", [4e6, 8e6, 20e6])
def test_no_reply_in_noise(port, rate):
    rng = np.random.default_rng(17)
    iq = (rng.standard_normal(2 * 600_000) * 0.01).astype(np.float32)
    assert oracle(port, iq, rate) == []


def test_golden_mode_s_scenes_have_no_reply(port):
    _, scenes = load_golden()
    seen = 0
    for s, iq in scenes:
        if s["rate"] < 4e6 or not s["use_pmf"]:
            continue
        assert mo.run_iq(port, iq, s["rate"], s["threshold_db"]) == [], s["name"]
        seen += 1
    assert seen >= 4


@pytest.mark.parametrize("rate,pinned", [(4e6, 3), (8e6, 6), (20e6, 3)])
def test_fruit_scenes(port, rate, pinned):
    """make_scene's Mode S bursts give no reply. Its FRUIT pairs (two pulses 1-13 x 1.45 us apart) never form one
    alone, but 300 of them at random times put some pulse of one 20.3 us after a pulse of another, with nothing in
    the gaps between: to the rules that is a reply (code 0 or a few bits), as it is to any receiver. The count is
    pinned per scene."""
    n = 400_000
    assert oracle(port, synth.make_scene(rate, n, 150, 5).iq, rate) == []
    got = oracle(port, synth.make_scene(rate, n, 150, 5, fruit=300).iq, rate)
    assert len(got) == pinned
    assert all(bin(r["code"]).count("1") <= 3 for r in got)


# ---- every comparison at its boundary: bb / avg arrays built so that one comparison sits on its edge ---------------
RATE = 8_000_000
G = mo.geometry(RATE)
THR = np.float32(blocks.query_geometry(RATE, 7.0, True).threshold)
I0 = 300


def reply_arrays(code=0b1010101010101 & ~0x40, spi=True, level=np.float32(1.0), floor=np.float32(0.01)):
    """bb / avg of one clean reply at I0: every pulse one sample of `level`, flat floor."""
    n = I0 + 400
    bb = np.full(n, np.float32(1e-4), np.float32)
    avg = np.full(n, floor, np.float32)
    ons = [0] + [G["slot"][k] for k in range(1, 14) if (code >> (13 - k)) & 1] + [G["slot"][14]] + ([G["spi"]] if spi else [])
    for o in ons:
        bb[I0 + o] = level
    return bb, avg


def found(bb, avg):
    ev = mo.evaluate(bb, avg, RATE, THR)
    return bool(ev["reply"][I0]), ev


def up(x):
    return np.nextafter(np.float32(x), np.float32(np.inf))


def down(x):
    return np.nextafter(np.float32(x), np.float32(-np.inf))


def test_clean_reply_decodes():
    code = 0b1010101010101 & ~0x40
    ok, ev = found(*reply_arrays(code))
    assert ok and ev["code"][I0] == code and ev["spi"][I0]


def test_rule1_threshold_edge():
    bb, avg = reply_arrays()
    lvl = np.float32(avg[I0] * THR)
    for v, want in ((lvl, False), (up(lvl), True)):
        b = bb.copy()
        b[I0] = v
        b[I0 + G["slot"][14]] = v
        assert found(b, avg)[1]["r12"][I0] == want


def test_rule1_peak_edges():
    bb, avg = reply_arrays()
    for before, after, want in ((down(1.0), np.float32(1.0), True), (np.float32(1.0), np.float32(0.5), False),
                                (np.float32(0.5), up(1.0), False), (np.float32(0.5), np.float32(1.0), True)):
        b = bb.copy()
        b[I0 - 1], b[I0 + 1] = before, after
        assert found(b, avg)[1]["r12"][I0] == want, (before, after)


def test_rule2_f2_edge():
    bb, avg = reply_arrays()
    lvl = np.float32(avg[I0] * THR)
    for v, want in ((down(lvl), False), (lvl, True)):
        b = bb.copy()
        b[I0 + G["slot"][14]] = v
        assert found(b, avg)[1]["r12"][I0] == want


def space_of(bb, avg):
    avgpeak = (bb[I0] + bb[I0 + G["slot"][14]]) / np.float32(2.0)
    return np.float32(avg[I0] + (avgpeak - avg[I0]) / THR)


@pytest.mark.parametrize("where", ["x"] + ["gap%d" % g for g in range(14)])
def test_rules_4_5_quiet_edges(where):
    bb, avg = reply_arrays()
    sp = space_of(bb, avg)
    o = G["slot"][7] if where == "x" else G["gap"][int(where[3:])]
    for v, want in ((sp, True), (up(sp), False)):
        b = bb.copy()
        b[I0 + o] = v
        assert found(b, avg)[0] == want


def test_rule4_framing_edges():
    bb, avg = reply_arrays(level=np.float32(0.2))
    clear = np.float32(np.float32(avg[I0] * THR) * THR)
    for v, want in ((clear, False), (up(clear), True)):
        b = bb.copy()
        b[I0 + G["slot"][14]] = v
        b[I0] = v
        assert found(b, avg)[1]["r15"][I0] == want
    # the weaker framing pulse against the space threshold of both
    bb, avg = reply_arrays()
    for f2 in (np.float32(0.25), np.float32(0.3)):
        b = bb.copy()
        b[I0 + G["slot"][14]] = f2
        sp = space_of(b, avg)
        assert found(b, avg)[1]["r15"][I0] == bool(f2 > sp)


@pytest.mark.parametrize("k", range(1, 14))
def test_rule6_code_and_spi_edges(k):
    if k == 7:
        return
    bb, avg = reply_arrays(code=0, spi=False)
    sp = space_of(bb, avg)
    for v, bit in ((sp, 0), (up(sp), 1)):
        b = bb.copy()
        b[I0 + G["slot"][k]] = v
        b[I0 + G["spi"]] = v
        ok, ev = found(b, avg)
        assert ok and ev["code"][I0] == bit << (13 - k) and ev["spi"][I0] == bool(bit)


def test_rule7_window_edge():
    """A start passing rules 1-5 exactly o(25.1) before drops the reply; one sample further it does not."""
    for d, want in ((G["back"], False), (G["back"] + 1, True)):
        bb, avg = reply_arrays(code=0, spi=False)
        j = I0 - d
        b = bb.copy()
        b[j] = np.float32(1.0)
        b[j + G["slot"][14]] = np.float32(1.0)
        ok, ev = found(b, avg)
        assert ev["r15"][j] and ok == want, d


def test_rule7_counts_dropped_starts_too():
    """Three starts each o(25.1) - 1 after the one before: the second is dropped by the first, the third by the dropped
    second."""
    d = G["back"] - 1
    n = I0 + 3 * d + 400
    bb = np.full(n, np.float32(1e-4), np.float32)
    avg = np.full(n, np.float32(0.01), np.float32)
    for s in (I0, I0 + d, I0 + 2 * d):
        bb[s] = bb[s + G["slot"][14]] = np.float32(1.0)
    ev = mo.evaluate(bb, avg, RATE, THR)
    assert ev["r15"][[I0, I0 + d, I0 + 2 * d]].all()
    assert list(np.flatnonzero(ev["reply"])) == [I0]


# ---- decoded fields -------------------------------------------------------------------------------------------------
def _reference_modules():
    if not os.path.exists(os.path.join(REF, "parse.py")):
        pytest.skip("the reference's python sources are not present")
    saved = {k: v for k, v in sys.modules.items() if k == "air_modes" or k.startswith("air_modes.")}
    pkg = types.ModuleType("air_modes")
    pkg.__path__ = []
    sys.modules["air_modes"] = pkg

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod
    try:
        exc = load("air_modes.exceptions", os.path.join(REF, "exceptions.py"))
        alt = load("air_modes.altitude", os.path.join(REF, "altitude.py"))
        mt = load("air_modes.modes_types", os.path.join(REF, "modes_types.py"))
        pkg.modes_report, pkg.stamp = mt.modes_report, mt.stamp
        parse = load("air_modes.parse", os.path.join(REF, "parse.py"))
        return exc, alt, parse
    finally:
        for k in [k for k in sys.modules if k == "air_modes" or k.startswith("air_modes.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_squawk_and_altitude_match_the_reference_for_every_code():
    exc, alt, parse = _reference_modules()
    for code in range(1 << 13):
        assert mo.decode_id(code) == parse.decode_id(code), code
        if code & 0x40:
            continue
        want = mo.altitude(code)
        if want == mo.NO_ALTITUDE:
            continue
        assert want == alt.decode_alt(code, True), code


def test_c_group_rule():
    valid = {0b001, 0b011, 0b010, 0b110, 0b100}
    n_alt = 0
    for code in range(1 << 13):
        if code & 0x40:
            continue
        has = mo.altitude(code) != mo.NO_ALTITUDE
        assert has == (not code & 0x10 and mo.c_group(code) in valid), code
        n_alt += has
        if has:
            assert -1200 <= mo.altitude(code) <= 126_700 and mo.altitude(code) % 100 == 0
    assert n_alt == 4096 // 2 * 5 // 8


def test_the_checker_does_not_depend_on_the_cut(port):
    rate = 4e6
    sc, _ = synth.make_modeac_scene(rate, 300_000, 300, 77, n_bursts=30)
    g = blocks.query_geometry(rate, 7.0, True)
    bb, avg = port.frontend(sc.iq, rate, True)
    whole = mo.replies(bb, avg, g.rate_int, g.threshold, g.history, chunk=bb.size)
    assert len(whole) >= 290
    for chunk in (97, 101, 4096, 65_537):
        assert mo.replies(bb, avg, g.rate_int, g.threshold, g.history, chunk=chunk) == whole
