"""Seeded message sets for the decoder option "opstatus" (tests/test_opstatus_*.py, tools/opstatus_yield.py). Frames come
from tests/decode_cases.py's encoders; the TC 31 and TC 29 ME words from the encoders here. Every generator returns
messages (hex, ecc, secs, frac) in time order; track_cases.frames_of() turns them into frames (every 97th one not
queued). Addresses stay below 2^15, so that the emulator's small pairing table holds every position squitter."""
from __future__ import annotations

import numpy as np

import decode_cases as dc
import local_cpr_cases as lc
import opstatus_oracle as oo

AIRBORNE_TC = (9, 10, 11, 12, 13, 14, 16, 17, 18)
SURFACE_TC = (5, 6, 7, 8)


def opstatus_me(sub, ver, cc=0, om=0, nica=0, nacp=0, gva=0, sil=0, baro=0, hrd=0, silsupp=0, nicc=None, lw=None,
                tail=0):
    """TC 31 ME word. For a surface message NIC-C (ME 20) and the length/width code (ME 21-24) override the low five
    capability-class bits when given; `tail` fills ME 56."""
    b = dc.Bits(56).put(1, 5, 31).put(6, 3, sub).put(9, 16, cc).put(25, 16, om).put(41, 3, ver).put(44, 1, nica) \
        .put(45, 4, nacp).put(49, 2, gva).put(51, 2, sil).put(53, 1, baro).put(54, 1, hrd).put(55, 1, silsupp) \
        .put(56, 1, tail)
    if nicc is not None:
        b.v &= ~(1 << (56 - 20))
        b.put(20, 1, nicc)
    if lw is not None:
        b.v &= ~(0xF << (56 - 24))
        b.put(21, 4, lw)
    return b.v


def target_state_me(sub=1, silsupp=0, alt_type=0, alt=0, baro=0, hdg_status=0, hdg=0, nacp=0, nicbaro=0, sil=0,
                    modes=0, tail=0):
    """TC 29 ME word, subtype `sub` (ME 6-7) with the version-2 layout; `tail` fills ME 55-56."""
    return dc.Bits(56).put(1, 5, 29).put(6, 2, sub).put(8, 1, silsupp).put(9, 1, alt_type).put(10, 11, alt) \
        .put(21, 9, baro).put(30, 1, hdg_status).put(31, 9, hdg).put(40, 4, nacp).put(44, 1, nicbaro) \
        .put(45, 2, sil).put(47, 8, modes).put(55, 2, tail).v


def position(aa, tc, nicb=0, rng=None, odd=0):
    """A DF17 position of type code `tc` with ME bit 8 = `nicb` (airborne; a surface position's ME 8 is movement)."""
    rng = rng or np.random.default_rng(aa)
    la, lo_ = int(rng.integers(0, 1 << 17)), int(rng.integers(0, 1 << 17))
    if tc <= 8:
        return dc.df17(aa, dc.me_surface(tc, int(rng.integers(0, 128)), 1, int(rng.integers(0, 128)), odd, la, lo_))
    return dc.df17(aa, dc.me_airborne(tc, dc.enc_alt12(int(rng.integers(0, 40000))), odd, la, lo_, saf=nicb))


def df18(aa, me):
    b = dc.Bits(88).put(1, 5, 18).put(6, 3, 0).put(9, 24, aa).put(33, 56, me)
    return dc.finish(b.bytes())


def _msgs(ev):
    ev.sort(key=lambda e: e[0])
    return [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc in ev]


def table_scene(seed=1):
    """Every row and every supplement combination of both tables, for versions 0, 1, 2 and no op status. Per address:
    a surface op status (NIC-A, NIC-C) and every surface type code; then an airborne op status with the same NIC-A and
    every airborne type code with NIC-B 0 and 1; then every surface type code again, now with an airborne writer later
    than the surface one."""
    rng = np.random.default_rng(seed)
    ev, aa, t = [], 0x100, 1.0
    for ver in (None, 0, 1, 2):
        for nica in (0, 1):
            for nicc in (0, 1):
                if ver is None and (nica or nicc):
                    continue
                if ver is not None:
                    ev.append((t, *dc.df17(aa, opstatus_me(1, ver, cc=int(rng.integers(0, 1 << 16)), nica=nica,
                                                           nicc=nicc, nacp=9))))
                for tc in SURFACE_TC:
                    t += 0.1
                    ev.append((t, *position(aa, tc, rng=rng, odd=int(rng.integers(0, 2)))))
                t += 0.1
                if ver is not None:
                    ev.append((t, *dc.df17(aa, opstatus_me(0, ver, cc=int(rng.integers(0, 1 << 16)), nica=nica,
                                                           nacp=10))))
                for tc in AIRBORNE_TC:
                    for nicb in (0, 1):
                        t += 0.1
                        ev.append((t, *position(aa, tc, nicb, rng, odd=nicb)))
                for tc in SURFACE_TC:
                    t += 0.1
                    ev.append((t, *position(aa, tc, rng=rng)))
                aa += 1
                t += 1.0
    return _msgs(ev)


def fields_scene(seed=2):
    """Every field of both messages at 0 and at its maximum, the "no data" encodings, each mode bit alone; TC 31
    versions 3..7 and subtypes 2..7, TC 29 subtypes 0, 2, 3; TC 15; DF18 carrying TC 31 / 29 / a position."""
    rng = np.random.default_rng(seed)
    mes = []
    for sub in (0, 1):
        for ver in (0, 1, 2):
            mes.append(opstatus_me(sub, ver))
            mes.append(opstatus_me(sub, ver, cc=0xFFFF, om=0xFFFF, nica=1, nacp=15, gva=3, sil=3, baro=1, hrd=1,
                                   silsupp=1, tail=1))
            for name, top in (("cc", 0xFFFF), ("om", 0xFFFF), ("nica", 1), ("nacp", 15), ("gva", 3), ("sil", 3),
                              ("baro", 1), ("hrd", 1), ("silsupp", 1)):
                mes.append(opstatus_me(sub, ver, **{name: top}))
            if sub:
                for nicc, lw in ((1, 0), (0, 15), (1, 15)):
                    mes.append(opstatus_me(sub, ver, nicc=nicc, lw=lw))
    for ver in range(3, 8):
        mes += [opstatus_me(0, ver, nica=1), opstatus_me(1, ver, nicc=1)]
    for sub in range(2, 8):
        mes += [opstatus_me(sub, 2, nica=1), opstatus_me(sub, 1)]
    mes.append(target_state_me())
    mes.append(target_state_me(silsupp=1, alt_type=1, alt=2047, baro=511, hdg_status=1, hdg=511, nacp=15, nicbaro=1,
                               sil=3, modes=0xFF, tail=3))
    for name, top in (("silsupp", 1), ("alt_type", 1), ("alt", 2047), ("alt", 1), ("baro", 511), ("baro", 1),
                      ("hdg_status", 1), ("hdg", 511), ("nacp", 15), ("nicbaro", 1), ("sil", 3)):
        mes.append(target_state_me(**{name: top}))
    for j in range(8):
        mes.append(target_state_me(modes=1 << j))
    for sub in (0, 2, 3):
        mes.append(target_state_me(sub=sub, alt=100, modes=0xFF))
    ev, t = [], 1.0
    for k, me in enumerate(mes):
        ev.append((t, *dc.df17(0x200 + k % 5, me)))
        t += 0.01
    for k in range(20):                                         # TC 15 and DF18 are not touched
        aa = 0x210 + k % 3
        ev.append((t, *dc.df17(aa, dc.me_airborne(15, 0, 0, int(rng.integers(0, 1 << 17)), 0))))
        ev.append((t + 0.001, *df18(aa, opstatus_me(0, 2, nica=1))))
        ev.append((t + 0.002, *df18(aa, target_state_me(alt=100))))
        ev.append((t + 0.003, *df18(aa, dc.me_airborne(11, 0, 0, 5, 5))))
        ev.append((t + 0.004, *position(aa, 11, 1, rng)))       # the DF18 op status did not count
        t += 0.01
    return _msgs(ev)


def age_scene(S=30, seed=3):
    """Per address: a writer exactly S old (counts), one 2^-40 s older (does not), one stamped later than the position
    (an earlier stream: does not, and nothing older is looked for), no writer at all; a surface writer exactly S old
    beside an airborne writer within S, and one past S."""
    rng = np.random.default_rng(seed)
    eps = 2.0 ** -40
    ev = []
    aa = 0x300
    for dt in (float(S), float(S) + eps, 1.0):
        for tc in (11, 7, 8):
            t0 = 10.5 + (aa - 0x300) * 1000.0
            ev.append((t0, *dc.df17(aa, opstatus_me(1, 2, nica=1, nicc=1))))
            ev.append((t0 + dt, *position(aa, tc, 1, rng)))
            aa += 1
    for tc in (11, 7, 8):                                       # the surface writer's age alone
        for dt in (float(S), float(S) + eps):
            t0 = 10.5 + (aa - 0x300) * 1000.0
            ev.append((t0, *dc.df17(aa, opstatus_me(1, 2, nica=1, nicc=1))))
            ev.append((t0 + dt - 1.0, *dc.df17(aa, opstatus_me(0, 2, nica=1))))
            ev.append((t0 + dt, *position(aa, tc, 1, rng)))
            aa += 1
    for tc in (11, 8):                                          # absent writer
        ev.append((5000.0 + aa, *position(aa, tc, 1, rng)))
        aa += 1
    msgs = _msgs(ev)
    # stamped later: the writer comes first in the stream but carries a later time than the position after it
    for tc in (11, 8):
        fr, ecc = dc.df17(aa, opstatus_me(1, 2, nica=1, nicc=1))
        msgs.append((fr.hex(), ecc, 90001, 0.5))
        fr, ecc = position(aa, tc, 1, rng)
        msgs.append((fr.hex(), ecc, 90001, 0.25))
        aa += 1
    return msgs


def _random_me(rng, aa_kind):
    r = rng.random()
    if r < 0.2:
        return opstatus_me(int(rng.integers(0, 2)), int(rng.choice([0, 1, 2, 2, 2, 3])), nica=int(rng.integers(0, 2)),
                           nicc=int(rng.integers(0, 2)), nacp=int(rng.integers(0, 16)), sil=int(rng.integers(0, 4)))
    if r < 0.3:
        return target_state_me(sub=int(rng.choice([1, 1, 1, 0])), alt=int(rng.integers(0, 2048)),
                               modes=int(rng.integers(0, 256)))
    return None


def bucket_scene(n_aircraft=32, n=3000, seed=9):
    """n_aircraft addresses sharing one bucket of the partition, each with op status of every kind and positions."""
    rng = np.random.default_rng(seed)
    addrs = lc.same_bucket_addresses(n_aircraft)
    ev = []
    for k in range(n):
        aa = int(addrs[k % n_aircraft])
        t = 0.02 * k
        me = _random_me(rng, 0)
        if me is not None:
            ev.append((t, *dc.df17(aa, me)))
        else:
            ev.append((t, *position(aa, int(rng.choice(AIRBORNE_TC + SURFACE_TC)), int(rng.integers(0, 2)), rng)))
    return _msgs(ev)


def burst_scene(seed=4):
    """One address with far more than 32 records back to back, so that lanes take an earlier lane's op status, the
    table's, or none; a second address now and then; gaps longer than S = 3."""
    rng = np.random.default_rng(seed)
    aa, bb = 0x2BCD, 0x2BCE
    ev, t = [], 10.0
    for k in range(240):
        who = bb if rng.random() < 0.1 else aa
        me = _random_me(rng, 0)
        if me is not None:
            ev.append((t, *dc.df17(who, me)))
        else:
            ev.append((t, *position(who, int(rng.choice(AIRBORNE_TC + SURFACE_TC)), int(rng.integers(0, 2)), rng)))
        if k % 70 == 69:
            t += 5.0                                            # older than S = 3
        t += float(rng.choice([0.0, 0.001, 0.01]))
    return _msgs(ev)


def fleet_scene(n_aircraft=300, seconds=60.0, seed=17, versions=(0, 1, 2, 2, 2), surface_share=0.15):
    """n_aircraft aircraft of ADS-B versions drawn from `versions` (None: no op status sent) over `seconds`: positions
    and velocities at about 2 Hz each, op status about every 2.5 s (version 2 and 1 on the ground also send the surface
    subtype), target state (version 2) about every 1.25 s. Each aircraft keeps one position type code, NIC-A, NIC-B and
    NIC-C. Returns (msgs, truth): truth[k] = (kind, version, tc, nica, nicb, nicc) with kind "opstatus",
    "target_state", "position" or None."""
    rng = np.random.default_rng(seed)
    addrs = rng.choice(np.arange(1, 1 << 15), n_aircraft, replace=False)
    ev = []
    for aa in addrs:
        aa = int(aa)
        ver = versions[int(rng.integers(0, len(versions)))]
        surface = rng.random() < surface_share
        tc = int(rng.choice(SURFACE_TC if surface else AIRBORNE_TC))
        nica, nicb, nicc = int(rng.integers(0, 2)), int(rng.integers(0, 2)), int(rng.integers(0, 2))
        t0 = float(rng.uniform(0, 5))
        t = t0
        while t < seconds:
            r = rng.random()
            if r < 0.41:
                ev.append((t, *position(aa, tc, nicb, rng, odd=int(rng.integers(0, 2))), ("position", ver, tc, nica,
                                                                                         nicb, nicc)))
            elif r < 0.82:
                me = dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(15, 10, 200).put(26, 10, 300).put(38, 9, 1).v
                ev.append((t, *dc.df17(aa, me), None))
            elif r < 0.90 and ver is not None:
                me = opstatus_me(1 if surface else 0, ver, cc=int(rng.integers(0, 1 << 16)), nica=nica, nicc=nicc,
                                 nacp=9, sil=3)
                ev.append((t, *dc.df17(aa, me), ("opstatus", ver, tc, nica, nicb, nicc)))
            elif ver == 2:
                me = target_state_me(alt=int(rng.integers(1, 2048)), baro=int(rng.integers(1, 512)), hdg_status=1,
                                     hdg=int(rng.integers(0, 512)), nacp=9, sil=3, modes=int(rng.integers(0, 256)))
                ev.append((t, *dc.df17(aa, me), ("target_state", ver, tc, nica, nicb, nicc)))
            t += float(rng.exponential(0.2))
    ev.sort(key=lambda e: e[0])
    msgs = [(fr.hex(), ecc, int(t), float(np.float64(t - int(t)))) for t, fr, ecc, _ in ev]
    return msgs, [e[3] for e in ev]


def expected_nic(version, tc, nica, nicb, nicc):
    """The (outcome, NIC or NUCp, Rc) a position of a fleet aircraft must get once its op status counts."""
    if version is None or version == 0:
        return oo.NUC, oo.NUCP[tc], None
    if version == 1:
        nicb, nicc = nica, 0
        if tc == 8:
            return oo.NIC, 0, None
    nic, rc = oo.lookup(tc, nica, nicc if tc <= 8 else nicb)
    return oo.NIC, nic, rc


def scenes():
    """(name, msgs, S) for the equality tests."""
    yield "table", table_scene(), 30
    yield "fields", fields_scene(), 30
    yield "age", age_scene(S=30), 30
    yield "bucket", bucket_scene(), 5
    yield "burst", burst_scene(), 3
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    yield "case14", lc.remap_addresses(msgs), 10
