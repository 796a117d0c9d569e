"""DF17 correction by at most M bits anywhere (option "ec_any") on the device: the scenarios of
tests/test_ec_any_simt.py, time-sharded spans, the device-side drain and the batch decoder, and a 2^24-sample dense
scene with garbled squitters and FRUIT - against the oracle plus the brute-force checkers of tests/ec_oracle.py and
tests/ec_any_oracle.py. Need an H100."""
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import shard, synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_any_cases as eac  # noqa: E402
import ec_any_oracle as ea  # noqa: E402
import ec_cases as ecc  # noqa: E402
import ec_oracle as eo  # noqa: E402

pytestmark = pytest.mark.gpu

RATE = 4e6


@pytest.fixture(scope="module")
def scene():
    return eac.any_scene(RATE, 400_000, 60, seed=17)


@pytest.mark.parametrize("k,m", [(0, 1), (0, 2), (ecc.K, 1), (ecc.K, 2)])
def test_split_form_slicer(port, k, m):
    statuses = eac.run_slicer_packets(port, k, m)
    anys = [s[1] for s in statuses]
    assert anys.count(ea.EC_FIXED) >= (5 if m == 1 else 14), statuses
    assert ea.EC_NO_SOLUTION in anys and ea.EC_NOT_TRIED in anys


@pytest.mark.parametrize("rate", [4e6, 10e6])
def test_fused_chain_one_shot_and_chunked(port, rate):
    iq, _ = eac.any_scene(rate, int(100_000 * rate / 2e6), 40, seed=int(rate / 1e6) + 20)
    msgs, frames, st = eac.run_chain(iq, rate, 0, eac.M)
    _, statuses = eac.check_chain(port, iq, rate, frames, msgs, 0, eac.M)
    fixed = eac.n_fixed(statuses)
    assert fixed >= 15 and st.ec_fixed == fixed and st.frames_passed == sum(f.passed for f in frames)
    n = iq.size // 2
    rng = np.random.default_rng(6)
    for resolver in (0, 1):
        chunks = [int(x) for x in rng.integers(1, n // 3, 4)] + [1, 511, 513, 65536]
        msgs2, frames2, _ = eac.run_chain(iq, rate, 0, eac.M, chunks=chunks, resolver=resolver)
        assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def test_both_options_on(port):
    iq, _ = eac.any_scene(RATE, 400_000, 60, seed=18, wrong_max=2)
    msgs, frames, st = eac.run_chain(iq, RATE, ecc.K, eac.M)
    _, statuses = eac.check_chain(port, iq, RATE, frames, msgs, ecc.K, eac.M)
    assert st.ec_fixed == eac.n_fixed(statuses)
    assert sum(s[0] == eo.EC_FIXED for s in statuses) >= 10 and sum(s[1] == ea.EC_FIXED for s in statuses) >= 10


def test_off_is_byte_identical_and_option_range(port, scene):
    iq, _ = scene
    msgs0, frames0, st0 = ecc.run_chain(iq, RATE, 0)
    msgs1, frames1, st1 = eac.run_chain(iq, RATE, 0, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert all(bytes(f.pad_) == b"\0" * 6 for f in frames0) and st0.ec_fixed == 0
    assert msgs0 == port.run_iq(iq, RATE, 7.0, True, co.MA_CANONICAL).msgs
    assert st1.kernel_launches == st0.kernel_launches
    # ec alone: what it made before ec_any existed, with one more launch per call
    msgs_k, frames_k, st_k = ecc.run_chain(iq, RATE, ecc.K)
    msgs_k1, frames_k1, st_k1 = eac.run_chain(iq, RATE, ecc.K, 0, set_zero_first=True)
    assert msgs_k1 == msgs_k and [bytes(f) for f in frames_k1] == [bytes(f) for f in frames_k]
    assert all(bytes(f.pad_)[2:] == b"\0" * 4 for f in frames_k)
    assert st_k.kernel_launches == st0.kernel_launches + 1 == st_k1.kernel_launches
    _, _, st_on = eac.run_chain(iq, RATE, ecc.K, eac.M)
    assert st_on.kernel_launches == st0.kernel_launches + 1
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True)
    for bad in (-1, 3):
        with pytest.raises(RuntimeError):
            rx.set_ec_any(bad)
    rx.close()


def _sharded_chain(iq, plan, opts):
    q = am.msg_queue()
    rxs = [am.rx_path(RATE, 7.0, q, use_pmf=True, **opts) for _ in plan]
    for rx, sp in zip(rxs, plan):
        rx.defer_resolve(True)
        rx.seek(sp.first_sample, sp.first_decision)
        rx.process(iq[2 * sp.first_sample: 2 * sp.end], flush=sp.flush, collect=False)
    frames, state, queued = [], (0, 0), 0
    for rx, sp in zip(rxs, plan):
        rx.resolve(state)
        if not sp.flush:
            state = rx.walk_state()
        rx._slicer._first = queued == 0
        queued += rx.drain()
        frames += rx.frames
    for rx in rxs:
        rx.close()
    return q.strings(), frames


def _sharded_speculative(iq, plan, opts):
    qs = [am.msg_queue() for _ in plan]
    rxs = [am.rx_path(RATE, 7.0, q, use_pmf=True, **opts) for q in qs]
    last = len(plan) - 1
    mines = []
    for rank, (rx, sp) in enumerate(zip(rxs, plan)):
        rx.defer_resolve(True)
        rx.seek(sp.first_sample, sp.first_decision)
        rx.process(iq[2 * sp.first_sample: 2 * sp.end], flush=sp.flush, collect=False)
        mine = [0] * 6
        if rank < last:
            rx.resolve(None)
            s = rx.walk_summary()
            mine = [s.pos, s.p, s.first_real, s.first_packet, s.exact_span, s.frames_passed]
        mines.append(mine)
    entries, queued, bad = shard.compose_entries(plan, mines)
    frames, handed = [], None
    for rank, (rx, sp) in enumerate(zip(rxs, plan)):
        if rank < bad:
            qd = queued[rank]
        else:
            if rank == bad:
                (pos, p), qd = entries[rank], queued[rank]
            else:
                pos, p, qd = handed
            rx.resolve((pos, p))
        rx._slicer._first = qd == 0
        if rank >= bad and not sp.flush:
            state = rx.walk_state()
            n = rx.drain()
            handed = state + (qd + n,)
        else:
            rx.drain()
        frames += rx.frames
        rx.close()
    return [m for q in qs for m in q.strings()], frames


def test_time_sharded_equals_one_shot(scene):
    iq, _ = scene
    n = iq.size // 2
    msgs, frames, _ = eac.run_chain(iq, RATE, 0, eac.M)
    passed = [f for f in frames if f.passed]
    assert passed[0].ec_any == ea.EC_FIXED                # the stream's first message is a corrected frame
    geo = am.query_geometry(RATE, 7.0, True)
    idx = [int(f.sample_index) for f in frames]
    fixed_idx = [int(f.sample_index) for f in frames if f.ec_any == ea.EC_FIXED]
    plans = [shard.time_shard_plan(n, s, geo) for s in (2, 3)]
    plans.append(shard.time_shard_plan(n, 2, geo, boundaries=[fixed_idx[0] + 3]))             # right after the first fix
    plans.append(shard.time_shard_plan(n, 3, geo, boundaries=[fixed_idx[0] + 1, fixed_idx[len(fixed_idx) // 2] + 2]))
    for plan in plans:
        for fn in (_sharded_chain, _sharded_speculative):
            m, f = fn(iq, plan, dict(ec_any=eac.M))
            assert [int(x.sample_index) for x in f] == idx, (fn.__name__, plan)
            assert m == msgs and [bytes(x) for x in f] == [bytes(x) for x in frames], (fn.__name__, plan)


def test_drain_device_and_batch_decoder(port, scene):
    import torch
    from gr_air_modes_b200 import decode
    from oracle import decode_oracle as do
    iq, _ = scene
    msgs, frames, _ = eac.run_chain(iq, RATE, 0, eac.M)
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ec_any=eac.M)
    dev = torch.from_numpy(iq).cuda()
    n = iq.size // 2
    for a, b in ((0, 100_000), (100_000, 250_001), (250_001, n)):
        rx.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx.drain_device()
    rx.close()
    assert fr.cpu().numpy().tobytes() == b"".join(bytes(f) for f in frames)
    d = decode.batch_decoder(None)
    out = d.decode_device(fr).cpu().numpy().view(decode.FIELDS_DTYPE)
    d.close()
    fixed = [i for i, f in enumerate(frames) if f.ec_any == ea.EC_FIXED]
    assert len(fixed) >= 15
    fmsgs = [m for m, f in zip(msgs, [f for f in frames if f.passed]) if f.ec_any == ea.EC_FIXED]
    want = do.decode_batch([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in fmsgs], None)
    assert len(want) == len(fixed)
    for i, w in zip(fixed, want):
        g = decode.record_to_dict(out[i])
        assert (g["df"], g["icao"], g["status"], g["altitude"], g["bds"]) == (w["df"], w["icao"], w["status"], w["altitude"], w["bds"])


def test_dense_garbled_scene_with_fruit(port):
    """configs[4]'s traffic model (10^4 bursts/s, 20 % of them garbled by 1-5 bits before modulation, FRUIT) on 2^24
    samples; every frame is checked, with the checker's syndrome table (equal to its brute force, test_ec_any_cpu)."""
    import torch
    n, seed = 1 << 24, 5
    nb = int(10_000 * n / RATE)
    iq_dev, _, _ = synth.make_scene_device(RATE, n, nb, seed, torch.device("cuda", 0), snr_db=(4.0, 30.0),
                                           garble_frac=0.2, fruit=nb // 4)
    want = port.run_iq(iq_dev.cpu().numpy(), RATE, 7.0, True, co.MA_CANONICAL)
    table = ea.SyndromeTable(eac.M)
    for k in (0, 8):
        q = am.msg_queue()
        rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ec=k, ec_any=eac.M)
        rx.process(iq_dev, flush=True)
        frames, msgs, st = list(rx.frames), q.strings(), rx.stats()
        rx.close()
        assert [f.sample_index for f in frames] == [int(x) for x in want.index]
        statuses = eac.check_frames(frames, want.frames, k, eac.M, table)
        assert msgs == ea.merged_messages(port, want.frames, k, eac.M, table=table)
        n_any = sum(s[1] == ea.EC_FIXED for s in statuses)
        assert n_any >= 200 and st.ec_fixed == eac.n_fixed(statuses)
