"""Error correction (option "ec") on the device: the scenarios of tests/test_ec_simt.py, a 2^24-sample low-SNR scene,
time-sharded spans, the device-side drain and the batch decoder - against the oracle plus the brute-force checker of
tests/ec_oracle.py. Need an H100."""
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import shard, synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ec_cases as ecc  # noqa: E402
import ec_oracle as eo  # noqa: E402
from test_ec_cpu import low_weight_codeword  # noqa: E402

pytestmark = pytest.mark.gpu

RATE = 4e6


@pytest.fixture(scope="module")
def codewords():
    return {n: low_weight_codeword(n) for n in (56, 112)}


@pytest.fixture(scope="module")
def scene():
    return ecc.ec_scene(RATE, 400_000, 60, seed=7)


def fixed_of(frames):
    return [f.ec == eo.EC_FIXED for f in frames]


def test_split_form_slicer_every_outcome(port, codewords):
    statuses = ecc.run_slicer_packets(port, codewords)
    for s in (eo.EC_FIXED, eo.EC_TOO_MANY, eo.EC_NO_SOLUTION, eo.EC_AMBIGUOUS, eo.EC_NOT_TRIED):
        assert s in statuses, (s, statuses)


@pytest.mark.parametrize("rate", [4e6, 10e6])
def test_fused_chain_one_shot_and_chunked(port, rate):
    iq, _ = ecc.ec_scene(rate, int(100_000 * rate / 2e6), 40, seed=int(rate / 1e6))
    msgs, frames, st = ecc.run_chain(iq, rate, ecc.K)
    _, statuses = ecc.check_chain(port, iq, rate, frames, msgs, ecc.K)
    fixed = statuses.count(eo.EC_FIXED)
    assert fixed >= 15 and st.ec_fixed == fixed and st.frames_passed == sum(f.passed for f in frames)
    n = iq.size // 2
    rng = np.random.default_rng(4)
    for resolver in (0, 1):
        chunks = [int(x) for x in rng.integers(1, n // 3, 4)] + [1, 511, 513, 65536]
        msgs2, frames2, _ = ecc.run_chain(iq, rate, ecc.K, chunks=chunks, resolver=resolver)
        assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def test_off_is_byte_identical_and_option_range(port, scene):
    iq, _ = scene
    msgs0, frames0, st0 = ecc.run_chain(iq, RATE, 0)
    msgs1, frames1, st1 = ecc.run_chain(iq, RATE, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert all(f.ec == 0 and f.ec_flips == 0 for f in frames0) and st0.ec_fixed == 0
    assert msgs0 == port.run_iq(iq, RATE, 7.0, True, co.MA_CANONICAL).msgs
    _, _, st_on = ecc.run_chain(iq, RATE, ecc.K)
    assert st_on.kernel_launches == st0.kernel_launches + 1 and st1.kernel_launches == st0.kernel_launches
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True)
    for bad in (-1, 24):
        with pytest.raises(RuntimeError):
            rx.set_ec(bad)
    rx.close()


def test_low_snr_scene(port):
    import torch
    k = 8
    iq_dev, _, _ = synth.make_scene_device(RATE, 1 << 24, 6000, 41, torch.device("cuda", 0), snr_db=(3, 9))
    iq = iq_dev.cpu().numpy()
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ec=k)
    rx.process(iq_dev, flush=True)
    frames, msgs, st = list(rx.frames), q.strings(), rx.stats()
    rx.close()
    _, statuses = ecc.check_chain(port, iq, RATE, frames, msgs, k)
    fixed = statuses.count(eo.EC_FIXED)
    assert fixed >= 20 and st.ec_fixed == fixed
    for s in (eo.EC_TOO_MANY, eo.EC_NO_SOLUTION):
        assert s in statuses
    # EC on minus the fixed frames is the EC-off run exactly
    q0 = am.msg_queue()
    rx0 = am.rx_path(RATE, 7.0, q0, use_pmf=True)
    rx0.process(iq_dev, flush=True)
    off_frames, off_msgs = list(rx0.frames), q0.strings()
    rx0.close()
    assert len(off_frames) == len(frames)
    for a, b in zip(frames, off_frames):
        if a.ec == eo.EC_FIXED:
            assert not b.passed and b.crc != 0 and bytes(a.lowconfbits) == bytes(b.lowconfbits)
        else:
            assert bytes(a)[:74] == bytes(b)[:74]
    fixed_msg = [f.ec == eo.EC_FIXED for f in frames if f.passed]
    kept = [m for m, fx in zip(msgs, fixed_msg) if not fx]
    if fixed_msg[0]:                                  # off, the first kept message is the stream's first (precision 6)
        kept, off_msgs = kept[1:], off_msgs[1:]
    assert kept == off_msgs


def _sharded_chain(iq, plan, k):
    q = am.msg_queue()
    rxs = [am.rx_path(RATE, 7.0, q, use_pmf=True, ec=k) for _ in plan]
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


def _sharded_speculative(iq, plan, k):
    qs = [am.msg_queue() for _ in plan]
    rxs = [am.rx_path(RATE, 7.0, q, use_pmf=True, ec=k) for q in qs]
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
    msgs, frames, _ = ecc.run_chain(iq, RATE, ecc.K)
    passed = [f for f in frames if f.passed]
    assert passed[0].ec == eo.EC_FIXED                # the stream's first message is a corrected frame
    geo = am.query_geometry(RATE, 7.0, True)
    idx = [int(f.sample_index) for f in frames]
    fixed_idx = [int(f.sample_index) for f in frames if f.ec == eo.EC_FIXED]
    plans = [shard.time_shard_plan(n, s, geo) for s in (2, 3)]
    plans.append(shard.time_shard_plan(n, 2, geo, boundaries=[fixed_idx[0] + 3]))             # right after the first fix
    plans.append(shard.time_shard_plan(n, 3, geo, boundaries=[fixed_idx[0] + 1, fixed_idx[len(fixed_idx) // 2] + 2]))
    for plan in plans:
        for fn in (_sharded_chain, _sharded_speculative):
            m, f = fn(iq, plan, ecc.K)
            assert [int(x.sample_index) for x in f] == idx, (fn.__name__, plan)
            assert m == msgs and [bytes(x) for x in f] == [bytes(x) for x in frames], (fn.__name__, plan)


def test_drain_device_and_batch_decoder(port, scene):
    import torch
    from gr_air_modes_b200 import decode
    from oracle import decode_oracle as do
    iq, _ = scene
    msgs, frames, _ = ecc.run_chain(iq, RATE, ecc.K)
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ec=ecc.K)
    dev = torch.from_numpy(iq).cuda()
    n = iq.size // 2
    for a, b in ((0, 100_000), (100_000, 250_001), (250_001, n)):
        rx.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx.drain_device()
    rx.close()
    assert fr.cpu().numpy().tobytes() == b"".join(bytes(f) for f in frames)
    # the fixed frames decode like the oracle's decode of their corrected payloads
    d = decode.batch_decoder(None)
    out = d.decode_device(fr).cpu().numpy().view(decode.FIELDS_DTYPE)
    d.close()
    fixed = [i for i, f in enumerate(frames) if f.ec == eo.EC_FIXED]
    assert len(fixed) >= 15
    fmsgs = [m for m, f in zip(msgs, [f for f in frames if f.passed]) if f.ec == eo.EC_FIXED]
    want = do.decode_batch([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in fmsgs], None)
    assert len(want) == len(fixed)
    for i, w in zip(fixed, want):
        g = decode.record_to_dict(out[i])
        assert (g["df"], g["icao"], g["status"], g["altitude"], g["bds"]) == (w["df"], w["icao"], w["status"], w["altitude"], w["bds"])
