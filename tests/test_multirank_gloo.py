"""world_size-2 gloo run of the multi-GPU plumbing (fan-out from the ingest rank, max-over-ranks timing,
result gather) on CPU. The per-channel processing function is injected: here the CPU oracle stands in for
the CUDA chain, which is what the -m gpu tests and bench.py --gpus N exercise on real devices."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gr_air_modes_b200 import shard, synth


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port_no, n, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import cpu_oracle as co
    dev = torch.device("cpu")

    def make(ch):
        sc = synth.make_scene(4e6, n, 12, seed=100 + ch)
        return torch.from_numpy(sc.iq.copy()), [b.frame.hex() for b in sc.bursts]

    iq, sent = shard.fan_out(make, rank, world, dev, 2 * n)
    expect = synth.make_scene(4e6, n, 12, seed=100 + rank)
    assert np.array_equal(iq.numpy(), expect.iq)                  # each rank got ITS channel, bit for bit
    assert sent == [b.frame.hex() for b in expect.bursts]
    msgs = co.Port().run_iq(iq.numpy(), 4e6, 7.0, True, co.MA_SLIDING64).msgs
    counts = shard.gather_counts(len(msgs), world, dev)
    slowest = shard.max_over_ranks(1.0 + rank, world, dev)
    assert slowest == float(world)
    assert counts[rank] == len(msgs) and len(counts) == world
    ret[rank] = counts
    dist.barrier()
    dist.destroy_process_group()


def test_fan_out_and_gather_world2():
    world, n = 2, 120_000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), n, ret), nprocs=world, join=True)
    assert ret[0] == ret[1] and all(c > 0 for c in ret[0])


def test_channel_ownership():
    assert shard.channels_of(1, 4, 8) == [1, 5]
    assert sorted(sum((shard.channels_of(r, 3, 8) for r in range(3)), [])) == list(range(8))
    assert shard.max_over_ranks(3.5, 1, None) == 3.5 and shard.gather_counts(7, 1, None) == [7]


# ---- time-sharded single stream: plan + hand-over chain (the CUDA side is tested under -m gpu) ----------------
class _Geom:
    def __init__(self, history, back, fwd):
        self.history, self.shard_back, self.shard_fwd = history, back, fwd


class _FakeRx:
    """Stands in for rx_path: records the protocol and turns an entry state into an exit state."""
    class _S:
        _first = True

    def __init__(self, n_msgs):
        self._slicer, self.log, self.n_msgs, self.entry = self._S(), [], n_msgs, None

    def defer_resolve(self, on=True): self.log.append(("defer", on))
    def seek(self, a, b): self.log.append(("seek", a, b)); self.span = (a, b)
    def process(self, iq, flush=False, collect=True): self.log.append(("process", len(iq), flush)); self.n = len(iq)
    def resolve(self, entry): self.log.append(("resolve", entry)); self.entry = entry
    def walk_state(self): return self.entry[0] + 1000, self.span[0] + self.n
    def drain(self): self.log.append(("drain", self._slicer._first)); return self.n_msgs


def _ts_worker(rank, world, port_no, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    plan = shard.time_shard_plan(1_000_000, world, _Geom(4, 101, 483))
    sp = plan[rank]
    rx = _FakeRx(n_msgs=0 if rank == 0 else 3)
    recv, send = shard.dist_state_exchange(rank, torch.device("cpu"))
    got = shard.process_time_sharded(rx, np.zeros(sp.end - sp.first_sample, np.float32), sp, recv, send)
    ret[rank] = (got, rx.entry, rx.log)
    dist.barrier()
    dist.destroy_process_group()


def test_time_shard_chain_world2():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_ts_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    plan = shard.time_shard_plan(1_000_000, 2, _Geom(4, 101, 483))
    assert ret[0][1] == (0, 0)
    assert ret[1][1] == (1000, plan[0].end)                          # rank 0's exit state is rank 1's entry
    assert ret[0][2][:3] == [("defer", True), ("seek", 0, 0), ("process", plan[0].end, False)]
    assert ret[1][2][2] == ("process", 1_000_000 - plan[1].first_sample, True)
    assert ret[0][2][-1] == ("drain", True) and ret[1][2][-1] == ("drain", True)   # rank 0 queued nothing
    assert (ret[0][0], ret[1][0]) == (0, 3)


def test_time_shard_plan_invariants():
    g = _Geom(4, 101, 483)
    for n in (10_000, 100_000, 1 << 20, (1 << 28) + 12345):
        for world in (1, 2, 3, 8):
            plan = shard.time_shard_plan(n, world, g)
            assert 1 <= len(plan) <= world and plan[0].first_sample == 0 and plan[0].first_decision == 0
            assert plan[-1].flush and plan[-1].end == n and not any(s.flush for s in plan[:-1])
            for a, b in zip(plan, plan[1:]):
                assert a.end == b.first_decision + g.shard_fwd <= n          # a decides exactly up to b's start
                assert b.first_sample % 512 == 0 and b.first_decision >= b.first_sample + g.shard_back
                assert b.first_decision - b.first_sample < g.shard_back + 512
    assert len(shard.time_shard_plan(10_000, 8, g)) == 1 and len(shard.time_shard_plan(20_000, 8, g)) == 3   # too short for 8
    import pytest
    with pytest.raises(ValueError):
        shard.time_shard_plan(100_000, 2, g, boundaries=[50])                # inside the first span's warm-up
    with pytest.raises(ValueError):
        shard.time_shard_plan(100_000, 2, g, boundaries=[99_900])            # no room for the forward halo
    with pytest.raises(ValueError):
        shard.time_shard_plan(100_000, 2, g, boundaries=[30_000, 60_000])    # more spans than ranks


def test_compose_entries_logic():
    g = _Geom(4, 101, 483)
    plan = shard.time_shard_plan(1 << 22, 4, g)
    X = 1 << 24
    # (pos, p, first_real, first_packet, exact_span, passed)
    ok = [(900_000, plan[1].first_decision, 5_000, 5_010, X, 7), (plan[1].first_decision, plan[2].first_decision, -1, -1, X, 0),
          (3_000_000, plan[3].first_decision + 100, plan[2].first_decision + 50, plan[2].first_decision + 60, X, 2), (0,) * 6]
    entries, queued, bad = shard.compose_entries(plan, ok)
    assert bad == 3 and queued == [0, 7, 7, 9]
    assert entries[1] == (900_000, plan[1].first_decision)
    assert entries[2] == (900_000, plan[2].first_decision)          # no packet in span 1: pos passes through
    assert entries[3] == (3_000_000, plan[3].first_decision + 100)
    # span 1 has a real candidate before the p handed over by span 0 -> speculation fails there
    s = list(ok); s[0] = (900_000, plan[1].first_decision + 300, 5_000, 5_010, X, 7)
    s[1] = (plan[1].first_decision, plan[2].first_decision, plan[1].first_decision + 200, -1, X, 0)
    assert shard.compose_entries(plan, s)[2] == 1
    s[1] = (plan[1].first_decision, plan[2].first_decision, plan[1].first_decision + 300, -1, X, 0)   # at p: still fine
    assert shard.compose_entries(plan, s)[2] == 3
    assert shard.compose_entries(plan, s)[0][2][1] == plan[2].first_decision      # exit p = max(p, entry p)
    # the first packet of span 2 lies too far from the true pos for the float skip to be exact
    s = list(ok); s[0] = (10, plan[1].first_decision, -1, -1, X, 0)
    s[2] = (X + 500_000, plan[3].first_decision, 2_200_000, X + 20, X, 1)
    assert shard.compose_entries(plan, s)[2] == 2
    assert shard.compose_entries([plan[0]], [(0,) * 6]) == ([(0, 0)], [0], 0)     # a single span is never speculated on


class _FakeSpecRx(_FakeRx):
    def __init__(self, n_msgs, summary):
        super().__init__(n_msgs); self.summary = summary

    def resolve(self, entry): self.log.append(("resolve", entry)); self.entry = entry if entry is not None else (-1, -1)

    def walk_summary(self):
        class S: pass
        s = S()
        s.pos, s.p, s.first_real, s.first_packet, s.exact_span, s.frames_passed = self.summary
        return s


def _spec_worker(rank, world, port_no, fail_at, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    plan = shard.time_shard_plan(1_000_000, 2, _Geom(4, 101, 483))      # world 3, two spans: rank 2 idles
    summary = (777, plan[1].first_decision + (600 if fail_at == 1 else 0), -1, -1, 1 << 24, 4) if rank == 0 else (0,) * 6
    rx = _FakeSpecRx(n_msgs=4 if rank == 0 else 2, summary=summary)
    recv, send = shard.dist_state_exchange(rank, torch.device("cpu"))
    sp = plan[rank] if rank < len(plan) else None
    iq = np.zeros((sp.end - sp.first_sample) if sp else 0, np.float32)
    got = shard.process_time_sharded_speculative(rx, iq, plan, rank, shard.dist_all_gather6(world, torch.device("cpu")), recv, send)
    ret[rank] = (got, rx.entry, [e for e in rx.log if e[0] in ("resolve", "drain")])
    dist.barrier()
    dist.destroy_process_group()


def test_speculative_runner_world3_gloo():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_spec_worker, args=(3, _free_port(), 0, ret), nprocs=3, join=True)
    plan = shard.time_shard_plan(1_000_000, 2, _Geom(4, 101, 483))
    # rank 0 speculated (resolve(None)) and kept it; rank 1 = last span resolves once with the composed entry
    assert ret[0][2] == [("resolve", None), ("drain", True)]
    assert ret[1][2] == [("resolve", (0, plan[1].first_decision)), ("drain", False)]      # 4 messages queued before it
    assert ret[2][0] == 0 and ret[2][2] == []
    assert (ret[0][0], ret[1][0]) == (4, 2)


# ---- both multi-GPU modes end to end at world size 2: gloo for the plumbing, the EMULATED build of the library (tests/
# simt/library_emul.cc: the library's own sources on a host SIMT emulator, see tests/test_library_simt.py) as each rank's
# "GPU". Every rank is its own process, so one emulated device per rank.
def _emul_worker(rank, world, port_no, lib_path, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gr_air_modes_b200 import _lib
    _lib.LIB_PATH, _lib._lib = lib_path, None
    import gr_air_modes_b200 as am
    from oracle import cpu_oracle as co
    dev = torch.device("cpu")
    port = co.Port()
    rate, n = 4e6, 90_000

    # (1) headline mode: one independent channel per rank, inputs fanned out from rank 0, no data-path collective
    def make(ch):
        sc = synth.make_scene(rate, n, 14, seed=300 + ch)
        return torch.from_numpy(sc.iq.copy()), [b.frame.hex() for b in sc.bursts]

    iq, _ = shard.fan_out(make, rank, world, dev, 2 * n)
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    rx.process(iq.numpy(), flush=True)
    mine = port.run_iq(synth.make_scene(rate, n, 14, seed=300 + rank).iq, rate, 7.0, True, co.MA_CANONICAL).msgs
    assert q.strings() == mine and len(mine) >= 5
    counts = shard.gather_counts(len(mine), world, dev)
    rx.close()

    # (2) secondary mode: ONE recording cut into `world` time spans; hand-over chain, then speculative resolution
    rec = synth.make_scene(rate, 2 * n, 40, seed=555)
    want = port.run_iq(rec.iq, rate, 7.0, True, co.MA_CANONICAL).msgs
    plan = shard.time_shard_plan(2 * n, world, am.query_geometry(rate, 7.0, True))
    sp = plan[rank]
    span_iq = rec.iq[2 * sp.first_sample: 2 * sp.end]
    recv, send = shard.dist_state_exchange(rank, dev)
    out = {}
    for mode in ("chain", "speculative"):
        q = am.msg_queue()
        rx = am.rx_path(rate, 7.0, q, use_pmf=True)
        if mode == "chain":
            shard.process_time_sharded(rx, span_iq, sp, recv, send)
        else:
            shard.process_time_sharded_speculative(rx, span_iq, plan, rank, shard.dist_all_gather6(world, dev), recv, send)
        out[mode] = q.strings()
        rx.close()
        dist.barrier()
    # (3) the speculative pass with nothing waiting on the host: summary kernel -> all-gather on the "device" -> compose
    # kernel on every rank -> the last span resolves from that kernel's output
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    rx.defer_resolve(True)
    scratch = shard.AsyncPass(world, len(plan), dev, steps=2)
    for step in range(2):                                     # twice: a pass leaves nothing behind
        row = shard.time_shard_pass_async(rx, span_iq, plan, rank, scratch, step)
    rx._ctx.call("amb_synchronize")
    verdict = int(row[0])
    rx._slicer._first = int(row[1 + 2 * len(plan) + rank]) == 0
    rx.drain()
    out["async"] = (verdict, len(plan) - 1, q.strings())
    rx.close()
    dist.barrier()
    ret[rank] = (counts, out["chain"], out["speculative"], want, out["async"])
    dist.barrier()
    dist.destroy_process_group()


def test_both_multi_gpu_modes_world2_with_the_emulated_library(tmp_path_factory):
    import emul_build
    lib = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_emul_worker, args=(2, _free_port(), lib, ret), nprocs=2, join=True)
    assert ret[0][0] == ret[1][0] and all(c >= 5 for c in ret[0][0])
    want = ret[0][3]
    assert len(want) >= 15
    assert ret[0][1] + ret[1][1] == want                 # the spans' messages, in rank order, are the one-shot run's
    assert ret[0][2] + ret[1][2] == want
    assert ret[0][4][0] == ret[0][4][1] == ret[1][4][0]       # the speculation held on every span (same verdict on both ranks)
    assert ret[0][4][2] + ret[1][4][2] == want                # ... and the device-side hand-over gives the same messages
