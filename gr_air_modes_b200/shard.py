"""Multi-GPU plumbing: independent IQ channels, one per rank (SURVEY.md 8e).

The receive chain has no cross-channel dependency, so there is no collective on the data path. NCCL (or
gloo in the CPU tests) is used only to (1) fan the input buffers out from the ingest rank, (2) agree on the
slowest rank's time and (3) gather the tiny per-rank results.
"""
from __future__ import annotations


def channels_of(rank: int, world: int, n_channels: int):
    """Round-robin channel ownership when there are more channels than ranks."""
    return [c for c in range(n_channels) if c % world == rank]


def fan_out(make_channel, rank: int, world: int, device, numel: int, timing: dict | None = None):
    """Rank 0 builds channel c with make_channel(c) -> (float32 tensor[numel], meta) and sends it to rank c.
    Returns this rank's (tensor, meta). `timing` (optional dict) receives, on rank 0, the transfers ALONE:
    "send_ms" (CUDA events around each dist.send on the current stream; host clock on CPU tensors) and "bytes"."""
    if world == 1:
        return make_channel(0)
    import time
    import torch
    import torch.distributed as dist
    if timing is not None and not timing.get("warm"):      # NCCL sets a peer connection up on first use: not part of the transfer
        timing["warm"] = True
        w = torch.zeros(4, dtype=torch.float32, device=device)
        if rank == 0:
            for ch in range(1, world):
                dist.send(w, dst=ch)
        else:
            dist.recv(w, src=0)
    if rank == 0:
        metas = [None] * world
        mine = None
        ms, nbytes = 0.0, 0
        for ch in range(world - 1, -1, -1):
            iq, meta = make_channel(ch)
            metas[ch] = meta
            if ch != 0:
                if iq.is_cuda:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    dist.send(iq, dst=ch)
                    e1.record()
                    e1.synchronize()
                    ms += e0.elapsed_time(e1)
                else:
                    t0 = time.perf_counter()
                    dist.send(iq, dst=ch)
                    ms += 1e3 * (time.perf_counter() - t0)
                nbytes += iq.numel() * iq.element_size()
                del iq
            else:
                mine = iq
        if timing is not None:
            timing["send_ms"] = timing.get("send_ms", 0.0) + ms
            timing["bytes"] = timing.get("bytes", 0) + nbytes
    else:
        mine = torch.empty(numel, dtype=torch.float32, device=device)
        dist.recv(mine, src=0)
        metas = None
    out = [None]
    dist.scatter_object_list(out, metas, src=0)
    return mine, out[0]


def max_over_ranks(value: float, world: int, device) -> float:
    if world == 1:
        return float(value)
    import torch
    import torch.distributed as dist
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_counts(value: int, world: int, device):
    """All ranks' integer results (e.g. frames decoded) on every rank."""
    if world == 1:
        return [int(value)]
    import torch
    import torch.distributed as dist
    t = torch.tensor([int(value)], dtype=torch.int64, device=device)
    out = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [int(x.item()) for x in out]


# ---- one long recording time-sharded over the ranks (SURVEY.md 8e, secondary mode) -----------------------------
# The dense stages of a span depend on its samples only; what the reference's scan loop carries across a cut is
# two integers (include/airmodes_b200.h, amb_seek). So every rank runs its span's dense stages at once, and the
# loop state then travels down the ranks: recv (16 B) -> walk + slice (sparse, tens of microseconds) -> send.
class Span:
    __slots__ = ("first_sample", "first_decision", "end", "flush")

    def __init__(self, first_sample, first_decision, end, flush):
        self.first_sample, self.first_decision, self.end, self.flush = first_sample, first_decision, end, flush

    def __repr__(self):
        return "Span(samples [%d, %d), decisions from %d%s)" % (self.first_sample, self.end, self.first_decision,
                                                                ", last" if self.flush else "")


def time_shard_plan(n_total: int, world: int, geometry, align: int = 512, boundaries=None):
    """Cut a recording of n_total samples into at most `world` spans (fewer if it is too short to be worth it).

    geometry: amb_query_geometry's struct (history, shard_back, shard_fwd). boundaries: optional explicit list of
    the reported indices where spans 1.. start (testing); default = equal shares. first_sample is rounded down to
    `align` samples so that device pointers into the recording stay TMA-aligned."""
    back, fwd = int(geometry.shard_back), int(geometry.shard_fwd)
    if boundaries is None:
        spans = max(1, min(world, n_total // (8 * (back + fwd) + align)))
        boundaries = [n_total * k // spans for k in range(1, spans)]
    boundaries = [0] + sorted(int(b) for b in boundaries)
    if len(boundaries) > world:
        raise ValueError("more spans than ranks")
    plan = []
    for k, r0 in enumerate(boundaries):
        last = k == len(boundaries) - 1
        first = 0 if k == 0 else max(0, (r0 - back) // align * align)
        if k and first and r0 < first + back:
            raise ValueError("span %d starts too early for its halo" % k)
        if k and first == 0:
            raise ValueError("boundary %d lies inside the first span's warm-up" % r0)
        end = n_total if last else boundaries[k + 1] + fwd
        if end > n_total or (not last and boundaries[k + 1] <= r0):
            raise ValueError("spans too short for the forward halo")
        plan.append(Span(first, r0, end, last))
    return plan


def process_time_sharded(rx, span_iq, span, recv_entry, send_exit):
    """Run one span on `rx` (a gr_air_modes_b200.rx_path). span_iq holds the samples [span.first_sample, span.end).
    recv_entry() -> (pos, p, queued) from the previous span (not called for the first span); send_exit((pos, p,
    queued)) hands this span's exit state to the next one (not called for the last). `queued` = messages queued by
    all earlier spans: the reference's slicer prints its very first message with 6 digits (slicer_impl.cc:192),
    and there is one slicer per stream, not per span. Returns the number of messages this span queued."""
    rx.defer_resolve(True)
    rx.seek(span.first_sample, span.first_decision)
    rx.process(span_iq, flush=span.flush, collect=False)       # dense stages: concurrent on all ranks
    pos, p, queued = (0, 0, 0) if span.first_decision == 0 else recv_entry()
    rx.resolve((pos, p))
    if not span.flush:
        pos, p = rx.walk_state()
    rx._slicer._first = queued == 0
    mine = rx.drain()
    if not span.flush:
        send_exit((pos, p, queued + mine))
    return mine


def dist_state_exchange(rank: int, device):
    """(recv_entry, send_exit) over torch.distributed point-to-point (nccl: device tensors; gloo: cpu)."""
    import torch
    import torch.distributed as dist

    def recv_entry():
        t = torch.zeros(3, dtype=torch.int64, device=device)
        dist.recv(t, src=rank - 1)
        return tuple(int(x) for x in t.tolist())

    def send_exit(state):
        dist.send(torch.tensor([int(x) for x in state], dtype=torch.int64, device=device), dst=rank + 1)

    return recv_entry, send_exit


# ---- speculative resolution: the chain leaves the critical path ---------------------------------------------------
# Every span but the last resolves at once with the default entry; one all-gather of six integers per span then
# tells every rank the true entry of every span, as long as each speculative result is provably what the true entry
# would have produced (include/airmodes_b200.h, amb_get_walk_summary). The first span that fails the test, and every
# span after it, falls back to the hand-over chain.
def compose_entries(plan, summaries):
    """summaries[k] = (pos, p, first_real, first_packet, exact_span, frames_passed) of span k's speculative
    resolution (anything for the last span). Returns (entries, queued, first_bad): entries[k] = true (pos, p) entry
    of span k and queued[k] = messages queued before it, both valid for k <= first_bad; first_bad = index of the
    first span whose speculation does not hold (len(plan) - 1, the never-speculated last span, if all hold)."""
    entries, queued = [(0, 0)], [0]
    last = len(plan) - 1
    for k in range(last):
        pos_in, p_in = entries[k]
        pos, p, first_real, first_packet, exact_span, passed = (int(x) for x in summaries[k])
        ok = (first_real < 0 or p_in <= first_real) and (first_packet < 0 or first_packet - pos_in < exact_span)
        if not ok:
            return entries, queued, k
        entries.append((pos if first_packet >= 0 else pos_in, max(p, p_in)))
        queued.append(queued[k] + passed)
    return entries, queued, last


def process_time_sharded_speculative(rx, span_iq, plan, rank, all_gather, recv_entry, send_exit):
    """As process_time_sharded, for every rank of the plan at once. all_gather(list of 6 ints) -> list over ranks.
    Returns the number of messages this span queued."""
    if rank >= len(plan):                                  # more ranks than spans: only take part in the collective
        all_gather([0] * 6)
        return 0
    span = plan[rank]
    last = len(plan) - 1
    rx.defer_resolve(True)
    rx.seek(span.first_sample, span.first_decision)
    rx.process(span_iq, flush=span.flush, collect=False)
    mine = [0] * 6
    if rank < last:
        rx.resolve(None)                                   # speculative: fresh entry at first_decision
        s = rx.walk_summary()
        mine = [s.pos, s.p, s.first_real, s.first_packet, s.exact_span, s.frames_passed]
    entries, queued, bad = compose_entries(plan, all_gather(mine))
    if rank < bad:                                         # speculation holds: done, nothing to wait for
        q = queued[rank]
    else:
        if rank == bad:
            pos, p = entries[rank]
            q = queued[rank]
        else:
            pos, p, q = recv_entry()
        rx.resolve((pos, p))                               # first resolution of the last span, or a re-resolution
    rx._slicer._first = q == 0
    if rank >= bad and not span.flush:
        state = rx.walk_state()
        n = rx.drain()
        send_exit(state + (q + n,))
        return n
    return rx.drain()


def dist_all_gather6(world: int, device):
    import torch
    import torch.distributed as dist

    def all_gather(vals):
        t = torch.tensor([int(v) for v in vals], dtype=torch.int64, device=device)
        out = torch.empty(world * 6, dtype=torch.int64, device=device)
        dist.all_gather_into_tensor(out, t)
        return out.view(world, 6).tolist()

    return all_gather


# ---- the speculative pass with nothing waiting on the host -----------------------------------------------------------
# process_time_sharded_speculative reads each span's summary back (a device synchronisation), all-gathers Python
# integers and composes the entries on the host: host-driven latency per pass that, on many GPUs, exceeds a span's
# scan share. Here a pass is a fixed sequence of enqueues: summary kernel -> all-gather of 6 int64 per span on the
# device -> compose kernel (every rank, all spans) -> the last span resolves with the entry that kernel wrote. The host
# looks at the verdict (out[0]) only after the passes it wants have been enqueued; a pass whose speculation failed
# (out[0] < len(plan) - 1: rare, a packet straddling a cut in an unlucky way) is redone with the functions above.
class AsyncPass:
    """Device scratch of one rank for time_shard_pass_async: one row per pass, so that passes in flight never share a
    buffer. `side`: a CUDA stream of the caller's on which the exchange runs (None: the current stream / CPU tensors)."""

    def __init__(self, world: int, n_spans: int, device, steps: int = 1, side=None):
        import torch
        self.mine = torch.zeros(steps, 6, dtype=torch.int64, device=device)
        self.all = torch.zeros(steps, world * 6, dtype=torch.int64, device=device)
        self.out = torch.zeros(steps, 1 + 3 * n_spans, dtype=torch.int64, device=device)
        self.n_spans, self.world, self.side = n_spans, world, side


def time_shard_pass_async(rx, span_iq, plan, rank, scratch: "AsyncPass", step: int = 0):
    """Enqueue one time-sharded pass of this rank (rx in deferred mode). Nothing here blocks on the device. The caller
    later checks scratch.out[step, 0] == len(plan) - 1 (every speculation held) before trusting the frames."""
    import contextlib
    import torch
    import torch.distributed as dist
    last = len(plan) - 1
    active = rank < len(plan)
    side = scratch.side
    sptr = side.cuda_stream if side is not None else 0
    mine, gathered, row = scratch.mine[step], scratch.all[step], scratch.out[step]
    if active:
        sp = plan[rank]
        rx.seek(sp.first_sample, sp.first_decision)
        rx.process(span_iq, flush=sp.flush, collect=False)
        if rank < last:
            rx.resolve(None)                               # speculative: fresh entry at first_decision
            rx.walk_summary_async(mine.data_ptr())
        rx.join_stream(sptr)                               # the stream the collective runs on waits for the summary
    with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
        if scratch.world > 1:
            dist.all_gather_into_tensor(gathered, mine)
        else:
            gathered.copy_(mine)
    if active:
        rx.compose_entries_async(gathered.data_ptr(), len(plan), row.data_ptr(), sptr)
        if rank == last:
            rx.resolve_device(row.data_ptr() + 8 * (1 + 2 * rank), sptr)
    return row
