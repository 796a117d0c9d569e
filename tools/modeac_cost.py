"""What the receive chain's option "modeac" costs. Scene: a configs[1]-like recording (4 Msps, 2^28 complex samples, 1000
DF11/DF17 bursts at mixed SNR, synth.make_scene_device) with --replies Mode A/C replies added at 15-30 dB. Each call is
one whole stream from device memory (amb_process with flush, on torch's stream, then amb_join), timed with CUDA events
from before the call to the end of its last kernel on any of the context's streams. Contexts with the option off and on
run interleaved; medians over --reps calls after --warmup. A separate run under torch.profiler gives the device time of
the option's two kernels. The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/modeac_cost.py [--n 268435456] [--replies 20000] [--reps 25] [--warmup 3] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import gr_air_modes_b200 as am  # noqa: E402
from gr_air_modes_b200 import synth  # noqa: E402
from track_cost import card  # noqa: E402

RATE = 4e6


def scene(n, replies, seed=1):
    import torch
    iq, _, _ = synth.make_scene_device(RATE, n, 1000, seed, torch.device("cuda", 0))
    spu = RATE / 1e6
    rng = np.random.default_rng(seed)
    starts = np.sort(rng.uniform(64 * spu, n - 64 * spu, replies))
    c = iq.view(torch.complex64)
    for s in starts:
        amp = float(np.sqrt(2.0 * 0.01 ** 2 * 10 ** (rng.uniform(15, 30) / 10)))
        n0, w = synth.modeac_waveform(int(rng.integers(0, 1 << 13)) & ~0x40, bool(rng.random() < 0.5), float(s), amp,
                                      float(rng.uniform(0, 2 * np.pi)), RATE / 2e6)
        c[n0:n0 + w.size] += torch.from_numpy(w).to(c.device)
    return iq


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, default=1 << 28)
    ap.add_argument("--replies", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    iq = scene(args.n, args.replies)
    stream = torch.cuda.current_stream()
    rx = {}
    for s in (0, 1):
        rx[s] = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True, modeac=bool(s))
        rx[s].use_stream(stream.cuda_stream)
    times = {0: [], 1: []}
    replies = frames = 0
    for r in range(args.warmup + args.reps):
        for s in (0, 1):
            rx[s].reset()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            rx[s].process(iq, flush=True, collect=False)
            rx[s].join()
            e1.record(stream)
            e1.synchronize()
            if r >= args.warmup:
                times[s].append(e0.elapsed_time(e1))
            rx[s].drain()
            frames = len(rx[s].frames)
            if s:
                replies = len(rx[s].modeac())
    kernels = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            rx[1].reset()
            rx[1].process(iq, flush=True, collect=False)
            rx[1].join()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "modeac" in ev.key:
            kernels[ev.key] = round(ev.device_time_total / max(ev.count, 1) / 1e3, 4)
    rx[1].drain()
    rx[1].modeac()
    for x in rx.values():
        x.close()
    result = {"card": name, "power_limit": pl, "rate": RATE, "n": args.n, "planted_replies": args.replies,
              "replies": replies, "frames": frames, "reps": args.reps,
              "ms_call_off": round(statistics.median(times[0]), 4), "ms_call_on": round(statistics.median(times[1]), 4),
              "ms_kernel": kernels}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
