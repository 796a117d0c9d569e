"""What the batch decoder's option "track" costs. Scene: tests/track_cases.fleet_scene - N aircraft over T seconds,
each heard about `rate` times per second (positions, velocities, idents, replies), arriving and leaving at random.
It reports, as device time (amb_decoder_stats, CUDA events around the call):
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
  ms_snapshot_host     one amb_decoder_aircraft call into host memory at the end of the scene (median of --reps,
                       wall clock: two count passes and the gather, as decode.batch_decoder.aircraft runs them)
  ms_snapshot_device   the same into device memory (aircraft_device with a buffer given)
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/track_cost.py [--aircraft 2000] [--seconds 600] [--track 60] [--batch 4096] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import track_cases as tc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--rate", type=float, default=0.5)
    ap.add_argument("--track", type=int, default=60)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    frames = tc.frames_of(tc.fleet_scene(args.aircraft, args.seconds, rate=args.rate), unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, track=args.track)}
    times = {0: [], 1: []}
    for lo in range(0, len(frames), args.batch):                       # off and on interleaved, batch by batch
        for s in (0, 1):
            dec[s].decode(frames[lo:lo + args.batch])
            times[s].append(dec[s].stats()[1])
    raw = torch.from_numpy(frames.view("u1").copy()).cuda()
    dev = {0: [], 1: []}
    for _ in range(args.reps):
        for s in (0, 1):
            dec[s].reset()
            dec[s].decode_device(raw)
            dev[s].append(dec[s].stats()[1])
    rows = len(dec[1].aircraft())
    buf = torch.empty(max(rows, 1) * 128, dtype=torch.uint8, device="cuda")
    snap_h, snap_d = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dec[1].aircraft()
        snap_h.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        dec[1].aircraft_device(out_dev=buf)
        snap_d.append((time.perf_counter() - t0) * 1e3)
    for d in dec.values():
        d.close()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "track": args.track, "batch": args.batch, "rows_at_end": rows,
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4),
              "ms_snapshot_host": round(statistics.median(snap_h), 4),
              "ms_snapshot_device": round(statistics.median(snap_d), 4)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
