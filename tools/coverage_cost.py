"""What the batch decoder's option "coverage" costs. Scene: the fleet of tests/track_cases.fleet_scene (positions,
velocities, idents, DF0/4/5/20/21 replies of --aircraft aircraft over --seconds), with a receiver location. Both decoders
run with no other option; only coverage differs. It reports, as device time (amb_decoder_stats, CUDA events around the
call):
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
and, as wall clock (median of --reps):
  ms_grid_host         amb_decoder_coverage into host memory
  ms_grid_device       amb_decoder_coverage_device into device memory
The grid is checked against tests/coverage_oracle.py on the same records. The card name and its power limit are printed
with the numbers. Needs an H100.

    python tools/coverage_cost.py [--aircraft 2000] [--seconds 600] [--batch 4096] [--reps 7] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import coverage_oracle as co  # noqa: E402
import track_cases as tc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402
from track_cost import card  # noqa: E402


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    frames = tc.frames_of(tc.fleet_scene(args.aircraft, args.seconds), unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, coverage=True)}
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
    grid = dec[1].coverage()
    out = torch.empty((72, 9), dtype=torch.float64, device="cuda")
    th, td = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dec[1].coverage()
        th.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        dec[1].coverage_device(out)
        td.append((time.perf_counter() - t0) * 1e3)
    h = decode.batch_decoder(loc)
    recs = h.decode(frames)
    h.close()
    for d in dec.values():
        d.close()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "batch": args.batch, "counted": sum(co.counted(r) is not None for r in recs),
              "cells_set": int((grid > 0).sum()), "grid_equals_checker": grid.tobytes() == co.grid_of(recs).tobytes(),
              "device_equals_host": out.cpu().numpy().tobytes() == grid.tobytes(),
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4),
              "ms_grid_host": round(statistics.median(th), 4), "ms_grid_device": round(statistics.median(td), 4)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
