"""What the batch decoder's option "track_ext" costs. Scene: the op-status fleet and the Comm-B fleet as one stream
(tests/track_ext_cases.fleet: tests/opstatus_cases.fleet_scene + tests/commb_cases.fleet_scene). Both decoders run
with opstatus, commb and track on; only track_ext differs. It reports, as device time (amb_decoder_stats, CUDA events
around the call):
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
  ms_snapshot_host     one amb_decoder_aircraft_ext call into host memory at the end of the scene (median of --reps,
                       wall clock: a count pass, then count + scan + gather, as decode.batch_decoder.aircraft_ext runs them)
  ms_snapshot_device   the same into device memory (aircraft_ext_device with buffers given)
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/track_ext_cost.py [--aircraft 300] [--seconds 60] [--track 60] [--ext 60] [--batch 4096] [--json out.json]
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

import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402
from track_cost import card  # noqa: E402


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--track", type=int, default=60)
    ap.add_argument("--ext", type=int, default=60)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    frames = tc.frames_of(xc.fleet(args.aircraft, args.seconds), unqueued_every=0)
    loc = [10.0, 20.0]
    kw = dict(opstatus=30, commb=30, track=args.track)
    dec = {0: decode.batch_decoder(loc, **kw), 1: decode.batch_decoder(loc, track_ext=args.ext, **kw)}
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
    rows, ext = dec[1].aircraft_ext()
    n = max(len(rows), 1)
    buf = torch.empty(n * 128, dtype=torch.uint8, device="cuda")
    xbuf = torch.empty(n * 144, dtype=torch.uint8, device="cuda")
    snap_h, snap_d = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dec[1].aircraft_ext()
        snap_h.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        dec[1].aircraft_ext_device(out_dev=buf, ext_dev=xbuf)
        snap_d.append((time.perf_counter() - t0) * 1e3)
    for d in dec.values():
        d.close()
    shown = {g: int(sum(1 for x in ext["shown"] if x & (1 << g))) for g in range(6)}
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "track": args.track, "track_ext": args.ext, "batch": args.batch, "rows_at_end": len(rows),
              "groups_shown_at_end": [shown[g] for g in range(6)],
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
