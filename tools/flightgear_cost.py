"""What the batch decoder's option "flightgear" costs. Scene: tests/track_cases.fleet_scene (positions, velocities,
idents and other replies of a fleet). Both decoders run with no other option; only flightgear differs. It reports,
as device time (amb_decoder_stats, CUDA events around the call), after one warm-up pass:
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
  ms_bytes_device      amb_decoder_flightgear_device of that call into device memory (wall clock, median of --reps)
  packets              the packets of the whole-scene call; packets_equal_checker: the same count as the checker's
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/flightgear_cost.py [--aircraft 2000] [--seconds 600] [--batch 4096] [--reps 25] [--json out.json]
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

import flightgear_oracle as fo  # noqa: E402
import track_cases as tc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402
from track_cost import card  # noqa: E402


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    frames = tc.frames_of(tc.fleet_scene(args.aircraft, args.seconds), unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, flightgear=True)}
    times = {0: [], 1: []}
    for warm in (True, False):                                         # off and on interleaved, batch by batch
        for lo in range(0, len(frames), args.batch):
            for s in (0, 1):
                dec[s].decode(frames[lo:lo + args.batch])
                if not warm and lo + args.batch <= len(frames):
                    times[s].append(dec[s].stats()[1])
        for d in dec.values():
            d.reset()
    raw = torch.from_numpy(frames.view("u1").copy()).cuda()
    dev = {0: [], 1: []}
    for r in range(args.reps + 1):
        for s in (0, 1):
            dec[s].reset()
            dec[s].decode_device(raw)
            if r:
                dev[s].append(dec[s].stats()[1])
    data = dec[1].flightgear_bytes()
    out = torch.empty(max(len(data), 1), dtype=torch.uint8, device="cuda")
    td = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dec[1].flightgear_bytes_device(out)
        td.append((time.perf_counter() - t0) * 1e3)
    h = decode.batch_decoder(loc)
    recs = h.decode(frames)
    h.close()
    want = fo.FgChecker().feed(frames, recs)
    for d in dec.values():
        d.close()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "batch": args.batch, "packets": len(data) // fo.PACKET_BYTES,
              "packets_equal_checker": len(data) == len(want),
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4),
              "ms_bytes_device": round(statistics.median(td), 4)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
