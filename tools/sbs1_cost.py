"""What the batch decoder's option "sbs1" costs. Scene: the op-status and Comm-B fleet of tests/track_ext_cases.fleet
(positions, velocities, idents, DF0/4/5/11/20/21 replies). Both decoders run with no other option; only sbs1 differs.
It reports, as device time (amb_decoder_stats, CUDA events around the call):
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
  ms_text_host         amb_decoder_sbs1 of that call into host memory (wall clock, median of --reps)
  ms_text_device       amb_decoder_sbs1_device of it into device memory (wall clock, median of --reps)
  text_bytes / record_bytes   the call's SBS-1 text against the 144-byte records it comes from
  ms_checker_host      HOST timing, for context: the Python checker (tests/sbs1_oracle.py) forming the same lines from
                       the same records on this machine's CPU
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/sbs1_cost.py [--aircraft 300] [--seconds 60] [--batch 4096] [--reps 7] [--json out.json]
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

import sbs1_oracle as so  # noqa: E402
import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402
from track_cost import card  # noqa: E402


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    frames = tc.frames_of(xc.fleet(args.aircraft, args.seconds), unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, sbs1=True)}
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
    text = dec[1].sbs1_text()
    out = torch.empty(max(len(text), 1), dtype=torch.uint8, device="cuda")
    th, td = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dec[1].sbs1_text()
        th.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        dec[1].sbs1_text_device(out)
        td.append((time.perf_counter() - t0) * 1e3)
    h = decode.batch_decoder(loc)
    recs = h.decode(frames)
    h.close()
    t0 = time.perf_counter()
    want = so.Sbs1Checker().feed(frames, recs)
    checker_ms = (time.perf_counter() - t0) * 1e3
    for d in dec.values():
        d.close()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "batch": args.batch, "lines": text.count(b"\r\n"), "text_equals_checker": text == want,
              "text_bytes": len(text), "record_bytes": len(frames) * 144,
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4),
              "ms_text_host": round(statistics.median(th), 4), "ms_text_device": round(statistics.median(td), 4),
              "ms_checker_host": round(checker_ms, 1)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
