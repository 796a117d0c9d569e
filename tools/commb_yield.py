"""What the batch decoder's option "commb" yields and costs. Scene: tests/commb_cases.fleet_scene - N aircraft over T
seconds, each sending its ADS-B velocity at about 2 Hz and DF20/21 replies carrying BDS 4,0 / 5,0 / 6,0 words drawn from
its flight state (GS and TAS with a wind, heading = track + crab + declination), some carrying "other" registers (1,7-
like capability words, 4,4-like met words, random words). It reports, per true register:
  decoded_right / decoded_wrong     outcome DECODED with the true register / another one
  resolved_right / resolved_wrong   outcome RESOLVED with the true register / another one
  ambiguous / none                  outcome AMBIGUOUS / NONE
(for "other", every DECODED / RESOLVED is a false decode), and as device time (amb_decoder_stats, CUDA events around the
call), off -> on:
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/commb_yield.py [--aircraft 300] [--seconds 200] [--commb 30] [--batch 4096] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import commb_cases as cc  # noqa: E402
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


def tally(recs, truth):
    """Outcome counts per true register (0x40 / 0x50 / 0x60 / "other")."""
    out = decode.commb_outcome(recs)
    reg = (np.asarray(recs["pad_"], dtype=np.uint64) >> np.uint64(16)) & np.uint64(0xFF)
    res = {}
    for name, key in (("4,0", 0x40), ("5,0", 0x50), ("6,0", 0x60), ("other", "other")):
        idx = np.array([k for k, t in enumerate(truth) if t == key], dtype=np.int64)
        o, g = out[idx], reg[idx]
        right = g == (key if key != "other" else -1)
        res[name] = {"replies": int(len(idx)), "not_tried": int(np.sum(o == decode.COMMB_NOT_TRIED)),
                     "decoded_right": int(np.sum((o == decode.COMMB_DECODED) & right)),
                     "decoded_wrong": int(np.sum((o == decode.COMMB_DECODED) & ~right)),
                     "resolved_right": int(np.sum((o == decode.COMMB_RESOLVED) & right)),
                     "resolved_wrong": int(np.sum((o == decode.COMMB_RESOLVED) & ~right)),
                     "ambiguous": int(np.sum(o == decode.COMMB_AMBIGUOUS)), "none": int(np.sum(o == decode.COMMB_NONE))}
    return res


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=200.0)
    ap.add_argument("--commb", type=int, default=30)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    msgs, truth = cc.fleet_scene(args.aircraft, args.seconds)
    frames = tc.frames_of(msgs, unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, commb=args.commb)}
    times = {0: [], 1: []}
    recs = []
    for lo in range(0, len(frames), args.batch):                       # off and on interleaved, batch by batch
        for s in (0, 1):
            r = dec[s].decode(frames[lo:lo + args.batch])
            times[s].append(dec[s].stats()[1])
            if s:
                recs.append(r)
    yields = tally(np.concatenate(recs), truth)
    raw = torch.from_numpy(frames.view("u1").copy()).cuda()
    dev = {0: [], 1: []}
    for _ in range(args.reps):
        for s in (0, 1):
            dec[s].reset()
            dec[s].decode_device(raw)
            dev[s].append(dec[s].stats()[1])
    for d in dec.values():
        d.close()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds, "frames": len(frames),
              "commb": args.commb, "batch": args.batch, "yield": yields,
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
