"""What the batch decoder's option "opstatus" yields and costs. Scene: tests/opstatus_cases.fleet_scene - N aircraft of
ADS-B versions 0, 1 and 2 over T seconds, each sending positions and velocities at about 2 Hz, its operational status
(TC 31, the surface subtype on the ground) about every 2.5 s and, for version 2, its target state (TC 29 subtype 1) about
every 1.25 s; each aircraft keeps one position type code and one set of NIC supplements. It reports:
  per version    op-status and target-state messages sent (queued) and decoded, and positions rated NIC / NUC
  positions      rated right (the outcome, NIC or NUCp and Rc the fleet's truth calls for), wrong, and NUC before the
                 aircraft's first op status (its op status had not been heard yet)
and as device time (amb_decoder_stats, CUDA events around the call), off -> on:
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/opstatus_yield.py [--aircraft 300] [--seconds 200] [--opstatus 30] [--batch 4096] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import opstatus_cases as oc  # noqa: E402
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


def tally(frames, recs, truth, S):
    """Counts per ADS-B version and for the positions, against the fleet's truth."""
    out = decode.opstatus_outcome(recs)
    nic = (np.asarray(recs["pad_"], dtype=np.uint64) >> np.uint64(56)) & np.uint64(0xFF)
    ts = frames["secs"].astype(np.float64) + frames["frac"]
    res = {v: {"opstatus_sent": 0, "opstatus_decoded": 0, "target_state_sent": 0, "target_state_decoded": 0,
               "positions": 0, "nic": 0, "nuc": 0} for v in (0, 1, 2)}
    pos = {"right": 0, "wrong": 0, "nuc_before_first_opstatus": 0, "nuc_opstatus_older_than_S": 0}
    heard = {}                                                  # address -> t of its latest queued op status
    for k, tr in enumerate(truth):
        if tr is None or not frames["passed"][k]:
            continue
        kind, ver, tcode, nica, nicb, nicc = tr
        a = int(recs["icao"][k])
        row = res[ver]
        if kind == "opstatus":
            row["opstatus_sent"] += 1
            row["opstatus_decoded"] += int(out[k] == decode.ES_OPSTATUS)
            heard[a] = float(ts[k])
        elif kind == "target_state":
            row["target_state_sent"] += 1
            row["target_state_decoded"] += int(out[k] == decode.ES_TARGET_STATE)
        else:
            row["positions"] += 1
            row["nic"] += int(out[k] == decode.ES_NIC)
            row["nuc"] += int(out[k] == decode.ES_NUC)
            if a not in heard or ts[k] - heard[a] > S:
                pos["nuc_before_first_opstatus" if a not in heard else "nuc_opstatus_older_than_S"] += \
                    int(out[k] == decode.ES_NUC)
                continue
            want_o, want_n, want_rc = oc.expected_nic(ver, tcode, nica, nicb, nicc)
            v = decode.opstatus_values(recs[k])
            rc = None if v is None else v["rc"]
            ok = out[k] == want_o and nic[k] == want_n and (rc is None if want_rc is None else
                                                              rc is not None and math.isclose(rc, want_rc, rel_tol=1e-6))
            pos["right" if ok else "wrong"] += 1
    return res, pos


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=200.0)
    ap.add_argument("--opstatus", type=int, default=30)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    msgs, truth = oc.fleet_scene(args.aircraft, args.seconds)
    frames = tc.frames_of(msgs, unqueued_every=0)
    loc = [10.0, 20.0]
    dec = {0: decode.batch_decoder(loc), 1: decode.batch_decoder(loc, opstatus=args.opstatus)}
    times = {0: [], 1: []}
    recs = []
    for lo in range(0, len(frames), args.batch):                       # off and on interleaved, batch by batch
        for s in (0, 1):
            r = dec[s].decode(frames[lo:lo + args.batch])
            times[s].append(dec[s].stats()[1])
            if s:
                recs.append(r)
    per_version, positions = tally(frames, np.concatenate(recs), truth, args.opstatus)
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
              "opstatus": args.opstatus, "batch": args.batch, "per_version": per_version, "positions": positions,
              "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
              "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4)}
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
