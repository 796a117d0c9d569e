"""What the batch decoder's option "local_cpr" adds in positions, how good they are, and what it costs.

Scenes: tests/local_cpr_cases.trajectory_scene - N aircraft on straight tracks around a receiver, one position squitter
every 0.4-0.6 s per aircraft (20 % of them surface vehicles), velocity squitters in between, every third aircraft fading
out for 5-25 s - with a share `drop` of all messages lost, to imitate weak and distant aircraft. Per scene and for the
option off and on (S = --seconds), it reports:
  pos_per_msg_off / _on   position messages that get a position, per position message
  local_share             share of the option-on positions that come from the local decode
  far_off / far_on        positions further than --far-km from the position that was sent (with a receiver location
                          these include the reference's surface fixes, which `zone` at cpr.py:145 moves by Python 3's
                          true division), far_local those of them that came from the local decode
  ms_batch_off / _on      device time of one amb_decode_frames call of --batch messages (H2D, kernels, D2H;
                          amb_decoder_stats), median over the scene's batches, off and on decoders interleaved
  ms_scene_dev_off / _on  device time of one amb_decode_frames_device call over the whole scene (median of --reps)
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/cpr_yield.py [--aircraft 300] [--seconds-scene 300] [--seconds 30] [--batch 4096] [--json out.json]
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

import local_cpr_cases as lc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402


def km(a, b):
    """Great-circle distance in km (spherical earth, 6371 km)."""
    la1, lo1, la2, lo2 = map(math.radians, (a[0], a[1], b[0], b[1]))
    h = math.sin((la2 - la1) / 2) ** 2 + math.cos(la1) * math.cos(la2) * math.sin((lo2 - lo1) / 2) ** 2
    return 2 * 6371.0 * math.asin(min(1.0, math.sqrt(h)))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def run_scene(msgs, truth, loc, S, batch, reps, far_km):
    import torch
    arr, n = decode.frames_from_messages(msgs)
    frames = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE)[:n].copy()
    dec = {0: decode.batch_decoder(loc), S: decode.batch_decoder(loc, local_cpr=S)}
    recs, times = {0: [], S: []}, {0: [], S: []}
    for lo in range(0, n, batch):                                       # off and on interleaved, batch by batch
        for s in (0, S):
            recs[s].append(dec[s].decode(frames[lo:lo + batch]))
            times[s].append(dec[s].stats()[1])
    raw = torch.from_numpy(frames.view(np.uint8).copy()).cuda()
    dev = {0: [], S: []}
    for _ in range(reps):
        for s in (0, S):
            dec[s].reset()
            dec[s].decode_device(raw)
            dev[s].append(dec[s].stats()[1])
    for d in dec.values():
        d.close()
    out = {"messages": n}
    ispos = np.array([t is not None for t in truth])
    out["position_messages"] = int(ispos.sum())
    for s, tag in ((0, "off"), (S, "on")):
        r = np.concatenate(recs[s])
        has = ((r["status"] & decode.FS_HAS_POS) != 0) & ispos
        out["pos_per_msg_" + tag] = round(float(has.sum()) / max(1, int(ispos.sum())), 4)
        far = np.array([bool(h) and km((r["lat"][k], r["lon"][k]), truth[k]) > far_km for k, h in enumerate(has)])
        out["far_" + tag] = int(far.sum())
        out["ms_batch_" + tag] = round(statistics.median(times[s]), 4)
        out["ms_scene_dev_" + tag] = round(statistics.median(dev[s]), 4)
        if s:
            local = (decode.local_outcome(r) == decode.LOCAL_DECODED) & ispos
            out["local_share"] = round(float(local.sum()) / max(1, int(has.sum())), 4)
            out["far_local"] = int((far & local).sum())
            out["local_outcomes"] = {name: int((decode.local_outcome(r)[ispos] == v).sum()) for name, v in (
                ("not_tried", 0), ("decoded", 1), ("no_ref", 2), ("stale", 3), ("rejected", 4))}
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=300)
    ap.add_argument("--seconds-scene", type=float, default=300.0)
    ap.add_argument("--seconds", type=int, default=30, help="local_cpr = S")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--far-km", type=float, default=1.0)
    ap.add_argument("--drops", type=str, default="0,0.5,0.8,0.9")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    result = {"card": name, "power_limit": pl, "S": args.seconds, "batch": args.batch, "far_km": args.far_km, "scenes": {}}
    loc = [48.0, 11.0]
    for drop in [float(x) for x in args.drops.split(",")]:
        for where, location in (("with_location", loc), ("no_location", None)):
            msgs, truth = lc.trajectory_scene(101, n_aircraft=args.aircraft, seconds=args.seconds_scene, drop=drop,
                                              location=tuple(loc), surface_share=0.2)
            key = "drop%.2f_%s" % (drop, where)
            result["scenes"][key] = run_scene(msgs, truth, location, args.seconds, args.batch, args.reps, args.far_km)
            print(key, json.dumps(result["scenes"][key]), flush=True)
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
