"""What the batch decoder's option "reports" costs. Scenes: the fleet of tests/track_cases.fleet_scene (positions,
velocities, idents, DF0/4/5/20/21 replies) of --aircraft aircraft over --seconds, and the op-status and Comm-B fleet of
tests/track_ext_cases.fleet of --ops-aircraft over --ops-seconds (the scene of tools/sbs1_cost.py), with a receiver
location; the decoders run with commb and opstatus on, and only reports differs. Per scene it reports, as device
time (amb_decoder_stats, CUDA events around the call):
  ms_batch_off / _on   one amb_decode_frames call of --batch frames (H2D, kernels, D2H), median over the scene's
                       batches, decoders with the option off and on interleaved
  ms_dev_off / _on     one amb_decode_frames_device call over the whole scene (median of --reps)
and, as wall clock (median of --reps):
  ms_text_host         amb_decoder_reports of the whole-scene call into host memory
  ms_text_device       amb_decoder_reports_device into device memory
  s_report_lines       report.report_lines on the host over the same messages and records (the per-message Python loop
                       the option replaces), once
with the bytes of text and of records. The text is checked against report.py on the same frames and records. The card
name and its power limit are printed with the numbers. Needs an H100.

    python tools/reports_cost.py [--aircraft 2000] [--seconds 600] [--ops-aircraft 300] [--ops-seconds 60]
                                 [--batch 4096] [--reps 7] [--json out.json]
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

import reports_cases as rc  # noqa: E402
import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
from gr_air_modes_b200 import decode, report  # noqa: E402
from track_cost import card  # noqa: E402


def measure(frames, args):
    import torch
    loc = [10.0, 20.0]
    dec = {s: decode.batch_decoder(loc, commb=30, opstatus=60, reports=bool(s)) for s in (0, 1)}
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
            recs_dev = dec[s].decode_device(raw)
            dev[s].append(dec[s].stats()[1])
    out = torch.empty(len(frames) * 480, dtype=torch.uint8, device="cuda")
    th, td = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        text = dec[1].report_text()
        th.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        n = dec[1].report_text_device(out)
        td.append((time.perf_counter() - t0) * 1e3)
    recs = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    for d in dec.values():
        d.close()
    msgs = [rc.slicer_text(f, k == 0) for k, f in enumerate(frames)]
    t0 = time.perf_counter()
    lines = report.report_lines(msgs, recs)
    s_lines = time.perf_counter() - t0
    return {"frames": len(frames), "lines": len(lines), "text_bytes": len(text), "record_bytes": recs.nbytes,
            "text_equals_report_py": text == "".join(line + "\n" for line in lines).encode("latin-1"),
            "device_equals_host": bytes(out[:n].cpu().numpy()) == text,
            "ms_batch_off": round(statistics.median(times[0]), 4), "ms_batch_on": round(statistics.median(times[1]), 4),
            "ms_dev_off": round(statistics.median(dev[0]), 4), "ms_dev_on": round(statistics.median(dev[1]), 4),
            "ms_text_host": round(statistics.median(th), 4), "ms_text_device": round(statistics.median(td), 4),
            "s_report_lines": round(s_lines, 3)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--aircraft", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--ops-aircraft", type=int, default=300)
    ap.add_argument("--ops-seconds", type=float, default=60.0)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    name, pl = card()
    result = {"card": name, "power_limit": pl, "aircraft": args.aircraft, "seconds": args.seconds,
              "ops_aircraft": args.ops_aircraft, "ops_seconds": args.ops_seconds, "batch": args.batch}
    for key, scene in (("fleet", lambda: tc.fleet_scene(args.aircraft, args.seconds)),
                       ("ops_commb_fleet", lambda: xc.fleet(args.ops_aircraft, args.ops_seconds))):
        result[key] = measure(tc.frames_of(scene(), unqueued_every=0), args)
        print(key, json.dumps(result[key]), flush=True)
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
