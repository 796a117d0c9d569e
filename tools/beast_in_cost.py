"""What Beast binary input (gr_air_modes_b200.beast.beast_reader) costs. Bytes: the fleet of
tests/track_cases.fleet_scene (positions, velocities, idents, DF0/4/5/20/21 replies of --aircraft aircraft over
--seconds), repeated later in time until there are --sizes frames (default 10^5 and 10^6), written as Beast binary by
tests/beast_oracle.py. For each size it times one process_device call over the whole stream in device memory (CUDA
events around the call, after torch's stream is idle) and one process call over the same bytes in pageable host
memory, and reports the median of --calls calls (at least 20) after --warmup, the achieved bytes/s and its share of the
H100 SXM's 3.35 TB/s HBM3 data-sheet bandwidth (the bound of a parse that reads every byte once), and the launches per
call. The frames are checked against tests/beast_in_oracle.py on the smaller size. The card name and its power limit
are read in the same run and printed with the numbers. Needs an H100.

    python tools/beast_in_cost.py [--sizes 100000 1000000] [--calls 25] [--warmup 3] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import beast_in_oracle as bi  # noqa: E402
import beast_oracle as bo  # noqa: E402
from beast_cost import frames  # noqa: E402
from gr_air_modes_b200 import beast  # noqa: E402
from track_cost import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def measure(data, args, check):
    import torch
    dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    host = np.frombuffer(data, np.uint8)
    r = beast.beast_reader()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms_dev, ms_host = [], []
    try:
        out = None
        for i in range(args.warmup + args.calls):
            r.reset()
            torch.cuda.synchronize()
            e0.record()
            out = r.process_device(dev, flush=True, out=out)
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                ms_dev.append(e0.elapsed_time(e1))
            r.reset()
            e0.record()
            r.process(host, flush=True)
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                ms_host.append(e0.elapsed_time(e1))
        st = r.stats()
        k0 = st["kernel_launches"]
        r.reset()
        got = beast.beast_reader.frames_from_device(r.process_device(dev, flush=True))
        st = r.stats()
        md, mh = statistics.median(ms_dev), statistics.median(ms_host)
        res = {"bytes": len(data), "frames": len(got), "ms_device": round(md, 4), "ms_host_pageable": round(mh, 4),
               "bytes_per_s_device": round(len(data) / (md * 1e-3), 0),
               "share_of_hbm_bound": round(len(data) / (md * 1e-3) / HBM_BYTES_PER_S, 4),
               "launches_per_call": st["kernel_launches"] - k0}
        if check:
            want, cnt, _ = bi.parse(data)
            res["equals_oracle"] = got.tobytes() == want.tobytes() and all(st[k] == v for k, v in cnt.items())
        return res
    finally:
        r.close()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--aircraft", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--calls", type=int, default=25)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args(argv)
    if args.calls < 20:
        ap.error("--calls: at least 20")
    name, pl = card()
    result = {"card": name, "power_limit": pl, "calls": args.calls, "sizes": {}}
    for k, n in enumerate(args.sizes):
        fr = frames(n, args)
        fr["passed"] = 1
        result["sizes"][str(n)] = measure(bo.beast(fr), args, check=k == 0)
        print(n, json.dumps(result["sizes"][str(n)]), flush=True)
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
