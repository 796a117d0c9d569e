"""What the batch decoder's options beast and avr cost. Frames: the fleet of tests/track_cases.fleet_scene (positions,
velocities, idents, DF0/4/5/20/21 replies of --aircraft aircraft over --seconds), repeated later in time until there are
enough, with one frame in 97 not queued. For --sizes frames per call (default 10^5 and 10^6) it times
amb_decode_frames_device (device time from CUDA events around the call, amb_decoder_stats) with the options off, with
beast on, with avr = 2 on and with both on, the four decoders' calls interleaved, and reports the median of --calls
calls (at least 20) after --warmup, the kernel launches per call, and the wall clock of a read-out of the bytes to host
and to device memory. The bytes are checked against tests/beast_oracle.py on the smaller size. The card name and its
power limit are read in the same run and printed with the numbers. Needs an H100.

    python tools/beast_cost.py [--sizes 100000 1000000] [--calls 25] [--warmup 3] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import beast_oracle as bo  # noqa: E402
import track_cases as tc  # noqa: E402
from gr_air_modes_b200 import decode  # noqa: E402
from track_cost import card  # noqa: E402

CONFIGS = {"off": dict(), "beast": dict(beast=True), "avr2": dict(avr=2), "both": dict(beast=True, avr=2)}


def frames(n, args):
    base = tc.frames_of(tc.fleet_scene(args.aircraft, args.seconds))
    reps = -(-n // len(base))
    out = np.concatenate([base] * reps)[:n].copy()
    out["secs"] += np.repeat(np.arange(reps, dtype=np.uint64) * np.uint64(int(args.seconds) + 1), len(base))[:n]
    return out


def measure(fr, args, check):
    import torch
    dev = torch.from_numpy(fr.view(np.uint8).reshape(-1).copy()).cuda()
    out = torch.empty(len(fr) * 144, dtype=torch.uint8, device="cuda")
    dec = {k: decode.batch_decoder([10.0, 20.0], **v) for k, v in CONFIGS.items()}
    ms = {k: [] for k in dec}
    launches = {}
    try:
        for i in range(args.warmup + args.calls):
            for k, d in dec.items():
                k0 = d.stats()[0]
                d.decode_device(dev, out)
                n_launch, t = d.stats()
                launches[k] = n_launch - k0
                if i >= args.warmup:
                    ms[k].append(t)
        res = {"frames": len(fr), "queued": int((fr["passed"] != 0).sum())}
        for k in dec:
            res["ms_%s" % k] = round(statistics.median(ms[k]), 4)
            res["launches_%s" % k] = launches[k]
        both = dec["both"]
        buf = torch.empty(len(fr) * 44, dtype=torch.uint8, device="cuda")
        for name, host, device in (("beast", both.beast_bytes, both.beast_bytes_device),
                                   ("avr2", both.avr_text, both.avr_text_device)):
            t0 = time.perf_counter()
            data = host()
            res["ms_%s_to_host" % name] = round((time.perf_counter() - t0) * 1e3, 3)
            t0 = time.perf_counter()
            nb = device(buf)
            res["ms_%s_to_device" % name] = round((time.perf_counter() - t0) * 1e3, 3)
            res["bytes_%s" % name] = len(data)
            if check:
                recs = out.cpu().numpy().view(decode.FIELDS_DTYPE)
                want = bo.beast(fr, recs) if name == "beast" else bo.avr(fr, 2, recs)
                res["%s_equals_oracle" % name] = data == want and bytes(buf[:nb].cpu().numpy()) == want
        return res
    finally:
        for d in dec.values():
            d.close()


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
        result["sizes"][str(n)] = measure(frames(n, args), args, check=k == 0)
        print(n, json.dumps(result["sizes"][str(n)]), flush=True)
    print(json.dumps(result))
    print("card: %s, power limit %s" % (name, pl))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
