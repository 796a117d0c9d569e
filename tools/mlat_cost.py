"""Time mlat_solver.process_device on the GPU with CUDA events: K stations x F frames per call (synthetic frames in
device memory, every transmission heard by every station), printing the card's name and power limit beside the numbers.

    python tools/mlat_cost.py --stations 8 --frames 100000 --iters 20
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=8)
    ap.add_argument("--frames", type=int, default=100_000, help="frames per station per call")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import mlat_cases as mc
    from gr_air_modes_b200 import mlat as ml
    if not torch.cuda.is_available():
        sys.exit("mlat_cost: no CUDA device")
    rng = np.random.default_rng(1)
    st, c = mc.random_geometry(rng, a.stations, 200)
    planes = [(0x400000 + i, c[0] + rng.uniform(-0.3, 0.3), c[1] + rng.uniform(-0.3, 0.3), int(rng.integers(40, 1600)) * 25)
              for i in range(200)]
    # one call's worth of transmissions, 20 us apart, quantized to 20 Msps
    frames, _ = mc.scene_frames(st, planes, a.frames, rng, rate=20e6, spacing=20e-6)
    dev = [torch.from_numpy(f.view(np.uint8).copy()).cuda() for f in frames]
    m = ml.mlat_solver(st)
    out = torch.empty(a.frames * ml.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    for _ in range(a.warmup):
        got = m.process_device(dev, flush=True, out_dev=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(a.iters):
        torch.cuda.synchronize()
        e0.record()
        got = m.process_device(dev, flush=True, out_dev=out)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    s = m.stats()
    print(json.dumps({"card": card(), "stations": a.stations, "frames_per_station": a.frames,
                      "fixes_per_call": got.numel() // ml.FIX_DTYPE.itemsize, "ms_median": float(np.median(times)),
                      "ms_min": float(np.min(times)), "device_ms_last": s["ms_last"],
                      "launches_per_call": s["kernel_launches"] // (a.iters + a.warmup)}))


if __name__ == "__main__":
    main()
