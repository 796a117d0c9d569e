"""What the opt-in error correction (options "ec" and "ec_any") adds on synthetic scenes, and what it costs.

For each scene (2^28 samples at 4 Msps: the configs[1] and configs[4] workloads of bench.py, and a low-SNR scene) and
each setting - "ec" = K for K in --ks alone, "ec_any" = M for M in --ec-any alone, and "ec" = 8 with "ec_any" = 2 -
next to both off, one pass of the chain over the device-resident recording reports:
  messages     frames queued (passed), corrections included
  fixed        frames a correction fixed, split by pass: fixed_ec (amb_frame.ec == AMB_EC_FIXED) and fixed_any
               (AMB_FRAME_EC_ANY == AMB_EC_FIXED)
  true / false fixed frames whose corrected payload is / is not one of the frames the scene generated, before or
               after garbling
  ms_step      device time of one pass (CUDA events on the caller's stream, process -> join), median over the
               steps; passes with the options off and on alternate in the same process
The synthetic scenes garble bits BEFORE modulation, so those errors are high-confidence: "ec", which only flips
low-confidence bits, is not expected to recover them; "ec_any" is. The card name and its power limit are printed with
the numbers. Needs an H100.

    python tools/ec_yield.py [--steps 5] [--log2n 28] [--ks 4,8,12] [--ec-any 1,2] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np

FIXED = 1   # AMB_EC_FIXED

SCENES = {   # bench.py's configs[1] / configs[4] scene arguments, and a low-SNR variant of configs[1]
    "configs[1]": dict(seed=0, snr_db=(6.0, 30.0), bursts_per_s=None, n_bursts=1000, garble_frac=0.0, fruit=False),
    "configs[4]": dict(seed=5, snr_db=(4.0, 30.0), bursts_per_s=10_000, n_bursts=None, garble_frac=0.2, fruit=True),
    "low_snr": dict(seed=41, snr_db=(3.0, 9.0), bursts_per_s=10_000, n_bursts=None, garble_frac=0.0, fruit=False),
}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out or "unknown"


def clean_frames(rate, n, nb, seed, garbled, nbytes):
    """The frames synth.make_scene_device generated before garbling them: its random draws replayed up to
    make_frames, with garble_frac 0. Checked against the garbled frames (equal, or at most 5 bits apart)."""
    from gr_air_modes_b200 import synth
    rng = np.random.Generator(np.random.PCG64(seed))
    span = 240 * rate / 2e6 + 8
    rng.uniform(span, n - 2 * span, nb)
    dfs = np.asarray((11, 17))[rng.integers(0, 2, nb)]
    clean, nb2 = synth.make_frames(dfs, rng, 0.0)
    diff = np.unpackbits(clean ^ garbled, axis=1).sum(axis=1)
    assert np.array_equal(nb2, nbytes) and diff.max() <= 5, "replay of make_scene_device out of step"
    return {clean[k, :nbytes[k]].tobytes() for k in range(nb)}


def one_pass(rx, dev, torch):
    """Device time of one pass over `dev` (a fresh stream), in ms; the frames stay on the context."""
    rx.reset()
    rx._slicer._first = True
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    rx.process(dev, flush=True, collect=False)
    rx.join()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def main():
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--ks", default="4,8,12")
    ap.add_argument("--ec-any", default="1,2")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    rate, n = 4e6, 1 << args.log2n
    dev0 = torch.device("cuda", 0)
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    rows = []
    for scene, cfg in SCENES.items():
        nb = cfg["n_bursts"] or int(cfg["bursts_per_s"] * n / rate)
        iq, _, (fr, nbytes) = synth.make_scene_device(rate, n, nb, cfg["seed"], dev0, noise_sigma=0.01, snr_db=cfg["snr_db"],
                                                      garble_frac=cfg["garble_frac"], fruit=nb // 4 if cfg["fruit"] else 0)
        sent = {fr[k, :nbytes[k]].tobytes() for k in range(nb)} | clean_frames(rate, n, nb, cfg["seed"], fr, nbytes)
        stream = torch.cuda.current_stream(dev0).cuda_stream
        off = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
        off.use_stream(stream)
        one_pass(off, iq, torch)                                  # warm-up
        base = off.drain()
        settings = [(int(k), 0) for k in args.ks.split(",") if k] + [(0, int(m)) for m in args.ec_any.split(",") if m]
        settings.append((8, 2))
        for k, m in settings:
            on = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, ec=k, ec_any=m)
            on.use_stream(stream)
            one_pass(on, iq, torch)
            msgs = on.drain()
            frames = on.frames
            fixed = [f for f in frames if f.ec == FIXED or f.ec_any == FIXED]
            true = sum(f.payload() in sent for f in fixed)
            t_off, t_on = [], []
            for _ in range(args.steps):                           # off and on alternate
                t_off.append(one_pass(off, iq, torch))
                t_on.append(one_pass(on, iq, torch))
            off.drain()
            on.drain()
            row = dict(scene=scene, samples=n, bursts=nb, k=k, m=m, messages_off=base, messages=msgs, fixed=len(fixed),
                       fixed_ec=sum(f.ec == FIXED for f in fixed), fixed_any=sum(f.ec_any == FIXED for f in fixed),
                       true_fixes=true, false_fixes=len(fixed) - true, ms_step_off=round(statistics.median(t_off), 3),
                       ms_step_on=round(statistics.median(t_on), 3), card=name, power_limit=power)
            rows.append(row)
            print(json.dumps(row), flush=True)
            on.close()
        off.close()
        del iq
        torch.cuda.empty_cache()
    print("\n%-11s %3s %2s %9s %9s %7s %7s %6s %6s %9s %9s" % ("scene", "K", "M", "msgs_off", "msgs_on", "fix_ec",
                                                              "fix_any", "true", "false", "ms_off", "ms_on"))
    for r in rows:
        print("%-11s %3d %2d %9d %9d %7d %7d %6d %6d %9.3f %9.3f" % (
            r["scene"], r["k"], r["m"], r["messages_off"], r["messages"], r["fixed_ec"], r["fixed_any"], r["true_fixes"],
            r["false_fixes"], r["ms_step_off"], r["ms_step_on"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
