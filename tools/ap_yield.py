"""What the opt-in address/parity check (option "ap_filter") removes and accepts on synthetic scenes, and what it costs.

Scenes (4 Msps, 2^28 samples by default): bench.py's configs[1] and configs[4] workloads (tools/ec_yield.py), which send
only DF11/DF17 with II = 0 - so every address/parity reply and every II/SI reply there is garbage, garbled squitters
included - and a fleet scene (synth.make_fleet_scene_device: 300 aircraft sending DF17, DF11 with and without an II
code, and DF0/4/5/16/20/21 replies, with FRUIT and overlapping bursts; no garbling, so what it sent is known exactly). With S = --seconds, one pass of the chain over the device-resident recording
reports per scene:
  messages_off / messages_on   frames queued with the option off / on
  garbage_dropped / _kept      AP subjects (passed DF not in {11, 17}) that the scene did not send, dropped / accepted
                               (accepted = their syndrome happens to be a confirmed address)
  true_dropped                 AP subjects the scene did send, dropped (cold start: before their aircraft's first
                               confirmer, or after a gap longer than S)
  iisi_true / iisi_false       DF11 II/SI replies accepted, sent by the scene / not
  ms_step_off / ms_step_on     device time of one pass, median over --steps passes, off and on alternating
The card name and its power limit are printed with the numbers. Needs an H100.

    python tools/ap_yield.py [--steps 5] [--log2n 28] [--seconds 60] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import ec_yield as ey  # noqa: E402

KNOWN, UNKNOWN = 1, 2   # AMB_AP_KNOWN, AMB_AP_UNKNOWN
FLEET = dict(seed=61, n_aircraft=300, bursts_per_s=2_000, snr_db=(6.0, 30.0), garble_frac=0.0, fruit=True)


def tally(frames, sent):
    g_drop = g_keep = t_drop = ii_t = ii_f = 0
    for f in frames:
        if f.ap == 0:
            continue
        ours = f.payload() in sent
        if f.df == 11:
            if f.ap == KNOWN:
                ii_t += ours
                ii_f += not ours
        elif f.ap == UNKNOWN:
            t_drop += ours
            g_drop += not ours
        else:
            g_keep += not ours
    return dict(garbage_dropped=g_drop, garbage_kept=g_keep, true_dropped=t_drop, iisi_true=ii_t, iisi_false=ii_f)


def main():
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    rate, n = 4e6, 1 << args.log2n
    dev0 = torch.device("cuda", 0)
    name, power = ey.card()
    print("card: %s, power limit %s" % (name, power))
    rows = []
    for scene in ("configs[1]", "configs[4]", "fleet"):
        if scene == "fleet":
            cfg = FLEET
            nb = int(cfg["bursts_per_s"] * n / rate)
            iq, (fr, nbytes, _, _) = synth.make_fleet_scene_device(
                rate, n, cfg["n_aircraft"], nb, cfg["seed"], dev0, snr_db=cfg["snr_db"], garble_frac=cfg["garble_frac"],
                fruit=nb // 4 if cfg["fruit"] else 0)
            sent = {fr[k, :nbytes[k]].tobytes() for k in range(nb)}
        else:
            cfg = ey.SCENES[scene]
            nb = cfg["n_bursts"] or int(cfg["bursts_per_s"] * n / rate)
            iq, _, (fr, nbytes) = synth.make_scene_device(rate, n, nb, cfg["seed"], dev0, noise_sigma=0.01,
                                                          snr_db=cfg["snr_db"], garble_frac=cfg["garble_frac"],
                                                          fruit=nb // 4 if cfg["fruit"] else 0)
            sent = set()                                          # only DF11/DF17 with II = 0: no subject is true
        stream = torch.cuda.current_stream(dev0).cuda_stream
        off = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
        on = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, ap_filter=args.seconds)
        for rx in (off, on):
            rx.use_stream(stream)
            ey.one_pass(rx, iq, torch)                            # warm-up (and the table's allocation)
        msgs_off = off.drain()
        msgs_on = on.drain()
        row = dict(scene=scene, samples=n, bursts=nb, seconds=args.seconds, messages_off=msgs_off, messages_on=msgs_on,
                   **tally(on.frames, sent))
        t_off, t_on = [], []
        for _ in range(args.steps):
            t_off.append(ey.one_pass(off, iq, torch))
            t_on.append(ey.one_pass(on, iq, torch))
        off.drain()
        on.drain()
        row.update(ms_step_off=round(statistics.median(t_off), 3), ms_step_on=round(statistics.median(t_on), 3),
                   card=name, power_limit=power)
        rows.append(row)
        print(json.dumps(row), flush=True)
        off.close()
        on.close()
        del iq
        torch.cuda.empty_cache()
    print("\n%-11s %9s %9s %8s %8s %8s %7s %7s %8s %8s" % ("scene", "msgs_off", "msgs_on", "g_drop", "g_keep", "t_drop",
                                                          "ii_t", "ii_f", "ms_off", "ms_on"))
    for r in rows:
        print("%-11s %9d %9d %8d %8d %8d %7d %7d %8.3f %8.3f" % (
            r["scene"], r["messages_off"], r["messages_on"], r["garbage_dropped"], r["garbage_kept"], r["true_dropped"],
            r["iisi_true"], r["iisi_false"], r["ms_step_off"], r["ms_step_on"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
