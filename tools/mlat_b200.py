"""Multilateration from K synchronized receivers' recordings: one rx_path per station, run in lockstep chunks, their
frames drained on the device (rx_path.drain_device) and handed to mlat_solver.process_device; one JSON line per fix.

    python tools/mlat_b200.py -r 4e6 --station 37.76,-122.44,100=a.cfile --station 37.68,-121.77,100=b.cfile \
        --station 37.39,-122.08,100=c.cfile [--start SECS.FRAC] [-o fixes.jsonl]

A station is LAT,LON,HEIGHT[,OFFSET]=FILE: degrees, degrees, metres above the WGS84 ellipsoid, an optional clock offset
in seconds, and a recording of complex64 samples (a GNU Radio .cfile) whose sample 0 is at --start on every station.
After each chunk the call's `end` is conservative: every station has been fed n samples, and the chain may still hold
frames that start in its last (max_late + packet_skip + shard_fwd + 4) samples (amb_geometry), so end = start + (n - that)
/ rate less the largest offset. The end of the recordings flushes.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_station(text):
    spec, _, path = text.partition("=")
    v = [float(x) for x in spec.split(",")]
    if len(v) not in (3, 4) or not path:
        raise argparse.ArgumentTypeError("station: LAT,LON,HEIGHT[,OFFSET]=FILE")
    return (v[0], v[1], v[2]), (v[3] if len(v) == 4 else 0.0), path


def parse_start(text):
    """SECS[.FRAC] as (int secs, float frac): a UTC time as one double would keep only ~2.4e-7 s."""
    whole, _, part = text.partition(".")
    return int(whole), float("0." + part) if part else 0.0


def end_stamp(start, n_fed, lookahead, rate, max_off):
    """(secs, frac) no later than any frame not yet delivered."""
    secs, frac = start
    k = max(n_fed - lookahead, 0)
    f = frac + (k % int(rate)) / rate - max_off
    s = secs + k // int(rate)
    while f < 0.0:
        f += 1.0
        s -= 1
    while f >= 1.0:
        f -= 1.0
        s += 1
    return s, f


def run(args, out):
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import mlat as ml
    stations = [s for s, _, _ in args.station]
    offsets = [o for _, o, _ in args.station]
    start = args.start
    g = am.query_geometry(args.rate, args.threshold, True)
    lookahead = g.max_late + g.packet_skip + g.shard_fwd + 4
    rx = []
    for _ in stations:
        r = am.rx_path(args.rate, args.threshold, am.msg_queue(), use_pmf=True)
        r.set_start_time(*start)
        rx.append(r)
    m = ml.mlat_solver(stations, window_us=args.window_us, offsets=offsets)
    files = [np.memmap(p, dtype=np.complex64, mode="r") for _, _, p in args.station]
    n = min(f.size for f in files)
    pos, written = 0, 0
    while pos < n:
        hi = min(pos + args.chunk, n)
        last = hi >= n
        frames = []
        for r, f in zip(rx, files):
            r.process(torch.from_numpy(np.ascontiguousarray(f[pos:hi])).cuda(), flush=last, collect=False)
            frames.append(r.drain_device())
        end = None if last else end_stamp(start, hi, lookahead, args.rate, max(offsets))
        fixes = ml.mlat_solver.fixes_from_device(m.process_device(frames, end=end, flush=last))
        for fx in fixes:
            out.write(json.dumps(ml.fix_to_dict(fx)) + "\n")
        written += len(fixes)
        pos = hi
    for r in rx:
        r.close()
    return written


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("-r", "--rate", type=float, required=True)
    ap.add_argument("--station", type=parse_station, action="append", required=True)
    ap.add_argument("-t", "--threshold", type=float, default=7.0)
    ap.add_argument("--start", type=parse_start, default=(0, 0.0), help="time of sample 0, SECS[.FRAC]")
    ap.add_argument("--window-us", type=float, default=None)
    ap.add_argument("--chunk", type=int, default=1 << 22, help="samples per station per call")
    ap.add_argument("-o", "--output", default="-")
    args = ap.parse_args(argv)
    if len(args.station) < 3:
        ap.error("at least three --station")
    out = sys.stdout if args.output == "-" else open(args.output, "w")
    try:
        n = run(args, out)
    finally:
        if out is not sys.stdout:
            out.close()
    print("%d fixes" % n, file=sys.stderr)
    return 0


if __name__ == "__main__":
    sys.exit(main())
