"""Multilateration on the H100: synthetic multi-station scenes through K rx_path contexts -> drain_device ->
mlat_solver.process_device, against the CPU checker (tests/mlat_oracle.py) over the same frames copied back, against
the truth within 4 * dop * c / rate, host path against device path byte for byte, and batch-split invariance on the
device."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mlat_cases as mc  # noqa: E402
import mlat_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu

T0 = (1_700_000_000, 0.25)
STATIONS = mc.SELFTEST_STATIONS + [(37.55, -122.25, 30.0)]
AIRCRAFT = [(0x4840D6, 37.617175, -122.400843, 8000.0), (0xA1B2C3, 37.60, -122.10, 3000.0),
            (0x3C6544, 37.70, -122.20, 11000.0), (0x7C1234, 37.50, -122.35, 6000.0)]


def run_receivers(rate, n, n_tx, seed):
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    scenes, truth = synth.make_mlat_scenes(rate, n, STATIONS, AIRCRAFT, n_tx, seed, t0=T0)
    frames_dev = []
    for sc in scenes:
        rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
        rx.set_start_time(*T0)
        rx.process(torch.from_numpy(sc.iq).cuda(), flush=True, collect=False)
        frames_dev.append(rx.drain_device().clone())
        rx.close()
    return frames_dev, truth


@pytest.mark.parametrize("rate,n,n_tx", [(20e6, 1 << 21, 80), (4e6, 1 << 19, 60)])
def test_receivers_to_fixes_on_the_device(rate, n, n_tx):
    from gr_air_modes_b200 import mlat as ml
    frames_dev, truth = run_receivers(rate, n, n_tx, seed=int(rate) % 97)
    host = [np.frombuffer(t.cpu().numpy().tobytes(), mc.FRAME) for t in frames_dev]
    assert all(len(h) >= n_tx * 9 // 10 for h in host)
    m = ml.mlat_solver(STATIONS)
    got = ml.mlat_solver.fixes_from_device(m.process_device(frames_dev, flush=True))
    ck = mo.Checker(STATIONS)
    want = ck.process(host, flush=True)
    bad = mo.compare(got, want)
    assert not bad, bad[:5]
    assert len(got) >= n_tx * 8 // 10
    s = m.stats()
    assert {k: s[k] for k in ck.counts} == ck.counts
    # the truth, within 4 dop c / rate (one sample of quantization)
    where = {tr["frame"]: tr["ecef"] for tr in truth}
    solved = [f for f in got if f["status"] == mo.SOLVED]
    assert len(solved) >= len(got) * 9 // 10
    errs = []
    for f in solved:
        e = float(np.linalg.norm(np.array([f["x"], f["y"], f["z"]]) - where[bytes(f["data"][:f["nbits"] // 8])]))
        errs.append(e)
        assert e <= 4 * f["dop"] * mo.CC / rate, (e, f["dop"])
    print("rate %.0f: %d fixes, median error %.2f m" % (rate, len(solved), float(np.median(errs))))
    # host path = device path, byte for byte
    assert ml.mlat_solver(STATIONS).process(host, flush=True).tobytes() == got.tobytes()


def test_batch_split_invariance_on_the_device():
    import torch
    from gr_air_modes_b200 import mlat as ml
    frames_dev, _ = run_receivers(20e6, 1 << 21, 80, seed=5)
    one = ml.mlat_solver(STATIONS).process_device(frames_dev, flush=True).cpu()
    host = [np.frombuffer(t.cpu().numpy().tobytes(), mc.FRAME) for t in frames_dev]
    m = ml.mlat_solver(STATIONS)
    parts = []
    for part, end in mc.split(host, T0, [0.02, 0.045, 0.07, 0.09]):
        dev = [torch.from_numpy(p.view(np.uint8).copy()).cuda() for p in part]
        parts.append(m.process_device(dev, end=end, flush=end is None).cpu())
    assert torch.cat(parts).numpy().tobytes() == one.numpy().tobytes()
    assert m.stats()["carried"] == 0


def _chain_launches(iq, rate):
    """Kernel launches of one receive chain over iq and of a batch decode of its drained frames."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200.decode import batch_decoder
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    rx.set_start_time(*T0)
    rx.process(torch.from_numpy(iq).cuda(), flush=True, collect=False)
    fr = rx.drain_device()
    chain = rx.stats().kernel_launches
    rx.close()
    d = batch_decoder()
    out = torch.empty(fr.numel() // 80 * 144, dtype=torch.uint8, device=fr.device)
    d.decode_device(fr, out)
    dec = d.stats()[0]
    d.close()
    return chain, dec, fr


def test_receive_chain_and_decoder_launch_counts_are_unchanged():
    from gr_air_modes_b200 import mlat as ml
    from gr_air_modes_b200 import synth
    scenes, _ = synth.make_mlat_scenes(4e6, 1 << 19, STATIONS, AIRCRAFT, 40, 9, t0=T0)
    before = [_chain_launches(sc.iq, 4e6) for sc in scenes]
    m = ml.mlat_solver(STATIONS)
    m.process_device([b[2] for b in before], flush=True)
    assert m.stats()["kernel_launches"] > 0
    after = [_chain_launches(sc.iq, 4e6) for sc in scenes]
    assert [b[:2] for b in before] == [a[:2] for a in after]


def test_cli_on_small_recordings(tmp_path):
    """tools/mlat_b200.py over five small cfiles in chunks that cut transmissions: its conservative ends give the fixes
    of one flushed call over the same frames."""
    import json
    import subprocess
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import mlat as ml
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 19
    scenes, _ = synth.make_mlat_scenes(rate, n, STATIONS, AIRCRAFT, 60, 13, t0=T0)
    args = [sys.executable, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools",
                                         "mlat_b200.py"), "-r", str(rate), "--start", "%d.25" % T0[0],
            "--chunk", "100000"]
    frames = []
    for k, (sc, s) in enumerate(zip(scenes, STATIONS)):
        p = tmp_path / ("s%d.cfile" % k)
        sc.iq.tofile(p)
        args += ["--station", "%r,%r,%r=%s" % (s[0], s[1], s[2], p)]
        rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
        rx.set_start_time(*T0)
        rx.process(torch.from_numpy(sc.iq).cuda(), flush=True, collect=False)
        frames.append(rx.drain_device().clone())
        rx.close()
    out = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [json.loads(x) for x in out.stdout.splitlines()]
    want = ml.mlat_solver.fixes_from_device(ml.mlat_solver(STATIONS).process_device(frames, flush=True))
    assert len(lines) == len(want) >= 50
    assert lines == [json.loads(json.dumps(ml.fix_to_dict(f))) for f in want]
