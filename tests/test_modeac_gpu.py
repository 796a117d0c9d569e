"""Mode A/C replies (option "modeac") on the H100, against tests/modeac_oracle.py record for record (peak and floor bit for
bit): scenes at every supported rate, a 2^28-sample 4 Msps recording with planted replies, host and device input, cuts
into calls, the DC blocker and int16 input, the device drain, the stamps, Mode S frames unchanged by the option, and the
CLI on a recorded cfile."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import modeac_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def torch_dev():
    import torch
    return torch


def run(iq, rate, modeac=True, chunks=(), device=False, dcblock=False, sc16=False, t0=None):
    """(replies, frames as bytes, replies drained on the device as bytes or None, rx stats) of one stream."""
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, use_dcblock=dcblock, modeac=modeac)
    if t0 is not None:
        rx.set_start_time(*t0)
    data = np.clip(np.rint(iq * 32768.0), -32768, 32767).astype(np.int16) if sc16 else iq
    if device:
        torch = torch_dev()
        data = torch.from_numpy(data).cuda()
    n = iq.size // 2
    frames, pos = [], 0
    for c in list(chunks) + [n]:
        c = int(min(c, n - pos))
        last = pos + c >= n
        rx.process(data[2 * pos: 2 * (pos + c)], flush=last)
        frames += [bytes(f) for f in rx.frames]
        pos += c
        if last:
            break
    reps = rx.modeac() if modeac else None
    st = rx.stats()
    rx.close()
    return reps, frames, st


def planted_found(got, planted, rate, history):
    """How many planted replies have exactly one record within the index tolerance, with their code and SPI."""
    spc = rate / 2e6
    idx = got["sample_index"].astype(np.int64) - (history - 1)
    ok = 0
    for p in planted:
        k = np.flatnonzero((idx >= p.start - 1) & (idx <= p.start + spc))
        ok += k.size == 1 and int(got["code"][k[0]]) == p.code and int(got["spi"][k[0]]) == int(p.spi)
    return ok


@pytest.mark.parametrize("rate", [4e6, 5e6, 8e6, 10e6, 20e6])
def test_scenes_equal_the_oracle(port, rate):
    n = 1 << 22
    sc, planted = synth.make_modeac_scene(rate, n, int(n / (70 * rate / 1e6)), 60 + int(rate / 1e6), n_bursts=200)
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    got, frames, _ = run(sc.iq, rate)
    assert mo.same(got, want)
    need = len(planted) if rate >= 8e6 else int(0.985 * len(planted))
    assert planted_found(got, planted, rate, am.query_geometry(rate, 7.0, True).history) >= need
    _, frames_off, _ = run(sc.iq, rate, modeac=False)
    assert frames == frames_off and len(frames) >= 150


def test_2p28_samples_at_4msps(port):
    torch = torch_dev()
    rate, n = 4e6, 1 << 28
    sc, planted = synth.make_modeac_scene(rate, n, 20_000, 91, n_bursts=20_000)
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    dev = torch.from_numpy(sc.iq).cuda()
    for drain_on_device in (False, True):
        rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, modeac=True)
        rx.process(dev, flush=True)
        frames_on = [bytes(f) for f in rx.frames]
        if drain_on_device:
            raw = rx.modeac_device().cpu().numpy()
            got = raw.view(am.MODEAC_DTYPE)
        else:
            got = rx.modeac()
        st = rx.modeac_stats()
        rx.close()
        assert mo.same(got, want) and st.replies == len(want)
        assert planted_found(got, planted, rate, am.query_geometry(rate, 7.0, True).history) >= int(0.985 * len(planted))
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    rx.process(dev, flush=True)
    assert [bytes(f) for f in rx.frames] == frames_on and len(frames_on) >= 19_000
    rx.close()


def test_cuts_host_and_device_input(port):
    rate, n = 4e6, 1 << 21
    sc, _ = synth.make_modeac_scene(rate, n, 2000, 5, n_bursts=300)
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    rng = np.random.default_rng(9)
    cuts = [int(x) for x in rng.integers(1, 300_000, 12)] + [1, 511, 513]
    for device in (False, True):
        got, frames, _ = run(sc.iq, rate, chunks=cuts, device=device)
        assert mo.same(got, want), device


def test_dc_blocker_int16_and_stamps(port):
    rate, n = 10e6, 1 << 22
    sc, _ = synth.make_modeac_scene(rate, n, 1500, 13, n_bursts=100)
    want = mo.run_iq(port, sc.iq, rate, 7.0, use_dcblock=True)
    got, _, _ = run(sc.iq, rate, dcblock=True, chunks=[1 << 20])
    assert len(want) > 1000 and mo.same(got, want)
    q = (np.clip(np.rint(sc.iq * 32768.0), -32768, 32767) / 32768.0).astype(np.float32)
    want16 = mo.run_iq(port, q, rate, 7.0)
    got16, _, _ = run(sc.iq, rate, sc16=True, device=True)
    assert mo.same(got16, want16)
    t0 = (1_700_000_000, 0.75)
    got, _, _ = run(sc.iq, rate, t0=t0)
    r = int(rate)
    for g in got:
        cnt = int(g["sample_index"])
        secs, frac = t0[0] + cnt // r, t0[1] + (cnt % r) / r
        if frac > 1.0:
            frac -= 1.0
            secs += 1
        assert int(g["secs"]) == secs and float(g["frac"]) == frac


def test_launches_per_call():
    rate, n = 4e6, 1 << 20
    sc, _ = synth.make_modeac_scene(rate, n, 200, 3)
    counts = []
    for modeac in (False, True):
        _, _, st = run(sc.iq, rate, modeac=modeac, chunks=[n // 2], device=True)
        counts.append(st.kernel_launches)
    assert counts[1] - counts[0] == 4                # two calls, two launches each


def test_cli_on_a_recorded_cfile(port, tmp_path):
    rate, n = 4e6, 1 << 21
    sc, _ = synth.make_modeac_scene(rate, n, 1500, 21, n_bursts=200)
    path = tmp_path / "capture.cfile"
    sc.iq.tofile(path)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "modes_rx_b200.py"), "-s", str(path), "-r", "4e6",
                          "--modeac", "--chunk", str(1 << 19)], capture_output=True, text=True, check=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("modeac ")]
    msgs = [ln for ln in out.stdout.splitlines() if not ln.startswith("modeac ")]
    want = mo.run_iq(port, sc.iq, rate, 7.0)
    assert len(lines) == len(want) > 1000 and len(msgs) >= 150
    r = int(rate)
    for ln, w in zip(lines, want):
        alt = "-" if w["altitude"] == mo.NO_ALTITUDE else "%d" % w["altitude"]
        expect = "modeac %04d %s %d %.6e %.6e %d %.9f" % (w["squawk"], alt, w["spi"], float(w["peak"]), float(w["floor"]),
                                                         w["sample_index"] // r, (w["sample_index"] % r) / r)
        assert ln == expect
