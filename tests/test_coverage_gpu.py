"""Decoder option "coverage" on the GPU (amb_decode_coverage.cuh after the local CPR stage, amb_decoder_coverage /
_device / _reset): the grid bit for bit equal to the sequential checker tests/coverage_oracle.py fed with the decoder's
own records, on every scene with and without a receiver location and with local_cpr on and off, in one call and under
random splits; a device-resident whole-scene call; host and device snapshots byte for byte; off = a fresh decoder
(records, launch count) for every combination of the other options; on = the same records and one launch more; resets;
10^5 positions in one call, all in one cell and spread over all 648 cells; IQ -> rx_path -> drain_device ->
decode_device -> coverage_device; the reference's grids of tests/golden/coverage_golden.json.gz. Need an H100."""
import gzip
import itertools
import json
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import coverage_oracle as co  # noqa: E402
import make_coverage_golden as mcg  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import test_coverage_cpu as cpu  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu
LOC = [47.9, 11.1]


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _device_grid(d):
    import torch
    out = torch.full((72, 9), float("nan"), dtype=torch.float64, device="cuda")
    assert d.coverage_device(out) is out
    return out.cpu().numpy()


def _run(decode, frames, cuts, loc, local_S):
    d = decode.batch_decoder(loc, local_cpr=local_S, coverage=True)
    chk = co.CoverageChecker()
    for a, b in cuts:
        recs = d.decode(frames[a:b])
        got = d.coverage()
        assert got.tobytes() == chk.feed(recs).tobytes(), (a, b)
        assert _device_grid(d).tobytes() == got.tobytes()
    d.close()
    return chk.array()


def _cuts(n, splits):
    out, pos = [], 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c > 0:
            out.append((pos, pos + c))
            pos += c
    return out


def test_every_scene_with_and_without_a_location_and_local_cpr(decode):
    rng = np.random.default_rng(3)
    for name, loc, msgs in mcg.scenes():
        frames = tc.frames_of(msgs)
        for where, local_S in itertools.product((loc, None), (0, 10)):
            whole = _run(decode, frames, [(0, len(frames))], where, local_S)
            split = _run(decode, frames, _cuts(len(frames), [int(x) for x in rng.integers(1, 400, 12)]), where, local_S)
            assert whole.tobytes() == split.tobytes(), (name, where, local_S)
            assert whole.any() == (where is not None), name


def test_a_device_resident_whole_scene_call(decode):
    import torch
    loc, msgs = [48.0, 11.0], next(m for n, _, m, _ in tc.scenes() if n == "traj")
    frames = tc.frames_of(msgs)
    want = _run(decode, frames, _cuts(len(frames), [333] * 7), loc, 10)
    d = decode.batch_decoder(loc, local_cpr=10, coverage=True)
    d.decode_device(torch.from_numpy(np.frombuffer(frames.tobytes(), dtype=np.uint8).copy()).cuda())
    assert d.coverage_device().cpu().numpy().tobytes() == d.coverage().tobytes() == want.tobytes()
    d.close()


def test_off_is_a_fresh_decoder_and_on_adds_one_launch(decode):
    frames = tc.frames_of(sc.mix_scene())
    cuts = [(0, 200), (200, len(frames))]
    for local, commb, ops, track, sbs1 in itertools.product((0, 10), (0, 30), (0, 30), (0, 20), (False, True)):
        kw = dict(local_cpr=local, commb=commb, opstatus=ops, track=track, track_ext=20 if track else 0, sbs1=sbs1)
        a = decode.batch_decoder(LOC, **kw)
        b = decode.batch_decoder(LOC, coverage=True, **kw)
        c = decode.batch_decoder(LOC, coverage=True, **kw)
        c.set_coverage(False)
        chk = co.CoverageChecker()
        for lo, hi in cuts:
            ra, rb, rc = a.decode(frames[lo:hi]), b.decode(frames[lo:hi]), c.decode(frames[lo:hi])
            assert ra.tobytes() == rb.tobytes() == rc.tobytes()
            assert b.coverage().tobytes() == chk.feed(rb).tobytes()
            if sbs1:
                assert a.sbs1_text() == b.sbs1_text()
        ka, kb, kc = a.stats()[0], b.stats()[0], c.stats()[0]
        assert kb == ka + len(cuts) and kc == ka, kw
        c.set_coverage(True)
        assert not c.coverage().any()                   # nothing was folded in while it was off
        for d in (a, b, c):
            d.close()


def test_resets(decode):
    """amb_decoder_reset clears the grid with everything else; reset_coverage clears only the grid."""
    loc, msgs = [48.0, 11.0], next(m for n, _, m, _ in tc.scenes() if n == "traj")
    frames = tc.frames_of(msgs)
    half = len(frames) // 2
    d = decode.batch_decoder(loc, local_cpr=10, coverage=True)
    ref = decode.batch_decoder(loc, local_cpr=10)
    d.decode(frames[:half])
    ref.decode(frames[:half])
    assert d.coverage().any()
    d.reset_coverage()
    assert not d.coverage().any() and not _device_grid(d).any()
    r1, r2 = d.decode(frames[half:]), ref.decode(frames[half:])
    assert r1.tobytes() == r2.tobytes()                 # the CPR state stayed
    assert d.coverage().tobytes() == co.grid_of(r1).tobytes()
    d.reset()
    ref.reset()
    assert not d.coverage().any()
    r1, r2 = d.decode(frames[:half]), ref.decode(frames[:half])
    assert r1.tobytes() == r2.tobytes() and d.coverage().tobytes() == co.grid_of(r1).tobytes()
    d.close()
    ref.close()


def _fleet(n_msgs, spread, seed):
    """n_msgs airborne positions (even/odd alternating per aircraft) around LOC: spread = False puts every aircraft in
    the cell (row 8, band 6), True puts one aircraft in each of the 648 cells (bearing 5 row, an altitude inside the
    band)."""
    rng = np.random.default_rng(seed)
    alts = (-1000, 500, 1500, 3000, 7000, 12000, 17000, 22000, 35000)
    craft = []
    if spread:
        for row in range(72):
            for band in range(9):
                craft.append((5.0 * row, 20.0 + 2.0 * band + 0.01 * row, alts[band]))
    else:
        for k in range(600):
            craft.append((40.0 + float(rng.uniform(-2.0, 2.0)), float(rng.uniform(10.0, 150.0)), 17000))
    ev = []
    per = n_msgs // len(craft) + 1
    for i, (brg, dist, alt) in enumerate(craft):
        lat = LOC[0] + dist * math.cos(math.radians(brg)) / 69.0
        lon = LOC[1] + dist * math.sin(math.radians(brg)) / (69.0 * math.cos(math.radians(LOC[0])))
        pair = [tc.position(0x100000 + i, lat, lon, odd, False, alt=alt) for odd in (0, 1)]   # the aircraft stands still
        t = float(rng.uniform(0, 1))
        for k in range(per):
            ev.append((t + 0.5 * k, *pair[k % 2]))
    return tc._msgs(ev)[:n_msgs]


@pytest.mark.parametrize("spread", [False, True], ids=["one_cell", "every_cell"])
def test_100000_positions_in_one_call(decode, spread):
    msgs = _fleet(100_000, spread, seed=5)
    frames = tc.frames_of(msgs, unqueued_every=0)
    d = decode.batch_decoder(LOC, coverage=True)
    recs = d.decode(frames)
    want = co.grid_of(recs)
    assert d.coverage().tobytes() == want.tobytes() == _device_grid(d).tobytes()
    n = sum(co.counted(r) is not None for r in recs)
    assert n > 90_000
    if spread:
        assert (want > 0).all()
    else:
        assert np.count_nonzero(want) == 3 and (want[8, 6:] > 0).all()
    d.close()


def test_iq_to_grid_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device -> coverage_device: the grid equals the host path's and
    the checker's on the drained frames."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 22
    rng = np.random.default_rng(31)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    craft = ((0xA1B2C3, 50.3, 8.4, 12000), (0x3C6444, 49.6, 7.5, 30000), (0x4840D6, 50.1, 7.9, 3000))
    while start < n - 2000:
        aa, lat, lon, alt = craft[sent % 3]
        frame, _ = tc.position(aa, lat + 0.002 * (sent // 3), lon, (sent // 3) % 2, False, alt=alt)
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 20000 + float(rng.uniform(0, 3000))
        sent += 1
    iq = iq.reshape(-1)
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    dev = torch.from_numpy(iq).cuda()
    for a, b in ((0, 1_000_000), (1_000_000, 2_500_001), (2_500_001, n)):
        rx.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx.drain_device()
    rx.close()
    loc = [50.0, 8.0]
    d = decode.batch_decoder(loc, coverage=True)
    recs_dev = d.decode_device(fr)
    got = d.coverage_device().cpu().numpy()
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the host path and the checker only
    h = decode.batch_decoder(loc, coverage=True)
    recs = h.decode(frames)
    host = h.coverage()
    h.close()
    assert recs.tobytes() == recs_dev.cpu().numpy().tobytes()
    assert got.tobytes() == host.tobytes() == co.grid_of(recs).tobytes()
    assert np.count_nonzero(got.any(axis=1)) >= 3


def _close(ours, ref):
    return ours[1] == ref[1] and all(abs(a - b) <= 1e-13 * abs(b) for a, b in ((ours[0], ref[0]), (ours[2], ref[2])))


def test_reference_grids_on_the_device(decode):
    """The device's grid against the reference az_map_output's of tests/golden/coverage_golden.json.gz, all options off,
    in one call and in random splits: the counted records are the reference's, and a cell may differ only in the row of
    a counted record whose range / bearing differs from CPython's, and then by at most 3 ulp. DESIGN.md §8 bounds the
    device's range and bearing against the same formula with correctly rounded libm calls; CPython's libm calls inside
    it may be an ulp off themselves, which a small bearing magnifies in ulps, so here a record's values are held to a
    relative 1e-13 of CPython's. Every such cell is printed."""
    with gzip.open(cpu.GOLDEN, "rb") as f:
        golden = json.loads(f.read())["scenes"]
    scenes = {name: (loc, msgs) for name, loc, msgs in mcg.scenes()}
    rng = np.random.default_rng(17)
    listed = {}
    for g in golden:
        loc, msgs = scenes[g["name"]]
        frames = tc.frames_of(msgs, unqueued_every=0)
        ref = {k: (b, a, r) for k, b, a, r in g["records"]}
        for cuts in ([(0, len(frames))], _cuts(len(frames), [int(x) for x in rng.integers(1, 300, 10)])):
            d = decode.batch_decoder(loc, coverage=True)
            recs = np.concatenate([d.decode(frames[a:b]) for a, b in cuts])
            grid = d.coverage()
            d.close()
            ours = {k: co.counted(r) for k, r in enumerate(recs) if co.counted(r) is not None}
            cells, unexplained, records = cpu.explain(grid, g["grid"], ours, ref, close=_close)
            assert not unexplained, (g["name"], unexplained)
            for i, j in cells:
                assert cpu._ulps(float(grid[i][j]), float(g["grid"][i][j])) <= 3, (g["name"], i, j)
            listed[g["name"]] = (cells, len(records))
    print("cells that differ from the reference's, by scene (cells, records whose range or bearing differs):", listed)


def test_cli_writes_the_checkers_grid(tmp_path):
    """tools/modes_rx_b200.py -s scene.cfile -r 4e6 -l LAT,LON --coverage PATH: the JSON holds coverage_to_dict of the
    checker's grid over the records of the messages the CLI's own receive chain finds in the recording."""
    import subprocess
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, synth
    rate, n = 4e6, 1 << 21
    rng = np.random.default_rng(43)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    craft = ((0x4840D6, 50.4, 8.3, 8000), (0x3C6444, 49.7, 7.6, 26000))
    while start < n - 2000:
        aa, lat, lon, alt = craft[sent % 2]
        frame, _ = tc.position(aa, lat, lon + 0.001 * (sent // 2), (sent // 2) % 2, False, alt=alt)
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 15000 + float(rng.uniform(0, 3000))
        sent += 1
    path = tmp_path / "scene.cfile"
    iq.reshape(-1).tofile(str(path))
    out = tmp_path / "cov.json"
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "modes_rx_b200.py")
    proc = subprocess.run([sys.executable, tool, "-s", str(path), "-r", "4e6", "-l", "50.0,8.0", "--coverage", str(out),
                           "--chunk", str(1 << 19)], capture_output=True, timeout=600)
    assert proc.returncode == 0, proc.stderr.decode()[-2000:]
    got = json.loads(out.read_text())
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    for a in range(0, n, 1 << 19):
        rx.process(iq.reshape(-1)[2 * a: 2 * min(n, a + (1 << 19))], flush=a + (1 << 19) >= n)
    msgs = q.strings()
    rx.close()
    h = decode.batch_decoder([50.0, 8.0])
    recs = h.decode_messages(msgs)
    h.close()
    want = co.grid_of(recs)
    assert got == json.loads(json.dumps(decode.coverage_to_dict(want, [50.0, 8.0])))
    assert np.count_nonzero(want.any(axis=1)) >= 2
