"""Address/parity check (option "ap_filter") on the device: fleet scenes one-shot and in ragged chunks (with cuts
between a confirmer and its subject, and a confirmer exactly S * rate_int samples before a subject in the next call),
both resolvers, both correction passes, the device-side drain and the batch decoder, one address beyond the
shared-memory tile, reset / set_rate, and 2^24-sample fleet and dense scenes - against the oracle plus the checkers of
tests/ec_oracle.py, tests/ec_any_oracle.py and tests/ap_oracle.py. Need an H100."""
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import synth
from oracle import cpu_oracle as co

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ap_cases as apc  # noqa: E402
import ap_oracle as apo  # noqa: E402
import ec_any_oracle as ea  # noqa: E402

pytestmark = pytest.mark.gpu

RATE, S = 4e6, 1


@pytest.fixture(scope="module")
def scene():
    return apc.fleet_scene(RATE, 400_000, 8, 200, seed=31)


@pytest.mark.parametrize("rate", [4e6, 10e6])
def test_fused_chain_one_shot_and_chunked(port, rate):
    n = int(200_000 * rate / 2e6)
    iq, _ = apc.fleet_scene(rate, n, 8, 200, seed=int(rate / 1e6) + 30)
    msgs, frames, st = apc.run_chain(iq, rate, S)
    _, statuses = apc.check_chain(port, iq, rate, frames, msgs, S)
    assert apc.count(statuses, apo.AP_KNOWN) >= 40 and apc.count(statuses, apo.AP_UNKNOWN) >= 2
    assert st.frames_passed == sum(f.passed for f in frames)
    idx = [int(f.sample_index) for f in frames]
    cuts = sorted({(idx[i - 1] + idx[i]) // 2 for i, f in enumerate(frames) if i and f.ap == apo.AP_KNOWN})[::7]
    rng = np.random.default_rng(6)
    for resolver in (0, 1):
        for ch in (list(np.diff([0] + cuts)), [int(x) for x in rng.integers(1, n // 3, 4)] + [1, 511, 513, 65536]):
            msgs2, frames2, _ = apc.run_chain(iq, rate, S, chunks=[int(c) for c in ch], resolver=resolver)
            assert msgs2 == msgs and [bytes(f) for f in frames2] == [bytes(f) for f in frames], resolver


def _place_exact(port, rate, n, placed, targets, seed):
    """Shift bursts by whole samples until the oracle detects burst j exactly targets[j] = (i, d) samples after burst i.
    Returns the IQ and the detection index of each placed burst (noise may add detections of its own)."""
    placed = list(placed)
    for _ in range(4):
        iq = apc.place_scene(rate, n, placed, seed)
        det = np.array([int(x) for x in port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL).index])
        idx = []
        for s, _ in placed:
            near = det[np.abs(det - s) < 40]
            assert near.size == 1, (s, near)
            idx.append(int(near[0]))
        miss = {j: idx[i] + d - idx[j] for j, (i, d) in targets.items() if idx[j] - idx[i] != d}
        if not miss:
            return iq, idx
        placed = [(s + miss.get(j, 0), f) for j, (s, f) in enumerate(placed)]
    raise AssertionError("could not place the bursts")


def test_window_edge_across_calls(port):
    w = S * int(RATE)
    rng = np.random.default_rng(32)
    a, b = 0x4840D6, 0xA1B2C3
    placed = [(5000, apc.one_frame(17, a, rng)), (15000, apc.one_frame(11, b, rng)),
              (5000 + w, apc.one_frame(20, a, rng)),
              (15000 + w + 1, apc.one_frame(11, b, rng, code=0x21))]
    iq, idx = _place_exact(port, RATE, w + 40_000, placed, {2: (0, w), 3: (1, w + 1)}, seed=3)
    cut = (idx[1] + idx[2]) // 2                                      # the subjects lie in the second call
    for chunks in ([], [cut], [cut, 7000]):
        msgs, frames, _ = apc.run_chain(iq, RATE, S, chunks=chunks)
        apc.check_chain(port, iq, RATE, frames, msgs, S)
        ours = [next(f for f in frames if f.sample_index == i) for i in idx]
        assert [f.ap for f in ours] == [0, 0, apo.AP_KNOWN, apo.AP_UNKNOWN]
        assert [f.passed for f in ours] == [1, 1, 1, 0]


def test_with_both_corrections(port):
    iq, _ = apc.fleet_scene(RATE, 400_000, 6, 200, seed=33, snr_db=(5.0, 30.0), garble_frac=0.3)
    msgs, frames, _ = apc.run_chain(iq, RATE, S, k=8, m=2)
    _, statuses = apc.check_chain(port, iq, RATE, frames, msgs, S, k=8, m=2)
    assert any(x[1] == ea.EC_FIXED for x in statuses)


def test_drain_device_and_batch_decoder(port, scene):
    import torch
    from gr_air_modes_b200 import decode
    from oracle import decode_oracle as do
    iq, _ = scene
    msgs, frames, _ = apc.run_chain(iq, RATE, S)
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True, ap_filter=S)
    dev = torch.from_numpy(iq).cuda()
    n = iq.size // 2
    for lo, hi in ((0, 100_000), (100_000, 250_001), (250_001, n)):
        rx.process(dev[2 * lo: 2 * hi], flush=(hi == n), collect=False)
    fr = rx.drain_device()
    rx.close()
    assert fr.cpu().numpy().tobytes() == b"".join(bytes(f) for f in frames)
    d = decode.batch_decoder(None)
    out = d.decode_device(fr).cpu().numpy().view(decode.FIELDS_DTYPE)
    d.close()
    known = [i for i, f in enumerate(frames) if f.ap == apo.AP_KNOWN]
    assert len(known) >= 40
    kmsgs = [m for m, f in zip(msgs, [f for f in frames if f.passed]) if f.ap == apo.AP_KNOWN]
    want = do.decode_batch([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in kmsgs], None)
    assert len(want) == len(known)
    for i, w in zip(known, want):
        g = decode.record_to_dict(out[i])
        assert (g["df"], g["icao"]) == (w["df"], w["icao"])


def test_one_address_beyond_the_tile(port):
    iq, _ = apc.fleet_scene(RATE, 1_100_000, 1, 2000, seed=34, snr_db=(10.0, 30.0))
    msgs, frames, _ = apc.run_chain(iq, RATE, S)
    _, statuses = apc.check_chain(port, iq, RATE, frames, msgs, S)
    assert sum(x[2] != apo.AP_NOT_CHECKED or x[3] == apo.CONF for x in statuses) > 1000


def test_reset_and_set_rate_clear_the_table(port, scene):
    iq, _ = scene
    half = iq.size // 4 * 2
    a, b = iq[:half], iq[half:]
    for how in ("reset", "set_rate"):
        q = am.msg_queue()
        rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ap_filter=S)
        apc.run_chain(a, RATE, S, rx=rx, q=q, close=False)
        rx.reset() if how == "reset" else rx.set_rate(RATE)
        q2 = am.msg_queue()
        rx._queue = rx._slicer._queue = q2
        rx._slicer._first = True                                       # the message precision rule restarts too
        msgs, frames, _ = apc.run_chain(b, RATE, S, rx=rx, q=q2)
        apc.check_chain(port, b, RATE, frames, msgs, S)                # b as a stream of its own
        assert rx.get_ap_filter() == S


def test_off_is_byte_identical_launches_and_refusals(port, scene):
    iq, _ = scene
    msgs0, frames0, st0 = apc.run_chain(iq, RATE, 0)
    msgs1, frames1, st1 = apc.run_chain(iq, RATE, 0, set_zero_first=True)
    assert msgs1 == msgs0 and [bytes(f) for f in frames1] == [bytes(f) for f in frames0]
    assert msgs0 == port.run_iq(iq, RATE, 7.0, True, co.MA_CANONICAL).msgs
    assert all(bytes(f.pad_) == b"\0" * 6 for f in frames0) and st1.kernel_launches == st0.kernel_launches
    _, _, st_on = apc.run_chain(iq, RATE, S)
    extra = st_on.kernel_launches - st0.kernel_launches                # four per call that slices
    assert extra > 0 and extra % 4 == 0
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True, ap_filter=60)
    for bad in (-1, 3601):
        with pytest.raises(RuntimeError):
            rx.set_ap_filter(bad)
    with pytest.raises(RuntimeError):
        rx.seek(0, 0)
    with pytest.raises(RuntimeError):
        rx.defer_resolve(True)
    rx.close()
    q = am.msg_queue()
    sl = am.slicer(q)
    sl._ctx.call("amb_set_option", b"ap_filter", 60)
    chips = np.zeros((2, 240), np.float32)
    rng = np.random.default_rng(35)
    for i, df in enumerate((17, 4)):
        c = synth.frame_chips(apc.one_frame(df, 0x3C6586, rng))
        chips[i, :c.size] = c
    assert [f.ap for f in sl.process(chips, [(0, 0.0)] * 2)] == [0, 0]


@pytest.mark.parametrize("kind", ["fleet", "dense"])
def test_long_scenes(port, kind):
    """2^24 samples: a fleet of 300 aircraft with garbling and FRUIT, and configs[4]'s traffic model (10^4 random-address
    bursts/s, 20 % garbled, FRUIT), with S = 60, every frame against the checker."""
    import torch
    n, dev0 = 1 << 24, torch.device("cuda", 0)
    nb = int(10_000 * n / RATE)
    if kind == "fleet":
        iq_dev, _ = synth.make_fleet_scene_device(RATE, n, 300, nb // 4, 7, dev0, garble_frac=0.1, fruit=nb // 8)
    else:
        iq_dev, _, _ = synth.make_scene_device(RATE, n, nb, 5, dev0, snr_db=(4.0, 30.0), garble_frac=0.2, fruit=nb // 4)
    want = port.run_iq(iq_dev.cpu().numpy(), RATE, 7.0, True, co.MA_CANONICAL)
    q = am.msg_queue()
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True, ap_filter=60)
    rx.process(iq_dev, flush=True)
    frames, msgs, st = list(rx.frames), q.strings(), rx.stats()
    rx.close()
    assert [f.sample_index for f in frames] == [int(x) for x in want.index]
    statuses = apc.check_frames(frames, want.frames, 0, 0, 60, int(RATE))
    assert msgs == apo.merged_messages(port, want.frames, 0, 0, 60, int(RATE))
    assert apc.count(statuses, apo.AP_UNKNOWN) >= 20 and st.frames_passed == sum(f.passed for f in frames)
