"""Decoder option "reports" on the GPU (amb_decode_reports.cuh after every other stage, amb_decoder_reports / _device):
the text byte for byte equal to report.format_report of each frame's slicer text (amb_format_message) and the
decoder's own record, on every golden scene in one call and in random splits, with the other stages on, and on every
op-status and Comm-B scene with those options on (every kind of line they add); host and
device text; off = a fresh decoder for every combination of the other options (records, launch count, SBS-1 text,
snapshots), on = three launches more with those unchanged; levels at every rssi boundary 10^(k/10) of the float32
range and their neighbours; 10^5 records in one device-resident call; IQ -> rx_path -> drain_device -> decode_device ->
report_text_device against the receive chain's own message text; the CLI printing exactly report.py's lines. Need an
H100."""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import reports_cases as rc  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import track_cases as tc  # noqa: E402
from helpers import load_decode_golden  # noqa: E402

pytestmark = pytest.mark.gpu
LOC = [47.9, 11.1]


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _device_text(d, n_frames):
    import torch
    out = torch.full((max(1, n_frames) * 480,), 0x5A, dtype=torch.uint8, device="cuda")
    n = d.report_text_device(out)
    assert not bool((out[n:] != 0x5A).any())
    return bytes(out[:n].cpu().numpy())


def _golden_frames(decode):
    for ci, case in enumerate(load_decode_golden()):
        arr, n = decode.frames_from_messages([tuple(m) for m in case["msgs"]])
        yield rc.frames_with_levels(arr, n, ci), case["location"]


def _cuts(n, sizes):
    """Consecutive non-empty pieces of the given sizes, the last one up to n (decode() of no frames leaves the last
    decode's text, as it leaves its records)."""
    out, a = [], 0
    for s in sizes:
        if a < n:
            out.append((a, min(n, a + s)))
        a = min(n, a + s)
    return out + ([(a, n)] if a < n else [])


def test_golden_scenes_in_one_call_and_in_random_splits(decode):
    rng = np.random.default_rng(11)
    for frames, loc in _golden_frames(decode):
        for cuts in ([(0, len(frames))], _cuts(len(frames), [int(x) for x in rng.integers(1, 400, 12)])):
            d = decode.batch_decoder(loc, reports=True)
            first = True
            for a, b in cuts:
                recs = d.decode(frames[a:b])
                want = rc.expected_text(frames[a:b], recs, first)
                first = False
                got = d.report_text()
                assert got == want, (a, b)
                assert _device_text(d, b - a) == got
            d.close()


def test_with_every_other_stage_on(decode):
    frames = tc.frames_of(sc.mix_scene())
    d = decode.batch_decoder(LOC, local_cpr=10, commb=30, opstatus=60, track=60, track_ext=60, sbs1=True,
                             coverage=True, reports=True)
    first = True
    for a, b in _cuts(len(frames), [300, 31, 32, 33, 1000]):
        recs = d.decode(frames[a:b])
        assert d.report_text() == rc.expected_text(frames[a:b], recs, first)
        first = False
    d.close()


def test_op_status_and_comm_b_lines(decode):
    """Every scene of the op-status and Comm-B case generators, and the op-status / Comm-B fleet of
    tests/track_ext_cases.py, with those options on, in one call and cut in three: byte for byte, and together every
    kind of line the two options add."""
    import track_ext_cases as xc
    scenes = list(rc.text_option_scenes())
    scenes.append(("ops_commb_fleet", tc.frames_of(xc.fleet(60, 20.0)), dict(commb=30, opstatus=60)))
    kinds = set()
    for name, frames, stages in scenes:
        n = len(frames)
        m = min(n, n // 3 + 33)
        for cuts in ([(0, n)], [c for c in ((0, n // 3), (n // 3, m), (m, n)) if c[0] < c[1]]):
            d = decode.batch_decoder(LOC, reports=True, **stages)
            first = True
            for a, b in cuts:
                recs = d.decode(frames[a:b])
                got = d.report_text()
                assert got == rc.expected_text(frames[a:b], recs, first), (name, a, b)
                assert _device_text(d, b - a) == got
                first = first and not np.any((recs["status"] & decode.FS_NOT_QUEUED) == 0)
                kinds |= rc.line_kinds(got)
            d.close()
    assert kinds >= rc.OPTION_LINE_KINDS, rc.OPTION_LINE_KINDS - kinds


def test_off_is_a_fresh_decoder_and_on_adds_three_launches(decode):
    frames = tc.frames_of(sc.mix_scene())
    cuts = [(0, 200), (200, len(frames))]
    for local, commb, ops, track, sbs1, cov in itertools.product((0, 10), (0, 30), (0, 30), (0, 20), (False, True),
                                                                 (False, True)):
        kw = dict(local_cpr=local, commb=commb, opstatus=ops, track=track, track_ext=20 if track else 0, sbs1=sbs1,
                  coverage=cov)
        a = decode.batch_decoder(LOC, **kw)
        b = decode.batch_decoder(LOC, reports=True, **kw)
        c = decode.batch_decoder(LOC, reports=True, **kw)
        c.set_reports(False)
        first = True
        for lo, hi in cuts:
            ra, rb, rc_ = a.decode(frames[lo:hi]), b.decode(frames[lo:hi]), c.decode(frames[lo:hi])
            assert ra.tobytes() == rb.tobytes() == rc_.tobytes()
            assert b.report_text() == rc.expected_text(frames[lo:hi], rb, first)
            first = False
            if sbs1:
                assert a.sbs1_text() == b.sbs1_text() == c.sbs1_text()
        ka, kb, kc = a.stats()[0], b.stats()[0], c.stats()[0]
        assert kb == ka + 3 * len(cuts) and kc == ka, kw
        if track:
            assert a.aircraft_ext()[0].tobytes() == b.aircraft_ext()[0].tobytes()
        if cov:
            assert a.coverage().tobytes() == b.coverage().tobytes()
        with pytest.raises(RuntimeError):
            c.report_text()
        for d in (a, b, c):
            d.close()


def test_levels_at_every_rssi_boundary(decode):
    """Float32 levels nearest 10^(k/10) for k = -80 .. 385 and their 3 neighbours each side, first message and later:
    the device's rssi equals CPython's."""
    base = np.array([np.float32(10.0 ** (k / 10.0)) for k in range(-80, 386)], dtype=np.float32)
    levels = np.concatenate([(base.view(np.int32) + i).view(np.float32) for i in range(-3, 4)])
    levels = levels[np.isfinite(levels)]
    msgs = [("5d4840d6aaaaaa", 0, 1700000000, 0.25)] * len(levels)
    arr, n = decode.frames_from_messages(msgs)
    frames = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=n).copy()
    frames["ref_level"] = levels
    for chunk in range(0, n, 997):                      # every level once as the stream's first message
        d = decode.batch_decoder(None, reports=True)
        part = np.ascontiguousarray(frames[chunk:chunk + 997])
        recs = d.decode(part)
        assert d.report_text() == rc.expected_text(part, recs, True)
        d.close()
    d = decode.batch_decoder(None, reports=True)
    for a, b in _cuts(n, [1] * 300):
        recs = d.decode(frames[a:b])
        assert d.report_text() == rc.expected_text(frames[a:b], recs, a == 0), a
    d.close()


def test_100000_records_in_one_device_resident_call(decode):
    import torch
    frames = tc.frames_of(sc.mix_scene())
    reps = 100_000 // len(frames) + 1
    big = np.concatenate([frames] * reps)[:100_000].copy()
    big["secs"] += np.repeat(np.arange(reps, dtype=np.uint64) * 1000, len(frames))[:100_000]
    d = decode.batch_decoder(LOC, reports=True, commb=30, opstatus=60)
    recs_dev = d.decode_device(torch.from_numpy(np.frombuffer(big.tobytes(), dtype=np.uint8).copy()).cuda())
    got = _device_text(d, len(big))
    d.close()
    recs = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    want = rc.expected_text(big, recs, True)
    assert got == want and got.count(b"\n") > 50_000


def _scene_iq(seed, n):
    from gr_air_modes_b200 import synth
    rate = 4e6
    rng = np.random.default_rng(seed)
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
    return rate, iq.reshape(-1)


def test_iq_to_text_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device -> report_text_device equals report.report_lines over
    the receive chain's own message text (rx_path.process with a queue) and the records of its frames."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import report
    n = 1 << 22
    rate, iq = _scene_iq(31, n)
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    dev = torch.from_numpy(iq).cuda()
    for a, b in ((0, 1_000_000), (1_000_000, 2_500_001), (2_500_001, n)):
        rx.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx.drain_device()
    rx.close()
    d = decode.batch_decoder([50.0, 8.0], reports=True)
    d.decode_device(fr)
    got = _device_text(d, fr.numel() // 80)
    d.close()
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    for a, b in ((0, 1_000_000), (1_000_000, 2_500_001), (2_500_001, n)):
        rx.process(iq[2 * a: 2 * b], flush=(b == n))
    msgs = q.strings()
    rx.close()
    h = decode.batch_decoder([50.0, 8.0])
    recs = h.decode(fr.cpu().numpy().view(decode.FRAME_DTYPE))
    h.close()
    queued = [r for r in recs if not int(r["status"]) & decode.FS_NOT_QUEUED]
    assert len(queued) == len(msgs) > 20
    want = "".join(line + "\n" for line in report.report_lines(msgs, queued)).encode()
    assert got == want


def test_cli_prints_report_py_lines_with_every_text_option(tmp_path):
    """tools/modes_rx_b200.py -s scene.cfile -l LAT,LON --commb 30 --opstatus 60 --local-cpr 10: stdout is exactly
    report.py's lines over the receive chain's messages and the records of a decoder with the same options."""
    import subprocess
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, report
    n = 1 << 21
    rate, iq = _scene_iq(43, n)
    path = tmp_path / "scene.cfile"
    iq.tofile(str(path))
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "modes_rx_b200.py")
    proc = subprocess.run([sys.executable, tool, "-s", str(path), "-r", "4e6", "-l", "50.0,8.0", "--commb", "30",
                           "--opstatus", "60", "--local-cpr", "10", "--chunk", str(1 << 19)], capture_output=True,
                          timeout=600)
    assert proc.returncode == 0, proc.stderr.decode()[-2000:]
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    want = []
    h = decode.batch_decoder([50.0, 8.0], local_cpr=10, commb=30, opstatus=60)
    seen = 0
    for a in range(0, n, 1 << 19):
        rx.process(iq[2 * a: 2 * min(n, a + (1 << 19))], flush=a + (1 << 19) >= n)
        msgs = q.strings()[seen:]                       # the chunk's messages, decoded as the CLI does per chunk
        seen += len(msgs)
        if msgs:
            want += report.report_lines(msgs, h.decode_messages(msgs))
    rx.close()
    h.close()
    assert proc.stdout.decode() == "".join(line + "\n" for line in want)
    assert len(want) > 20
