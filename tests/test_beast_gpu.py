"""The Beast binary and AVR raw feeds on the H100 (decoder options beast and avr; DESIGN.md §8 "Beast and AVR feeds"):
synthetic scenes at 4, 10 and 20 Msps through rx_path -> drain_device -> decode_device with both options on give the
bytes of tests/beast_oracle.py over the same drained frames, in host and device read-outs alike, and leave the records,
SBS-1 lines and text reports as a decoder without them writes them; the adversarial frames of the oracle module give
its bytes too; and tools/modes_rx_b200.py --beast / --avr --avr-mlat serves a recording to localhost TCP clients whose
parsed frames are the oracle's."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_oracle as bo  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def decode():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from gr_air_modes_b200 import decode as dec
    return dec


def _device_bytes(fetch, n_frames, per_frame):
    import torch
    out = torch.full((max(1, n_frames * per_frame),), 0xEE, dtype=torch.uint8, device="cuda")
    k = fetch(out)
    return bytes(out[:k].cpu().numpy())


def _check(decode, fr_dev, loc):
    """Both options on beside the SBS-1 feed and the text reports, against a decoder with only those two."""
    import torch
    fr = fr_dev.cpu().numpy().view(decode.FRAME_DTYPE)
    n = len(fr)
    on = decode.batch_decoder(loc, sbs1=True, reports=True, beast=True, avr=2)
    on1 = decode.batch_decoder(loc, avr=1)
    off = decode.batch_decoder(loc, sbs1=True, reports=True)
    try:
        recs = on.decode_device(fr_dev)
        on1.decode_device(fr_dev)
        recs_off = off.decode_device(fr_dev)
        torch.cuda.synchronize()
        assert torch.equal(recs, recs_off)
        assert on.sbs1_text() == off.sbs1_text() and on.report_text() == off.report_text()
        r = recs.cpu().numpy().view(decode.FIELDS_DTYPE)
        want_b, want_a2, want_a1 = bo.beast(fr, r), bo.avr(fr, 2, r), bo.avr(fr, 1, r)
        assert on.beast_bytes() == want_b and on.avr_text() == want_a2 and on1.avr_text() == want_a1
        assert _device_bytes(on.beast_bytes_device, n, 44) == want_b
        assert _device_bytes(on.avr_text_device, n, 43) == want_a2
        assert _device_bytes(on1.avr_text_device, n, 43) == want_a1
        assert [p for _, _, p in bo.parse_beast(want_b)] == [bo.payload(f) for f in fr[fr["passed"] != 0]]
        return fr
    finally:
        for d in (on, on1, off):
            d.close()


@pytest.mark.parametrize("rate,start", [(4e6, None), (10e6, (1_700_000_000, 0.25)), (20e6, None)])
def test_iq_to_feeds_without_leaving_the_device(decode, rate, start):
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    n = int(rate // 4e6) << 20
    sc = synth.make_scene(rate, n, 60, seed=int(rate // 1e6) + 70, garble_frac=0.2)
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, ec=4)
    if start is not None:
        rx.set_start_time(*start)
    dev = torch.from_numpy(sc.iq).cuda()
    cut = (n // 3) * 2
    rx.process(dev[:cut], collect=False)
    rx.process(dev[cut:], flush=True, collect=False)
    fr_dev = rx.drain_device()
    rx.close()
    fr = _check(decode, fr_dev, [50.0, 8.0])
    q = fr[fr["passed"] != 0]
    assert len(q) >= 20 and (fr["passed"] == 0).any()
    ts = [bo.timestamp(f["secs"], f["frac"]) for f in q]
    assert all(b >= a for a, b in zip(ts, ts[1:]))                      # one stream, no wrap at these stamps
    if start is None:                                                    # a free-running sample clock
        assert ts == [round(int(f["sample_index"]) * 12e6 / rate) for f in q]


def test_adversarial_frames(decode):
    import torch
    fr = bo.adversarial_frames()
    _check(decode, torch.from_numpy(fr.view(np.uint8).reshape(-1).copy()).cuda(), None)


def test_cli_serves_a_recording_to_beast_and_avr_clients(tmp_path):
    """tools/modes_rx_b200.py -s scene.cfile -r 4e6 -n --beast P --avr Q --avr-mlat: clients on loopback read exactly the
    oracle's bytes of the frames the CLI's own receive chain drains from the recording, chunk by chunk."""
    import socket
    import subprocess
    import threading
    import time
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, synth
    rate, n, chunk = 4e6, 1 << 21, 1 << 19
    sc = synth.make_scene(rate, n, 80, seed=77, garble_frac=0.1)
    path = tmp_path / "scene.cfile"
    sc.iq.tofile(str(path))
    ports = []
    for _ in range(2):
        with socket.socket() as probe:
            probe.bind(("127.0.0.1", 0))
            ports.append(probe.getsockname()[1])
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "modes_rx_b200.py")
    proc = subprocess.Popen([sys.executable, tool, "-s", str(path), "-r", "4e6", "-n", "--beast", str(ports[0]),
                             "--avr", str(ports[1]), "--avr-mlat", "--feed-wait", "60", "--chunk", str(chunk)],
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    got, readers, clients = {}, [], []
    try:
        for port in ports:
            for _ in range(600):
                try:
                    client = socket.create_connection(("127.0.0.1", port))
                    break
                except OSError:
                    time.sleep(0.1)
            clients.append(client)
            t = threading.Thread(target=lambda c=client, p=port: got.__setitem__(p, b"".join(iter(lambda: c.recv(65536), b""))))
            t.start()
            readers.append(t)
        out, err = proc.communicate(timeout=600)
        for t in readers:
            t.join(timeout=60)
    finally:
        for c in clients:
            c.close()
        if proc.poll() is None:
            proc.kill()
            proc.wait()
    assert proc.returncode == 0, err.decode()[-2000:]
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    frames = []
    for a in range(0, n, chunk):
        rx.process(sc.iq[2 * a: 2 * min(n, a + chunk)], flush=a + chunk >= n)
        frames += rx.frames
    rx.close()
    fr = np.frombuffer(bytes((decode.Frame * len(frames))(*frames)), dtype=decode.FRAME_DTYPE)
    q = fr[fr["passed"] != 0]
    assert len(q) >= 20
    assert got[ports[0]] == bo.beast(fr) and got[ports[1]] == bo.avr(fr, 2)
    parsed = bo.parse_beast(got[ports[0]])
    assert parsed == [(bo.timestamp(f["secs"], f["frac"]), bo.signal(f["ref_level"]), bo.payload(f)) for f in q]
    assert bo.parse_avr(got[ports[1]]) == [(t, p) for t, _, p in parsed]
