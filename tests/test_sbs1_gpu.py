"""Decoder option "sbs1" on the GPU (amb_decode_sbs1.cuh after every other stage, amb_decoder_sbs1 / _device): the text
byte for byte equal to the sequential checker tests/sbs1_oracle.py fed with the decoder's own records, on every scene
of tests/sbs1_cases.py with every on/off combination of local_cpr, commb, opstatus and track, also under random
splits; off = a fresh decoder (records, launch count); on = ten launches more per decode with records, track snapshots
and Comm-B / op-status bytes unchanged; host and device text byte for byte; reset; about 12,000 aircraft crossing the
window; IQ -> rx_path -> drain_device -> decode_device -> sbs1_text_device; the golden scenes of the unmodified
reference sbs1.py (tests/golden/sbs1_golden.json.gz) byte for byte, in one call and in random splits; the CLI with
-P serving a recording to a BaseStation client on loopback. Need an H100."""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_cases as dc  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import sbs1_oracle as so  # noqa: E402
import test_sbs1_golden_cpu as gold  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu
COMBOS = list(itertools.product((0, 10), (0, 30), (0, 30), (0, 20)))   # local_cpr, commb, opstatus, track


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _decoder(decode, combo, **kw):
    local, commb, ops, track = combo
    return decode.batch_decoder([47.9, 11.1], local_cpr=local, commb=commb, opstatus=ops, track=track,
                                track_ext=20 if track else 0, **kw)


def _device_text(d, n_frames):
    import torch
    out = torch.full((max(1, n_frames) * 192,), 0x5A, dtype=torch.uint8, device="cuda")
    n = d.sbs1_text_device(out)
    assert not bool((out[n:] != 0x5A).any())
    return bytes(out[:n].cpu().numpy())


def _run(decode, frames, combo, cuts, tz=0):
    d = _decoder(decode, combo, sbs1=True, sbs1_tz=tz)
    chk = so.Sbs1Checker(tz)
    out = []
    for a, b in cuts:
        recs = d.decode(frames[a:b])
        want = chk.feed(frames[a:b], recs)
        got = d.sbs1_text()
        assert got == want, (combo, a, b)
        assert _device_text(d, b - a) == got
        out.append(got)
    d.close()
    return b"".join(out)


def _cuts(n, splits):
    out, pos = [], 0
    for c in list(splits) + [n]:
        c = min(c, n - pos)
        if c > 0:
            out.append((pos, pos + c))
            pos += c
    return out


def test_every_scene_and_option_combination(decode):
    rng = np.random.default_rng(3)
    for name, msgs in sc.scenes():
        frames = tc.frames_of(msgs)
        for combo in COMBOS:
            whole = _run(decode, frames, combo, [(0, len(frames))], tz=-300 if combo[0] else 0)
            split = _run(decode, frames, combo, _cuts(len(frames), [int(x) for x in rng.integers(1, 100, 12)]),
                         tz=-300 if combo[0] else 0)
            assert whole == split, (name, combo)


def test_off_is_a_fresh_decoder_and_on_adds_ten_launches(decode):
    frames = tc.frames_of(sc.mix_scene())
    cuts = [(0, 200), (200, len(frames))]
    for combo in ((0, 0, 0, 0), (10, 30, 30, 20)):
        a = _decoder(decode, combo)
        b = _decoder(decode, combo, sbs1=True)
        c = _decoder(decode, combo, sbs1=True)
        c.set_sbs1(False)
        for lo, hi in cuts:
            ra, rb, rc = a.decode(frames[lo:hi]), b.decode(frames[lo:hi]), c.decode(frames[lo:hi])
            assert ra.tobytes() == rb.tobytes() == rc.tobytes()    # records, Comm-B and op-status bytes included
            if combo[3]:
                sa, sb, sc_ = a.aircraft_ext(), b.aircraft_ext(), c.aircraft_ext()
                for x in (sb, sc_):
                    assert sa[0].tobytes() == x[0].tobytes() and sa[1].tobytes() == x[1].tobytes()
        ka, kb, kc = a.stats()[0], b.stats()[0], c.stats()[0]
        assert kb == ka + 10 * len(cuts) and kc == ka
        for d in (a, b, c):
            d.close()


def test_reset_then_earlier_stamps(decode):
    a = tc.frames_of(sc.mix_scene(seed=4))
    b = tc.frames_of(sc.mix_scene(seed=5))
    b["secs"] -= 3600 * 24 * 400
    d = decode.batch_decoder(None, local_cpr=10, sbs1=True)
    chk = so.Sbs1Checker()
    for fr, reset in ((a, False), (b, True), (a[:100], False)):
        if reset:
            d.reset()
            chk.reset()
        recs = d.decode(fr)
        assert d.sbs1_text() == chk.feed(fr, recs)
    d.close()


def test_twelve_thousand_aircraft_cross_the_window(decode):
    d = decode.batch_decoder(None, sbs1=True)
    chk = so.Sbs1Checker()
    for msgs in sc.window_calls(n_first=12000, revisit=300) + [sc.big_call(n=12000, revisit=2000)]:
        fr = tc.frames_of(msgs, unqueued_every=0)
        recs = d.decode(fr)
        assert d.sbs1_text() == chk.feed(fr, recs)
    assert chk.n > 24000
    d.close()


def test_iq_to_text_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device -> sbs1_text_device: the text equals the host path's and
    the checker's on the drained frames."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 22
    rng = np.random.default_rng(31)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    addrs = (0xA1B2C3, 0x3C6444, 0x4840D6)
    while start < n - 2000:
        aa = addrs[sent % 3]
        kind = (sent // 3) % 3
        if kind == 0:
            frame, _ = tc.ident(aa, 4, "TEST%04d" % (sent % 10000))
        elif kind == 1:
            frame, _ = sc.df11(aa)
        else:
            frame, _ = tc.position(aa, 50.0 + 0.01 * (sent % 3), 8.0, (sent // 9) % 2, False)
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
    d = decode.batch_decoder(None, sbs1=True)
    recs_dev = d.decode_device(fr)
    out = torch.empty(fr.numel() // 80 * 192, dtype=torch.uint8, device=fr.device)
    nb = d.sbs1_text_device(out)
    got = bytes(out[:nb].cpu().numpy())
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the host path and the checker only
    h = decode.batch_decoder(None, sbs1=True)
    recs = h.decode(frames)
    host = h.sbs1_text()
    h.close()
    assert recs.tobytes() == recs_dev.cpu().numpy().tobytes()
    assert host == got == so.Sbs1Checker().feed(frames, recs)
    kinds = {ln.split(b",")[1] for ln in got.split(b"\r\n") if ln}
    assert kinds == {b"1", b"3", b"8"}


def test_golden_scenes_on_the_device(decode):
    """The device's text equals what the unmodified sbs1.py wrote for the same messages, all options off, in one call
    and in random splits."""
    rng = np.random.default_rng(17)
    for sc_ in gold.golden():
        frames = tc.frames_of([tuple(m) for m in sc_["msgs"]], unqueued_every=0)
        want = gold.golden_text(sc_)
        for cuts in ([(0, len(frames))], _cuts(len(frames), [int(x) for x in rng.integers(1, 300, 10)])):
            d = decode.batch_decoder(sc_["location"], sbs1=True)
            got = b""
            for a, b in cuts:
                d.decode(frames[a:b])
                got += d.sbs1_text()
            d.close()
            assert got == want, sc_["name"]


def test_cli_serves_a_recording_to_a_basestation_client(tmp_path):
    """tools/modes_rx_b200.py -s scene.cfile -r 4e6 -l LAT,LON -P PORT: a client on loopback reads exactly the
    checker's lines for the messages the CLI's own receive chain finds in the recording."""
    import socket
    import subprocess
    import threading
    import time
    from gr_air_modes_b200 import decode, synth
    rate, n = 4e6, 1 << 21
    rng = np.random.default_rng(41)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    while start < n - 2000:
        aa = (0x4840D6, 0x3C6444)[sent % 2]
        kind = (sent // 2) % 3
        if kind == 0:
            frame, _ = tc.ident(aa, 4, "CLITEST%d" % (sent % 10))
        elif kind == 1:
            frame, _ = sc.df11(aa)
        else:
            frame, _ = tc.position(aa, 50.0 + 0.01 * (sent % 2), 8.0, (sent // 6) % 2, False)
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 15000 + float(rng.uniform(0, 3000))
        sent += 1
    path = tmp_path / "scene.cfile"
    iq.reshape(-1).tofile(str(path))
    with socket.socket() as probe:
        probe.bind(("127.0.0.1", 0))
        port = probe.getsockname()[1]
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "modes_rx_b200.py")
    env = dict(os.environ, TZ="UTC")
    proc = subprocess.Popen([sys.executable, tool, "-s", str(path), "-r", "4e6", "-l", "50.0,8.0", "-P", str(port),
                             "--sbs1-wait", "60", "--chunk", str(1 << 19)], stdout=subprocess.PIPE,
                            stderr=subprocess.PIPE, env=env)
    try:
        for _ in range(600):
            try:
                client = socket.create_connection(("127.0.0.1", port))
                break
            except OSError:
                time.sleep(0.1)
        got = []
        reader = threading.Thread(target=lambda: got.append(b"".join(iter(lambda: client.recv(65536), b""))))
        reader.start()
        out, err = proc.communicate(timeout=600)
        reader.join(timeout=60)
        client.close()
    finally:
        if proc.poll() is None:
            proc.kill()
            proc.wait()
    assert proc.returncode == 0, err.decode()[-2000:]
    text = got[0]
    # the checker on the CLI's own messages: the printed reports come from the same decoder, so re-run the chain here
    import gr_air_modes_b200 as am
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    for a in range(0, n, 1 << 19):
        rx.process(iq.reshape(-1)[2 * a: 2 * min(n, a + (1 << 19))], flush=a + (1 << 19) >= n)
    msgs = q.strings()
    rx.close()
    h = decode.batch_decoder([50.0, 8.0])
    frames, k = decode.frames_from_messages(msgs)
    frames = np.frombuffer(bytes(frames), dtype=decode.FRAME_DTYPE)[:k].copy()
    recs = h.decode(frames)
    h.close()
    want = so.Sbs1Checker().feed(frames, recs)
    assert text == want
    kinds = {ln.split(b",")[1] for ln in text.split(b"\r\n") if ln}
    assert kinds == {b"1", b"3", b"8"}
