"""Beast binary input on the H100 (gr_air_modes_b200.beast, DESIGN.md §8 "Beast input"): synthetic IQ at 4, 10 and
20 Msps through rx_path -> drain_device -> decode_device (option beast) -> beast_bytes_device -> beast_reader.
process_device -> decode_device, without leaving the device: the frames equal tests/beast_in_oracle.py's, the records
equal a decoder's given the oracle's frames, and the writer re-encodes the reader's frames to the very input bytes. A
stream of 2^24 bytes and more with injected garbage gives the oracle's frames and counters from host and device memory
and in random cuts. tools/modes_rx_b200.py --input beast decodes a recorded file into text reports and relays a live
loopback feed byte for byte."""
import os
import socket
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beast_in_oracle as bi  # noqa: E402
import beast_oracle as bo  # noqa: E402

pytestmark = pytest.mark.gpu
TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "modes_rx_b200.py")


@pytest.fixture(scope="module")
def torch():
    import torch as t
    if not t.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return t


def _same(got, want):
    assert len(got) == len(want)
    for name in want.dtype.names:
        assert got[name].tobytes() == want[name].tobytes(), name


def _scene_bytes(torch, rate, seed):
    """rx_path's frames of a synthetic scene written by the decoder's Beast feed, all on the device."""
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, synth
    n = int(rate // 4e6) << 20
    sc = synth.make_scene(rate, n, 60, seed=seed, garble_frac=0.2)
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True, ec=4)
    rx.process(torch.from_numpy(sc.iq).cuda(), flush=True, collect=False)
    fr_dev = rx.drain_device()
    rx.close()
    d = decode.batch_decoder([50.0, 8.0], beast=True)
    try:
        d.decode_device(fr_dev)
        out = torch.empty(44 * max(1, fr_dev.numel() // 80), dtype=torch.uint8, device="cuda")
        k = d.beast_bytes_device(out)
    finally:
        d.close()
    return out[:k]


@pytest.mark.parametrize("rate", [4e6, 10e6, 20e6])
def test_iq_to_beast_and_back_on_the_device(torch, rate):
    from gr_air_modes_b200 import beast, decode
    data_dev = _scene_bytes(torch, rate, int(rate // 1e6) + 90)
    data = bytes(data_dev.cpu().numpy())
    r = beast.beast_reader()
    try:
        fr_dev = r.process_device(data_dev, flush=True)
    finally:
        r.close()
    got = beast.beast_reader.frames_from_device(fr_dev)
    want, cnt, _ = bi.parse(data)
    _same(got, want)
    assert len(got) >= 20 and cnt["truncated"] == cnt["skipped"] == 0
    recs = []
    for src in (fr_dev, torch.from_numpy(want.view(np.uint8).reshape(-1).copy()).cuda()):
        d = decode.batch_decoder([50.0, 8.0], beast=True, sbs1=True, reports=True)
        try:
            recs.append((bytes(d.decode_device(src).cpu().numpy()), d.sbs1_text(), d.report_text(), d.beast_bytes()))
        finally:
            d.close()
    assert recs[0] == recs[1]
    assert recs[0][3] == data                          # the writer re-encodes the reader's frames to the input bytes


def test_a_long_stream_with_garbage_in_host_and_device_memory_and_cuts(torch):
    from gr_air_modes_b200 import beast
    rng = np.random.default_rng(31)
    written = bo.beast(bo.adversarial_frames())
    parts = []
    while sum(map(len, parts)) < (1 << 24) + 12345:
        parts.append(written if rng.random() < 0.7 else bi.garbage(rng, int(rng.integers(1, 5000)), 0.6))
    data = b"".join(parts)
    want, cnt, _ = bi.parse(data)
    r = beast.beast_reader()
    try:
        host = r.process(data, flush=True)
        st1 = r.stats()
        r.reset()
        dev = beast.beast_reader.frames_from_device(r.process_device(torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(),
                                                                     flush=True))
        st2 = r.stats()
        r.reset()
        cuts = sorted(set(rng.integers(0, len(data), 40).tolist()))
        bounds = [0] + cuts + [len(data)]
        pieces = [r.process(data[bounds[k]: bounds[k + 1]], flush=k == len(bounds) - 2) for k in range(len(bounds) - 1)]
        st3 = r.stats()
    finally:
        r.close()
    for got in (host, dev, np.concatenate(pieces)):
        _same(got, want)
    for st in (st1, st2, st3):
        assert {k: st[k] for k in cnt} == cnt and st["bytes_in"] == len(data)
    assert cnt["truncated"] > 0 and cnt["skipped"] > 0 and cnt["other"] > 0


def _messages(frames):
    """The message lines (amb_format_messages, the stream's first message first) of the passed frames."""
    import ctypes as C
    from gr_air_modes_b200 import _lib
    cap = 128 * len(frames) + 16
    buf = C.create_string_buffer(cap)
    k = _lib.check(_lib.load().amb_format_messages(C.c_void_p(frames.ctypes.data), len(frames), 1, buf, cap))
    return buf.value.decode("ascii").split("\n") if k else []


def test_cli_file_to_reports(torch, tmp_path):
    from gr_air_modes_b200 import decode
    data = bytes(_scene_bytes(torch, 4e6, 41).cpu().numpy())
    path = tmp_path / "feed.bin"
    path.write_bytes(data)
    out = subprocess.run([sys.executable, TOOL, "--input", "beast", "-s", str(path), "--reports", "--chunk", "5000"],
                         capture_output=True, timeout=600)
    assert out.returncode == 0, out.stderr.decode()[-2000:]
    want, _, _ = bi.parse(data)
    d = decode.batch_decoder(None, reports=True)
    try:
        d.decode_messages(_messages(want))
        text = d.report_text()
    finally:
        d.close()
    assert out.stdout == text and text.count(b"\n") >= 20
    assert ("%d Mode S frames" % len(want)) in out.stderr.decode()


def _free_ports(k):
    ports = []
    for _ in range(k):
        with socket.socket() as probe:
            probe.bind(("127.0.0.1", 0))
            ports.append(probe.getsockname()[1])
    return ports


def _connect(port, timeout=60.0):
    t0 = time.time()
    while True:
        try:
            return socket.create_connection(("127.0.0.1", port))
        except OSError:
            if time.time() - t0 > timeout:
                raise
            time.sleep(0.1)


def _listening(port) -> bool:
    """Whether a TCP socket listens on `port` (read from /proc/net/tcp, without connecting to it)."""
    for name in ("/proc/net/tcp", "/proc/net/tcp6"):
        try:
            with open(name) as f:
                rows = f.read().splitlines()[1:]
        except OSError:
            continue
        if any(r.split()[1].rsplit(":", 1)[1] == "%04X" % port and r.split()[3] == "0A" for r in rows):
            return True
    return False


def test_cli_loopback_relay(torch, tmp_path):
    """CLI 1 serves a recording's frames on --beast P1; CLI 2 reads them with --input beast -s 127.0.0.1:P1 and serves
    its own frames on --beast P2. CLI 2 waits for its client before it connects, and CLI 1 for CLI 2 before it reads
    the recording, so no byte is missed: the client of P2 reads exactly the bytes CLI 1 writes, the writer's bytes of
    the frames its receive chain drains."""
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode, synth
    rate, n, chunk = 4e6, 1 << 21, 1 << 19
    sc = synth.make_scene(rate, n, 80, seed=78, garble_frac=0.1)
    path = tmp_path / "scene.cfile"
    sc.iq.tofile(str(path))
    p1, p2 = _free_ports(2)
    procs, got, outs = [], {}, []
    client = None
    try:
        procs.append(subprocess.Popen([sys.executable, TOOL, "-s", str(path), "-r", "4e6", "-n", "--beast", str(p1),
                                       "--feed-wait", "300", "--chunk", str(chunk)],
                                      stdout=subprocess.PIPE, stderr=subprocess.PIPE))
        t0 = time.time()
        while not _listening(p1):                                # CLI 2 connects to P1 at once: it must be open
            assert time.time() - t0 < 300 and procs[0].poll() is None
            time.sleep(0.2)
        procs.append(subprocess.Popen([sys.executable, TOOL, "--input", "beast", "-s", "127.0.0.1:%d" % p1, "-n",
                                       "--beast", str(p2), "--feed-wait", "300"],
                                      stdout=subprocess.PIPE, stderr=subprocess.PIPE))
        client = _connect(p2, 300)
        t = threading.Thread(target=lambda: got.__setitem__(p2, b"".join(iter(lambda: client.recv(65536), b""))))
        t.start()
        outs = [p.communicate(timeout=600) for p in procs]
        t.join(timeout=60)
    finally:
        if client is not None:
            client.close()
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for p, (_, err) in zip(procs, outs):
        assert p.returncode == 0, err.decode()[-2000:]
    rx = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    frames = []
    for a in range(0, n, chunk):
        rx.process(sc.iq[2 * a: 2 * min(n, a + chunk)], flush=a + chunk >= n)
        frames += rx.frames
    rx.close()
    fr = np.frombuffer(bytes((decode.Frame * len(frames))(*frames)), dtype=decode.FRAME_DTYPE)
    first = bo.beast(fr)
    assert len(bo.parse_beast(first)) >= 20
    assert got[p2] == first
