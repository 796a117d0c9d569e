"""The FlightGear multiplayer feed on the H100 (decoder option flightgear; DESIGN.md §8 "FlightGear multiplayer
feed"), against tests/flightgear_oracle.py over the device's own records: every byte equal except the three ECEF
doubles (each within 8 ulp) and the three orientation floats (equal or 1 float32 ulp apart), the device's sin / cos /
acos being CUDA's, not the host libm's; the histograms of both are printed. Covered: the golden scenes in one call and
in splits; the headings BDS0,9 subtype 1 words give, at positions from real CPR pairs, global and local; option off
against a fresh decoder; the chain IQ -> rx_path -> drain_device -> decode_device -> flightgear_bytes_device; and
tools/modes_rx_b200.py -m 127.0.0.1:PORT sending a recording's packets to a UDP listener."""
import collections
import gzip
import json
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_cases as dc  # noqa: E402
import flightgear_cases as fc  # noqa: E402
import flightgear_oracle as fo  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ECEF_ULP, ORIENT_ULP = 8, 1
HIST = {"ecef": collections.Counter(), "orientation": collections.Counter(), "orientation negated at angle pi": collections.Counter()}


@pytest.fixture(scope="module")
def decode():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from gr_air_modes_b200 import decode as dec
    yield dec
    for name, h in HIST.items():
        print("\nFlightGear %s ulp distance on the device: %s" % (name, dict(sorted(h.items()))))


def _ulp64(a: bytes, b: bytes) -> int:
    x, y = struct.unpack(">q", a)[0], struct.unpack(">q", b)[0]
    x, y = (x if x >= 0 else -(x & 0x7FFFFFFFFFFFFFFF)), (y if y >= 0 else -(y & 0x7FFFFFFFFFFFFFFF))
    return abs(x - y)


def _ulp32(a: bytes, b: bytes) -> int:
    x, y = struct.unpack(">i", a)[0], struct.unpack(">i", b)[0]
    x, y = (x if x >= 0 else -(x & 0x7FFFFFFF)), (y if y >= 0 else -(y & 0x7FFFFFFF))
    return abs(x - y)


def _neg_ulp(g: bytes, w: bytes):
    neg = bytes(b ^ 0x80 if i % 4 == 0 else b for i, b in enumerate(w))
    return [_ulp32(g[4 * i:4 * i + 4], neg[4 * i:4 * i + 4]) for i in range(3)]


def _negated_at_pi(g: bytes, w: bytes) -> bool:
    """The device's orientation is the checker's negated (within 1 float32 ulp each) and its angle is pi."""
    o = struct.unpack(">3f", w)
    return max(_neg_ulp(g, w)) <= ORIENT_ULP and abs(float(np.sqrt(sum(x * x for x in o))) - np.pi) < 1e-5


def same_packets(got: bytes, want: bytes, what=""):
    """Packet for packet: equal outside the ECEF and orientation fields, those within their ulp bounds."""
    P = fo.PACKET_BYTES
    assert len(got) == len(want), (what, len(got) // P, len(want) // P)
    for k in range(0, len(want), P):
        g, w = got[k:k + P], want[k:k + P]
        assert g[:144] == w[:144] and g[180:] == w[180:], (what, k // P)
        for i in range(3):
            d = _ulp64(g[144 + 8 * i:152 + 8 * i], w[144 + 8 * i:152 + 8 * i])
            HIST["ecef"][d] += 1
            assert d <= ECEF_ULP, (what, k // P, "ecef", i, d)
        e = [_ulp32(g[168 + 4 * i:172 + 4 * i], w[168 + 4 * i:172 + 4 * i]) for i in range(3)]
        if max(e) > ORIENT_ULP and _negated_at_pi(g[168:180], w[168:180]):
            # w of the product quaternion within rounding of 0: the host's cancels to 0.0 (or not) where the device's
            # does not (or does), and _set_q's sign rule flips every sign - the same rotation by pi about -axis
            HIST["orientation negated at angle pi"][max(_neg_ulp(g[168:180], w[168:180]))] += 1
            continue
        for i in range(3):
            HIST["orientation"][e[i]] += 1
            assert e[i] <= ORIENT_ULP, (what, k // P, "orientation", i, e[i])


def _device_bytes(d, n_frames):
    import torch
    out = torch.full((max(1, n_frames * fo.PACKET_BYTES),), 0xEE, dtype=torch.uint8, device="cuda")
    k = d.flightgear_bytes_device(out)
    return bytes(out[:k].cpu().numpy())


def _golden():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "flightgear_golden.json.gz")) as f:
        return json.loads(f.read())["scenes"]


@pytest.mark.parametrize("cuts", [0, 3, 17])
def test_golden_scenes_on_the_device(decode, cuts):
    """Every golden scene (every frame queued), in one call or cut into `cuts` + 1 calls: the reference's packets."""
    for scn in _golden():
        frames = tc.frames_of([tuple(m) for m in scn["msgs"]], unqueued_every=0)
        want = b"".join(bytes.fromhex(p) for o in scn["out"] for p in o[0])
        d = decode.batch_decoder(scn["location"], flightgear=True)
        try:
            got = []
            edges = np.linspace(0, len(frames), cuts + 2).astype(int)
            for lo, hi in zip(edges[:-1], edges[1:]):
                d.decode(np.ascontiguousarray(frames[lo:hi]))
                got.append(d.flightgear_bytes())
            same_packets(b"".join(got), want, scn["name"])
        finally:
            d.close()


def _heading_messages(local):
    """Every distinct heading BDS0,9 subtype 1 words give (ME subtypes 3 / 4 have none; the reference's subtype 1 is
    ME subtypes 1 and 2), over the velocity words with vew, vns in 0..1023 and both signs: one aircraft per 512 words,
    each followed by a position of that aircraft. The first two positions of an aircraft are a global pair; without
    `local` the later ones follow 0.01 s apart (global fixes), with it 15 s apart (the pair has expired), so that
    local_cpr makes them local fixes."""
    ew, ns = np.meshgrid(np.arange(1024), np.arange(1024), indexing="ij")
    ew, ns = ew.ravel().astype(float), ns.ravel().astype(float)
    with np.errstate(divide="ignore", invalid="ignore"):
        h = np.where(ns == 0, 0.0, np.degrees(np.arctan(ew / np.where(ns == 0, 1, ns))))
    _, first = np.unique(np.round(h, 9), return_index=True)        # one word per distinct heading
    words = [(int(ew[i]), int(ns[i]), s_ew, s_ns) for i in first for s_ew in (0, 1) for s_ns in (0, 1)]
    rng = np.random.default_rng(5)
    msgs, t = [], 0.0
    per = 512
    for a0 in range(0, len(words), per):
        aa = 0x10000 + a0 // per
        lat, lon = float(rng.uniform(-60, 60)), float(rng.uniform(-179, 179))
        ev = [dc.df17(aa, dc.me_ident(4, 3, "HDG%05d" % (a0 // per))), tc.position(aa, lat, lon, 0, False),
              tc.position(aa, lat, lon, 1, False)]
        for j, (vew, vns, dew, dns) in enumerate(words[a0:a0 + per]):
            ev.append(sc.velocity(aa, 1, vew, vns, dew, dns))
            ev.append(tc.position(aa, lat + 1e-4 * (j % 7), lon, j % 2, False))
        for k, (f, ecc) in enumerate(ev):
            t += 15.0 if local and k > 3 and k % 2 == 0 else 0.01
            secs = int(t)
            msgs.append((f.hex(), ecc, fc.T0 + secs, t - secs))
    return msgs


@pytest.mark.parametrize("local", [0, 600])
def test_headings_at_global_and_local_fixes(decode, local):
    frames = tc.frames_of(_heading_messages(local), unqueued_every=0)
    d = decode.batch_decoder(None, flightgear=True, local_cpr=local)
    try:
        recs = d.decode(frames)
        got = d.flightgear_bytes()
    finally:
        d.close()
    want = fo.FgChecker().feed(frames, recs)
    n_local = int(((decode.local_outcome(recs) == 1) & (recs["bds"] == 5)).sum())
    assert (n_local > 1000) == (local > 0)
    assert len(want) // fo.PACKET_BYTES > 10000
    same_packets(got, want, "headings local=%d" % local)


def test_option_off_equals_a_fresh_decoder(decode):
    frames = tc.frames_of(fc.late_scene() + fc.category_scene())
    x = decode.batch_decoder(fc.LOCATION, flightgear=True, sbs1=True)
    y = decode.batch_decoder(fc.LOCATION, sbs1=True)
    try:
        half = len(frames) // 2
        x.decode(np.ascontiguousarray(frames[:half]))
        y.decode(np.ascontiguousarray(frames[:half]))
        x.set_flightgear(False)
        rx, ry = x.decode(np.ascontiguousarray(frames[half:])), y.decode(np.ascontiguousarray(frames[half:]))
        assert rx.tobytes() == ry.tobytes() and x.sbs1_text() == y.sbs1_text()
        with pytest.raises(RuntimeError, match="option flightgear is off"):
            x.flightgear_bytes()
    finally:
        x.close()
        y.close()


def _iq_of(msgs, rate=4e6, gap_us=400.0, seed=3):
    """The messages as clean bursts at 4 Msps, gap_us apart, in noise: a recording the receive chain decodes."""
    from gr_air_modes_b200 import synth
    rng = np.random.default_rng(seed)
    spc = rate / 2e6
    step = gap_us * 1e-6 * rate
    n = int(step * (len(msgs) + 2))
    c = (rng.standard_normal((n, 2)).astype(np.float32) * np.float32(0.01)).view(np.complex64).reshape(n)
    for k, (h, _, _, _) in enumerate(msgs):
        b = synth.Burst(step * (k + 1) + 0.3, bytes.fromhex(h), 0.5, float(rng.uniform(0, 2 * np.pi)))
        n0, w = synth.burst_waveform(b, spc)
        c[n0:n0 + w.size] += w
    return c.view(np.float32).reshape(2 * n)


def test_iq_to_packets_without_leaving_the_device(decode):
    import torch
    import gr_air_modes_b200 as am
    msgs = fc.category_scene()
    iq = _iq_of(msgs)
    rx = am.rx_path(4e6, 7.0, am.msg_queue(), use_pmf=True)
    dev = torch.from_numpy(iq).cuda()
    cut = (iq.size // 4) * 2
    rx.process(dev[:cut], collect=False)
    rx.process(dev[cut:], flush=True, collect=False)
    fr_dev = rx.drain_device()
    rx.close()
    d = decode.batch_decoder(fc.LOCATION, flightgear=True)
    try:
        recs_dev = d.decode_device(fr_dev)
        got = _device_bytes(d, fr_dev.numel() // decode.FRAME_DTYPE.itemsize)
    finally:
        d.close()
    fr = fr_dev.cpu().numpy().view(decode.FRAME_DTYPE)
    recs = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    assert int((fr["passed"] != 0).sum()) >= len(msgs) - 2
    want = fo.FgChecker().feed(fr, recs)
    assert len(want) // fo.PACKET_BYTES > 100
    same_packets(got, want, "iq chain")


def test_cli_sends_a_recordings_packets_to_a_udp_listener(tmp_path):
    """tools/modes_rx_b200.py -s scene.cfile -l LAT,LON -n -m 127.0.0.1:PORT: a UDP listener receives exactly the
    packets the checker writes for the records of the CLI's own decode of its messages, chunk by chunk."""
    import socket
    import subprocess
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import decode
    msgs = fc.late_scene() + [(h, e, s + 1000, f) for h, e, s, f in fc.category_scene()]
    iq = _iq_of(msgs)
    path = tmp_path / "scene.cfile"
    iq.tofile(str(path))
    chunk = 1 << 19
    rxs = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    rxs.setsockopt(socket.SOL_SOCKET, socket.SO_RCVBUF, 8 << 20)
    rxs.bind(("127.0.0.1", 0))
    rxs.settimeout(0.5)
    tool = os.path.join(ROOT, "tools", "modes_rx_b200.py")
    proc = subprocess.Popen([sys.executable, tool, "-s", str(path), "-r", "4e6", "-n", "-l", "%g,%g" % tuple(fc.LOCATION),
                             "-m", "127.0.0.1:%d" % rxs.getsockname()[1], "--chunk", str(chunk)],
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    got = []
    try:
        while True:
            try:
                got.append(rxs.recvfrom(4096)[0])
            except socket.timeout:
                if proc.poll() is not None:
                    break
        out, err = proc.communicate(timeout=600)
    finally:
        rxs.close()
        if proc.poll() is None:
            proc.kill()
            proc.wait()
    assert proc.returncode == 0, err.decode()[-2000:]
    class texts_of(list):                           # the CLI's report_queue.handle: each message's text
        def insert_tail(self, msg):
            t = msg.to_string()
            self.append(t.decode("ascii") if isinstance(t, bytes) else t)

        handle = insert_tail

    n = iq.size // 2
    q = texts_of()
    rx = am.rx_path(4e6, 7.0, q, use_pmf=True)
    d = decode.batch_decoder(fc.LOCATION, flightgear=True)
    chk = fo.FgChecker()
    want, dev = [], []
    try:
        for a in range(0, n, chunk):
            rx.process(iq[2 * a: 2 * min(n, a + chunk)], flush=a + chunk >= n)
            texts = list(q)
            q.clear()
            if texts:
                arr, k = decode.frames_from_messages(texts)
                recs = d.decode(arr, k)
                fr = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=k)
                want.append(chk.feed(fr, recs))
                dev.append(d.flightgear_bytes())
    finally:
        rx.close()
        d.close()
    assert all(len(p) == fo.PACKET_BYTES and p[:4] == b"FGFS" for p in got)
    assert len(got) > 100
    assert b"".join(got) == b"".join(dev)
    same_packets(b"".join(got), b"".join(want), "cli")
