"""SURVEY.md 8 row f4 on the GPU: amb_decoder (fields / CPR pairing / resolve kernels) against the reference's golden
and the CPU oracle. Named test_zz_* so that it runs after the hot-path parity tests.

Tolerances: integers, strings, status flags exact. Latitude/longitude: the kernels use only IEEE +,-,*,/,floor,fmod in
double with -fmad=false and are bit-identical to the reference's on the golden set (asserted there); the seeded
oracle comparisons use 1e-12 relative. Velocity/heading/range/bearing go through hypot/atan2/sin/cos/pow, where CUDA's and glibc's last place
differ: 1e-12 relative.
"""
import math

import numpy as np
import pytest

from helpers import compare_decode, load_decode_golden

pytestmark = pytest.mark.gpu
TOL = 1e-12


@pytest.fixture()
def dec_mod():
    from gr_air_modes_b200 import decode
    return decode


def _dicts(decode, out):
    return [decode.record_to_dict(r) for r in out]


def _same(a, b, where):
    """Two product records must be identical (chunking / batching must not change a single bit)."""
    for k, v in a.items():
        w = b[k]
        for x, y in (zip(v, w) if isinstance(v, list) else [(v, w)]):
            assert x == y or (isinstance(x, float) and math.isnan(x) and math.isnan(y)), (where, k, a, b)


def test_decode_matches_reference_golden(dec_mod):
    n = exact = npos = 0
    for ci, case in enumerate(load_decode_golden()):
        d = dec_mod.batch_decoder(case["location"])
        recs = _dicts(dec_mod, d.decode_messages([tuple(m) for m in case["msgs"]]))
        assert d.stats()[0] == 7                       # fields + five pairing kernels (bucket partition) + resolve
        d.close()
        assert len(recs) == len(case["ref"])
        for k, (rec, ref) in enumerate(zip(recs, case["ref"])):
            compare_decode(rec, ref, TOL, "case %d msg %d" % (ci, k))
            if "pos" in ref:
                npos += 1
                exact += (rec["lat"] == ref["pos"][0] and rec["lon"] == ref["pos"][1])
            n += 1
    print("decode golden: %d messages, %d positions, %d bit-identical lat/lon" % (n, npos, exact))
    assert n > 5000 and npos > 2000
    assert exact == npos            # every latitude/longitude bit-identical to the reference's


def test_decode_equals_oracle_record_for_record(dec_mod):
    import decode_cases
    from oracle import decode_oracle as do
    for seed, loc in ((301, (35.7, 139.7)), (302, None), (303, (-54.8, -68.3))):
        loc_, msgs = decode_cases.make_case(seed, location=loc, seconds=30.0, surface_share=0.4, n_random=600)
        want = do.decode_batch(msgs, loc_)
        d = dec_mod.batch_decoder(loc_)
        got = _dicts(dec_mod, d.decode_messages(msgs))
        d.close()
        for k, (g, w) in enumerate(zip(got, want)):
            for key, wv in w.items():
                near = key in ("val", "range", "bearing", "lat", "lon")
                gv = g[key]
                for a, b in (zip(gv, wv) if isinstance(wv, list) else [(gv, wv)]):
                    if isinstance(b, float) and math.isnan(b):
                        assert math.isnan(a), (seed, k, key, g, w)
                    elif near:
                        assert abs(a - b) <= TOL * max(1.0, abs(b)), (seed, k, key, g, w)
                    else:
                        assert a == b, (seed, k, key, g, w)


def test_batching_does_not_change_results(dec_mod):
    """The report table carries the per-aircraft state from batch to batch like one cpr_decoder instance: any
    chunking of the stream (down to single messages, and chunk edges inside a 32-frame step) gives identical records."""
    import decode_cases
    loc, msgs = decode_cases.make_case(401, location=(52.3, 4.8), seconds=30.0, surface_share=0.3, n_random=300)
    d = dec_mod.batch_decoder(loc)
    one = _dicts(dec_mod, d.decode_messages(msgs))
    rng = np.random.default_rng(1)
    for plan in ("ones", "odd", "random"):
        d.reset()
        got, pos = [], 0
        while pos < len(msgs):
            c = 1 if plan == "ones" and pos < 200 else (33 if plan == "odd" else int(rng.integers(1, 400)))
            got += _dicts(dec_mod, d.decode_messages(msgs[pos:pos + c]))
            pos += c
        assert len(got) == len(one)
        for k, (a, b) in enumerate(zip(got, one)):
            _same(a, b, (plan, k))
    d.close()


def test_pairing_inside_one_step_and_across_many_warps(dec_mod):
    """Stress of the pairing kernel: a few aircraft sending even/odd reports back to back (several reports of one
    aircraft inside one 32-frame step, both formats, equal timestamps), then a large batch spread over many warps."""
    import decode_cases as dc
    from oracle import decode_oracle as do
    rng = np.random.default_rng(7)
    msgs, t = [], 0.0
    craft = [(int(rng.integers(1, 1 << 24)), 40.0 + rng.uniform(-1, 1), -3.0 + rng.uniform(-1, 1)) for _ in range(3)]
    for k in range(4000):
        aa, lat, lon = craft[int(rng.integers(0, len(craft)))]
        odd = int(rng.integers(0, 2))
        surface = rng.random() < 0.25
        la, lo = dc.cpr_encode(lat + 1e-4 * rng.standard_normal(), lon + 1e-4 * rng.standard_normal(), odd, surface)
        me = dc.me_surface(6, 10, 1, 5, odd, la, lo) if surface else dc.me_airborne(11, dc.enc_alt12(30000), odd, la, lo)
        frame, ecc = dc.df17(aa, me)
        if rng.random() < 0.7:
            t += float(rng.choice([0.0, 1e-4, 0.3]))       # equal timestamps happen
        if k == 2000:
            t += 30.0                                      # everything expires once
        msgs.append((frame.hex(), ecc, int(t), t - int(t)))
    loc = (40.4, -3.7)
    want = do.decode_batch(msgs, loc)
    d = dec_mod.batch_decoder(loc)
    got = _dicts(dec_mod, d.decode_messages(msgs))
    for k, (g, w) in enumerate(zip(got, want)):
        assert g["status"] == w["status"], (k, g, w)
        if w["status"] & do.FS_HAS_POS:
            assert abs(g["lat"] - w["lat"]) <= TOL * 90 and abs(g["lon"] - w["lon"]) <= TOL * 180, (k, g, w)
    assert sum(1 for w in want if w["status"] & do.FS_HAS_POS) > 2000

    # large batch: ~60 k messages of 300 aircraft -> more than 200 pairing warps, each owning a share of the aircraft
    big, t = [], 0.0
    fleet = [(int(a), float(rng.uniform(-60, 60)), float(rng.uniform(-170, 170))) for a in rng.choice(1 << 24, 300, replace=False)]
    for k in range(60000):
        aa, lat, lon = fleet[int(rng.integers(0, len(fleet)))]
        odd = int(rng.integers(0, 2))
        la, lo = dc.cpr_encode(lat, lon, odd, False)
        frame, ecc = dc.df17(aa, dc.me_airborne(12, dc.enc_alt12(12000), odd, la, lo))
        t += 2e-4
        big.append((frame.hex(), ecc, int(t), t - int(t)))
    want = do.decode_batch(big, loc)
    d.reset()
    arr, nbig = dec_mod.frames_from_messages(big)
    got = d.decode(arr, nbig)
    print("decode of %d frames: %.3f ms on the device (H2D + 3 kernels + D2H)" % (nbig, d.stats()[1]))
    assert got.size == len(want)
    st = np.array([w["status"] for w in want], dtype=np.uint8)
    assert np.array_equal(got["status"], st)
    ok = (st & do.FS_HAS_POS) != 0
    wl = np.array([w["lat"] for w in want])
    wo = np.array([w["lon"] for w in want])
    assert ok.sum() > 50000
    assert np.all(np.abs(got["lat"][ok] - wl[ok]) <= TOL * 90) and np.all(np.abs(got["lon"][ok] - wo[ok]) <= TOL * 180)
    d.close()


def test_not_queued_frames_reset_and_location(dec_mod):
    import decode_cases as dc
    aa = 0x4840D6
    la0, lo0 = dc.cpr_encode(52.25, 3.92, 0)
    la1, lo1 = dc.cpr_encode(52.25, 3.92, 1)
    f0, e0 = dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(38000), 0, la0, lo0))
    f1, e1 = dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(38000), 1, la1, lo1))
    arr, n = dec_mod.frames_from_messages([(f0.hex(), e0, 0, 0.1), (f1.hex(), e1, 0, 0.6)])
    d = dec_mod.batch_decoder(None)
    out = d.decode(arr, n)
    assert out["status"][0] & dec_mod.FS_CPR_NO_POS and out["status"][1] & dec_mod.FS_HAS_POS
    assert not (out["status"][1] & dec_mod.FS_HAS_RANGE)
    assert abs(out["lat"][1] - 52.25) < 1e-3 and abs(out["lon"][1] - 3.92) < 1e-3 and out["altitude"][1] == 38000
    # a frame the slicer did not queue is not decoded and leaves no report behind
    d.reset()
    arr[0].passed = 0
    out = d.decode(arr, n)
    assert out["status"][0] == dec_mod.FS_NOT_QUEUED and out["status"][1] & dec_mod.FS_CPR_NO_POS
    # reset() forgets the reports; set_location() turns range/bearing on (cpr.py:192-193, 233-237)
    arr[0].passed = 1
    d.reset()
    d.set_location([52.0, 4.0])
    out = d.decode(arr, n)
    assert out["status"][1] & dec_mod.FS_HAS_RANGE and 0 < out["range"][1] < 30 and 0 <= out["bearing"][1] < 360
    d.reset()
    out = d.decode(arr[1:2], 1)
    assert out["status"][0] & dec_mod.FS_CPR_NO_POS
    assert d.decode(arr, 0).size == 0
    d.close()


def test_receive_chain_to_positions(port):
    """IQ -> rx_path (hot path) -> frames -> batch_decoder: the decoded records equal the oracle's decode of the
    message strings the slicer queued."""
    import gr_air_modes_b200 as am
    import decode_cases as dc
    from gr_air_modes_b200 import decode, synth
    from oracle import decode_oracle as do
    rate, n = 4e6, 1 << 21
    rng = np.random.default_rng(21)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, odd, sent = 3000.0, 0, 0
    while start < n - 2000:
        aa = (0x3C6444, 0xA1B2C3)[sent % 2]
        lat, lon = (50.03 + 1e-4 * sent, 8.57) if sent % 2 == 0 else (49.9, 8.2 + 1e-4 * sent)
        la, lo = dc.cpr_encode(lat, lon, odd, False)
        frame, _ = dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(10000 + 25 * sent), odd, la, lo))
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 20000 + float(rng.uniform(0, 3000))
        sent += 1
        if sent % 2 == 0:
            odd ^= 1
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    rx.process(iq.reshape(-1), flush=True)
    msgs = q.strings()
    assert len(msgs) >= sent
    d = decode.batch_decoder([50.0, 8.5])
    out = d.decode(rx.frames)
    d.close()
    queued = [decode.record_to_dict(r) for r, f in zip(out, rx.frames) if f.passed]
    assert all(r["status"] == decode.FS_NOT_QUEUED for r, f in zip(out, rx.frames) if not f.passed)
    want = do.decode_batch([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in msgs], [50.0, 8.5])
    assert len(queued) == len(want)
    npos = 0
    for k, (g, w) in enumerate(zip(queued, want)):
        assert (g["df"], g["icao"], g["status"], g["altitude"], g["bds"]) == (w["df"], w["icao"], w["status"], w["altitude"], w["bds"]), (k, g, w)
        if w["status"] & do.FS_HAS_POS:
            npos += 1
            assert abs(g["lat"] - w["lat"]) <= TOL * 90 and abs(g["lon"] - w["lon"]) <= TOL * 180
            assert abs(g["range"] - w["range"]) <= 1e-9 and abs(g["bearing"] - w["bearing"]) <= 1e-9
    assert npos >= sent - 6


def _position_scene(rate, n, seed):
    import decode_cases as dc
    from gr_air_modes_b200 import synth
    rng = np.random.default_rng(seed)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, odd, sent = 3000.0, 0, 0
    while start < n - 2000:
        aa = (0x3C6444, 0xA1B2C3)[sent % 2]
        lat, lon = (50.03 + 1e-4 * sent, 8.57) if sent % 2 == 0 else (49.9, 8.2 + 1e-4 * sent)
        la, lo = dc.cpr_encode(lat, lon, odd, False)
        if sent % 7 == 3:
            me = dc.me_ident(4, 3, "DLH%03d" % sent)
        elif sent % 7 == 5:
            me = dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(15, 10, 200 + sent).put(26, 10, 300).put(38, 9, 17).v
        else:
            me = dc.me_airborne(11, dc.enc_alt12(10000 + 25 * sent), odd, la, lo)
        frame, _ = dc.df17(aa, me)
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 20000 + float(rng.uniform(0, 3000))
        sent += 1
        if sent % 2 == 0:
            odd ^= 1
    return iq.reshape(-1), sent


def test_cli_prints_the_reference_printers_reports(port, tmp_path):
    """Row f1 + f4: `modes_rx_b200.py -l LAT,LON` prints what apps/modes_rx prints by default - the text reports of
    python/msprint.py. Expected lines: the oracle's messages, decoded by the decode oracle, formatted by report.py
    (which tests/test_decode_cpu.py pins line for line against the unmodified msprint.py)."""
    import os
    import subprocess
    import sys
    from gr_air_modes_b200 import report
    from oracle import cpu_oracle as co
    from oracle import decode_oracle as do
    rate, n = 4e6, 1 << 20
    iq, sent = _position_scene(rate, n, 33)
    msgs = port.run_iq(iq, rate, 7.0, True, co.MA_CANONICAL).msgs
    recs = do.decode_batch([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in msgs], [50.0, 8.5])
    want = report.report_lines(msgs, recs)
    assert sum("position report" in ln for ln in want) >= sent // 2 and any("ident DLH" in ln for ln in want)
    assert any("track report" in ln for ln in want)
    path = tmp_path / "pos.cfile"
    iq.tofile(path)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for chunk in ("300001", str(1 << 24)):
        out = subprocess.run([sys.executable, os.path.join(root, "tools", "modes_rx_b200.py"), "-s", str(path), "-r", "4e6",
                              "-l", "50.0,8.5", "--chunk", chunk], capture_output=True, text=True, check=True).stdout.split("\n")
        assert [ln for ln in out if ln] == want


def test_cpr_decoder_dropin_class(dec_mod):
    """decode.cpr_decoder = the reference's cpr_decoder API (cpr.py:183-240) one message per call on the GPU decoder;
    against the decode oracle's CprState on one injected clock (the class itself is pinned against the unmodified
    reference class in tests/test_decode_cpu.py with the host build of the same arithmetic)."""
    import decode_cases as dc
    from gr_air_modes_b200.errors import CPRBoundaryStraddleError, CPRNoPositionError
    from oracle import decode_oracle as do
    now = [1000.0]
    loc = [35.0, -100.0]
    ours = dec_mod.cpr_decoder(list(loc), clock=lambda: now[0])
    ref = do.CprState(list(loc))
    ok = 0
    for i in range(300):
        lat, lon = i / (300 / 170.) - 85, i / (300 / 360.) - 180
        surface = int(i % 5 == 0)
        if surface:
            lat, lon = 35.0 + i * 1e-3, -100.0 + i * 1e-3
        icao = (i * 7919) & 0xFFFFFF
        now[0] += 0.3 + (30.0 if i == 150 else 0.0)
        for odd, dl in ((0, 0.0), (1, 1e-3)):
            la, lo = dc.cpr_encode(lat + dl, min(lon + dl, 180), odd, bool(surface))
            now[0] += 0.01
            want = ref.decode(icao, la, lo, odd, surface, now[0])
            try:
                got = ours.decode(icao, la, lo, odd, surface)
            except CPRBoundaryStraddleError:
                got = "straddle"
            except CPRNoPositionError:
                got = "nopos"
            if want[0] != "ok":
                assert got == want[0], (i, odd, got, want)
            else:
                assert abs(got[0] - want[1]) <= TOL * 90 and abs(got[1] - want[2]) <= TOL * 180, (i, odd, got, want)
                rng, brg = do.range_bearing(loc, [want[1], want[2]])
                assert abs(got[2] - rng) <= 1e-9 * max(1.0, rng) and abs(got[3] - brg) <= 1e-9 * 360
                ok += 1
    ours.close()
    assert ok >= 290


def test_device_resident_decode_equals_the_host_path(dec_mod):
    """amb_decode_frames_device: frames and records stay in device memory; byte-identical to the host-array path."""
    import torch
    import decode_cases
    loc, msgs = decode_cases.make_case(907, location=(48.1, 11.5), seconds=60.0, surface_share=0.3, n_random=900, n_aircraft=40)
    arr, n = dec_mod.frames_from_messages(msgs)
    d1, d2 = dec_mod.batch_decoder(loc), dec_mod.batch_decoder(loc)
    want = d1.decode(arr, n)
    raw = np.frombuffer(bytes(arr), dtype=np.uint8)[: n * 80].copy()
    out = d2.decode_device(torch.from_numpy(raw).cuda())
    got = out.cpu().numpy().view(dec_mod.FIELDS_DTYPE)
    assert got.size == n and got.tobytes() == want.tobytes()
    d1.close(); d2.close()


def test_iq_to_positions_without_leaving_the_device(dec_mod):
    """The whole chain on the GPU: IQ (device) -> rx_path -> drain_device (frames ordered and stamped on the device) ->
    batch_decoder.decode_device -> records on the device. Byte-identical to the host-driven chain (drain() ->
    decode())."""
    import torch
    import gr_air_modes_b200 as am
    rate, n = 4e6, 1 << 22
    iq, sent = _position_scene(rate, n, 33)
    loc = [50.0, 8.5]
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    rx.set_start_time(1_600_000_000, 0.125)
    rx.process(iq, flush=True)
    frames = list(rx.frames)
    rx.close()
    assert len(frames) >= sent
    d1 = dec_mod.batch_decoder(loc)
    want = d1.decode(frames)
    d1.close()
    assert int(((want["status"] & dec_mod.FS_HAS_POS) != 0).sum()) >= sent // 2

    q2 = am.msg_queue()
    rx2 = am.rx_path(rate, 7.0, q2, use_pmf=True)
    rx2.set_start_time(1_600_000_000, 0.125)
    dev = torch.from_numpy(iq).cuda()
    cuts = [0, 1_000_000, 1_000_000 + 777_776, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        rx2.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx2.drain_device()
    assert fr.numel() == 80 * len(frames) and fr.cpu().numpy().tobytes() == b"".join(bytes(f) for f in frames)
    d2 = dec_mod.batch_decoder(loc)
    out = d2.decode_device(fr)
    assert out.is_cuda and out.cpu().numpy().tobytes() == want.tobytes()
    assert q2.strings() == []                       # nothing was formatted on the host for these frames
    d2.close(); rx2.close()
