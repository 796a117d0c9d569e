"""Decoder option "track_ext" on the GPU (amb_decode_track_ext.cuh after the track stage, amb_decoder_aircraft_ext):
snapshots byte for byte equal to the sequential checker tests/track_ext_oracle.py fed with the decoder's own records,
on every scene of tests/track_ext_cases.py with local_cpr, commb and opstatus on and off; random batch splits; off = a
fresh decoder (records, base snapshot, launch count); on = six launches more per decode, records and base snapshot
unchanged, three launches per snapshot; host and device snapshots byte for byte; t[INTEG] == pos_t with opstatus on
from the start; reset; about 10^5 messages from 300 aircraft; IQ -> rx_path -> drain_device -> decode_device ->
aircraft_ext_device. Need an H100."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_cases as dc  # noqa: E402
import opstatus_cases as oc  # noqa: E402
import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
import track_ext_oracle as xo  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _device_snapshot(decode, d, now):
    out, ext = d.aircraft_ext_device(now)
    return (out.cpu().numpy().view(decode.AIRCRAFT_DTYPE), ext.cpu().numpy().view(decode.AIRCRAFT_EXT_DTYPE))


def test_scenes_equal_the_checker(decode):
    shown = {}
    for name, msgs, S, S2 in xc.scenes():
        frames = tc.frames_of(msgs)
        ts = frames["secs"].astype(float) + frames["frac"]
        for local in (0, 10):
            for commb in (0, 30):
                for ops in (0, 30):
                    kw = dict(local_cpr=local, commb=commb, opstatus=ops, track=S)
                    plain = decode.batch_decoder(None, **kw)
                    want = plain.decode(frames)
                    k_off = plain.stats()[0]
                    base = plain.aircraft()
                    plain.close()
                    d = decode.batch_decoder(None, track_ext=S2, **kw)
                    got = d.decode(frames)
                    assert got.tobytes() == want.tobytes(), name
                    assert d.stats()[0] == k_off + 6
                    assert d.aircraft().tobytes() == base.tobytes(), name
                    chk = xo.ExtTracker(S, S2)
                    chk.feed(frames, got)
                    for now in (None, float(ts[len(ts) // 2]), float(ts[-1]) + S2 / 2):
                        k = d.stats()[0]
                        snap = d.aircraft_ext(now)
                        assert d.stats()[0] - k == (5 if len(snap[0]) else 2)
                        xo.assert_snapshots_equal(snap, chk.snapshot_arrays(now), (name, kw, now))
                        dev = _device_snapshot(decode, d, now)
                        assert dev[0].tobytes() == snap[0].tobytes() and dev[1].tobytes() == snap[1].tobytes()
                    if ops and commb and not local:
                        shown[name] = int(np.bitwise_or.reduce(d.aircraft_ext()[1]["shown"], initial=0))
                    d.close()
    print("groups shown per scene:", shown)
    assert np.bitwise_or.reduce(list(shown.values())) == 0x3F


def test_random_batch_splits(decode):
    frames = tc.frames_of(xc.merge(xc.bucket_scene(), xc.absence_scene()))
    one = decode.batch_decoder(None, opstatus=30, commb=30, track=30, track_ext=20)
    one.decode(frames)
    want = one.aircraft_ext()
    one.close()
    rng = np.random.default_rng(8)
    for plan in ("ones", "steps", "random"):
        d = decode.batch_decoder(None, opstatus=30, commb=30, track=30, track_ext=20)
        pos = 0
        while pos < len(frames):
            c = 1 if plan == "ones" and pos < 200 else (int(rng.choice([31, 32, 33])) if plan == "steps" else int(rng.integers(1, 300)))
            d.decode(frames[pos:pos + c])
            pos += c
        got = d.aircraft_ext()
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), plan
        d.close()


def test_off_is_a_fresh_decoder(decode):
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    msgs = xc.merge(msgs, oc.table_scene(), xc.bucket_scene())
    frames = tc.frames_of(msgs)
    for local in (0, 10):
        for commb in (0, 30):
            for ops in (0, 30):
                for track in (0, 60):
                    kw = dict(local_cpr=local, commb=commb, opstatus=ops, track=track)
                    a = decode.batch_decoder(loc, **kw)
                    b = decode.batch_decoder(loc, track_ext=0, **kw)
                    c = decode.batch_decoder(loc, track_ext=0 if track else 600, **kw)   # no track: no effect
                    ra = a.decode(frames)
                    assert ra.tobytes() == b.decode(frames).tobytes() == c.decode(frames).tobytes()
                    assert a.stats()[0] == b.stats()[0] == c.stats()[0]
                    if track:
                        assert a.aircraft().tobytes() == b.aircraft().tobytes()
                    for x in (a, b, c):
                        x.close()
    d = decode.batch_decoder(loc, track=60)
    d.set_track_ext(30)
    d.set_track_ext(0)
    d.decode(frames)
    assert d.stats()[0] == 13
    with pytest.raises(RuntimeError):
        d.aircraft_ext()
    d.set_track_ext(3600)
    d.decode(frames)
    assert d.stats()[0] == 13 + 19
    for bad in (-1, 3601):
        with pytest.raises(ValueError):
            d.set_track_ext(bad)
        assert d._lib.amb_decoder_set_option(d._h, b"track_ext", bad) == -1
    d.close()


def test_integrity_time_is_the_position_time(decode):
    frames = tc.frames_of(xc.merge(oc.table_scene(), xc.bucket_scene(), xc.absence_scene()))
    d = decode.batch_decoder([48.0, 11.0], opstatus=30, commb=30, track=3600, track_ext=3600)
    d.decode(frames)
    rows, ext = d.aircraft_ext()
    d.close()
    on = (ext["shown"] & decode.AXG_INTEG) != 0
    assert np.sum(on) >= 30
    assert np.array_equal(ext["t"][on, 2], rows["pos_t"][on])
    assert np.all(rows["flags"][on] & decode.AC_HAS_POS)


def test_reset_forgets_every_group(decode):
    rng = np.random.default_rng(11)
    a_ev, b_ev = [], []
    for j, aa in enumerate((0x4840D6, 0x3C6444)):
        e, _ = xc.life(aa, 1000.0 + j, rng, n=18)
        a_ev += e
        for k in range(6):
            b_ev.append((990.0 + j + 0.1 * k, *tc.position(aa, 47.0, 8.0, k % 2, False)))
    fa, fb = tc.frames_of(xc._msgs(a_ev), unqueued_every=0), tc.frames_of(xc._msgs(b_ev), unqueued_every=0)
    d = decode.batch_decoder(None, opstatus=30, commb=30, track=60, track_ext=600)
    d.decode(fa)
    assert np.all(d.aircraft_ext()[1]["shown"] == 0x3F)
    d.reset()
    assert len(d.aircraft_ext()[0]) == 0
    recs = d.decode(fb)
    chk = xo.ExtTracker(60, 600)
    chk.feed(fb, recs)
    for now in (None, 1003.0, 1010.0):
        got = d.aircraft_ext(now)
        xo.assert_snapshots_equal(got, chk.snapshot_arrays(now), ("after reset", now))
        assert len(got[0]) == 2 and np.all(got[1]["shown"] == decode.AXG_INTEG)
    d.close()


def test_stress_1e5_messages_from_300_aircraft(decode):
    msgs = xc.fleet(n_aircraft=300, seconds=40.0)
    assert len(msgs) >= 100000
    frames = tc.frames_of(msgs)
    chk = xo.ExtTracker(60, 30)
    d = decode.batch_decoder([10.0, 20.0], opstatus=30, commb=30, track=60, track_ext=30)
    pos = 0
    for c in (1, 4095, 30000, len(frames)):
        if pos >= len(frames):
            break
        part = slice(pos, pos + c)
        recs = d.decode(frames[part])
        print("decode of %d frames with track_ext: %.3f ms on the device" % (len(recs), d.stats()[1]))
        chk.feed(frames[part], recs)
        xo.assert_snapshots_equal(d.aircraft_ext(), chk.snapshot_arrays(), ("batch at", pos))
        pos += c
    rows, ext = d.aircraft_ext()
    d.close()
    assert len(rows) >= 250
    for g in range(6):
        assert np.sum(ext["shown"] & (1 << g)) >= 20, g


def test_iq_to_snapshot_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device -> aircraft_ext_device: the snapshot equals the host
    path's and the checker's on the drained frames."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 22
    rng = np.random.default_rng(29)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    addrs = (0xA1B2C3, 0x3C6444, 0x4840D6)
    while start < n - 2000:
        aa = addrs[sent % 3]
        kind = (sent // 3) % 4
        if kind == 0:
            frame, _ = dc.df17(aa, oc.opstatus_me(0, 2, nica=1, nacp=10))
        elif kind == 1:
            frame, _ = dc.df17(aa, oc.target_state_me(alt=1001, baro=267, hdg_status=1, hdg=100, modes=0xC6))
        else:
            frame, _ = tc.position(aa, 50.0 + 0.01 * (sent % 3), 8.0, (sent // 12) % 2, False)
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
    d = decode.batch_decoder(None, opstatus=30, track=60, track_ext=60)
    recs_dev = d.decode_device(fr)
    out_dev, ext_dev = d.aircraft_ext_device()
    assert recs_dev.is_cuda and out_dev.is_cuda and ext_dev.is_cuda
    got = (out_dev.cpu().numpy().view(decode.AIRCRAFT_DTYPE), ext_dev.cpu().numpy().view(decode.AIRCRAFT_EXT_DTYPE))
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the host path and the checker only
    h = decode.batch_decoder(None, opstatus=30, track=60, track_ext=60)
    recs = h.decode(frames)
    host = h.aircraft_ext()
    h.close()
    assert recs.tobytes() == recs_dev.cpu().numpy().tobytes()
    assert host[0].tobytes() == got[0].tobytes() and host[1].tobytes() == got[1].tobytes()
    chk = xo.ExtTracker(60, 60)
    chk.feed(frames, recs)
    xo.assert_snapshots_equal(got, chk.snapshot_arrays(), "iq")
    assert len(got[0]) == 3 and np.all(got[1]["shown"] == decode.AXG_OPS | decode.AXG_TS | decode.AXG_INTEG)
    assert not math.isnan(float(got[1]["t"][0][0]))
