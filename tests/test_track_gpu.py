"""Decoder option "track" on the GPU (amb_decode_track.cuh after the decode and the local CPR stage): snapshots against
the sequential checker tests/track_oracle.py fed with the decoder's own records, on every scene of tests/track_cases.py
with local_cpr on and off and with and without a receiver location; after every batch of a random split; option off =
the plain decoder byte for byte with 7 launches (13 with local_cpr); records unchanged by the option; reset; host and
device snapshots byte-identical; 2000 aircraft over 600 s; IQ -> rx_path -> drain_device -> decode_device ->
aircraft_device. Rows are copies of record and frame values, so the comparison is bit for bit (any NaN equals any NaN).
Need an H100."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_cases as dc  # noqa: E402
import track_cases as tc  # noqa: E402
import track_oracle as to  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _device_rows(decode, d, now=None):
    dev = d.aircraft_device(now)
    return dev.cpu().numpy().view(decode.AIRCRAFT_DTYPE)


def test_snapshots_equal_the_checker(decode):
    shown = {}
    for name, loc, msgs, S in tc.scenes():
        frames = tc.frames_of(msgs)
        ts = to.t_of(frames)
        for where in (loc, None) if loc is not None else (None,):
            for local in (0, 30):
                plain = decode.batch_decoder(where, local_cpr=local)
                want_recs = plain.decode(frames)
                plain.close()
                d = decode.batch_decoder(where, local_cpr=local, track=S)
                recs = d.decode(frames)
                assert d.stats()[0] == (19 if local else 13)
                assert recs.tobytes() == want_recs.tobytes(), name       # the option leaves the records alone
                tr = to.Tracker(S)
                tr.feed(frames, recs)
                tag = (name, where is not None, local)
                for now in (None, ts[len(ts) // 3], ts[-1] + S / 2, ts[-1] + S + 1):
                    host = d.aircraft(now)
                    to.assert_rows_equal(host, tr.snapshot_array(now), tag + (now,))
                    assert _device_rows(decode, d, now).tobytes() == host.tobytes(), tag
                shown[tag] = len(d.aircraft())
                d.close()
    print("rows shown at the end of each scene:", shown)
    assert sum(shown.values()) >= 100


def test_snapshot_after_every_batch_of_a_random_split(decode):
    msgs = tc.life_scene(seed=3) + []
    frames = tc.frames_of(msgs, seed=3)
    loc = [51.5, -0.2]
    rng = np.random.default_rng(8)
    for plan in ("ones", "steps", "random"):
        d = decode.batch_decoder(loc, local_cpr=10, track=20)
        tr = to.Tracker(20)
        pos, last = 0, None
        while pos < len(frames):
            c = 1 if plan == "ones" and pos < 200 else (int(rng.choice([31, 32, 33])) if plan == "steps" else int(rng.integers(1, 300)))
            part = frames[pos:pos + c]
            tr.feed(part, d.decode(part))
            last = d.aircraft()
            to.assert_rows_equal(last, tr.snapshot_array(), (plan, pos))
            pos += c
        if plan == "ones":
            first = last
        else:
            to.assert_rows_equal(last, first, plan)                     # the split does not matter
        d.close()


def test_off_is_the_plain_decoder(decode):
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    frames = tc.frames_of(msgs)
    fresh = decode.batch_decoder(loc)
    want = fresh.decode(frames)
    assert fresh.stats()[0] == 7
    fresh.close()
    d = decode.batch_decoder(loc, track=0)
    assert d.get_track() == 0 and d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 7
    with pytest.raises(RuntimeError):
        d.aircraft()
    d.close()
    d = decode.batch_decoder(loc)
    d.set_track(60)
    d.set_track(0)
    assert d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 7
    d.set_local_cpr(30)
    k = d.stats()[0]
    d.decode(frames)
    assert d.stats()[0] - k == 13
    for bad in (-1, 3601):
        with pytest.raises(ValueError):
            d.set_track(bad)
    for name, v in ((b"track", 3601), (b"track", -1)):
        assert d._lib.amb_decoder_set_option(d._h, name, v) == -1
    d.close()


def test_reset_empties_the_table(decode):
    msgs = tc.burst_scene()
    frames = tc.frames_of(msgs, unqueued_every=0)
    d = decode.batch_decoder(None, track=3)
    d.decode(frames)
    assert len(d.aircraft()) >= 1
    d.reset()
    assert len(d.aircraft()) == 0 and len(d.aircraft(to.t_of(frames)[-1])) == 0 and d.get_track() == 3
    assert d.aircraft_device().numel() == 0
    tr = to.Tracker(3)
    tr.feed(frames[:50], d.decode(frames[:50]))                        # the table starts over
    to.assert_rows_equal(d.aircraft(), tr.snapshot_array(), "after reset")
    # a decode with the option off leaves the table as it was
    d.set_track(0)
    d.decode(frames[50:])
    d.set_track(3)
    to.assert_rows_equal(d.aircraft(), tr.snapshot_array(), "untouched while off")
    d.close()


def test_host_and_device_snapshots_are_byte_identical(decode):
    import torch
    name, loc, msgs, S = next(s for s in tc.scenes() if s[0] == "bucket")
    frames = tc.frames_of(msgs)
    d = decode.batch_decoder(loc, track=S)
    d.decode(frames)
    host = d.aircraft()
    assert len(host) == 32
    big = torch.full((64 * 128,), 0x5A, dtype=torch.uint8, device="cuda")
    got = d.aircraft_device(out_dev=big)
    assert got.numel() == 32 * 128 and got.cpu().numpy().tobytes() == host.tobytes()
    assert torch.all(big[32 * 128:] == 0x5A)                            # nothing written past the rows
    small = torch.full((31 * 128,), 0x5A, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):
        d.aircraft_device(out_dev=small)                                # AMB_ERR_OVERFLOW, nothing written
    assert torch.all(small == 0x5A)
    d.close()


def test_stress_2000_aircraft_over_600_s(decode):
    msgs = tc.fleet_scene(n_aircraft=2000, seconds=600.0)
    frames = tc.frames_of(msgs)
    ts = to.t_of(frames)
    d = decode.batch_decoder([10.0, 20.0], track=60)
    tr = to.Tracker(60)
    pos = 0
    for c in (1, 4095, 60000, 1 << 17, len(frames)):
        part = frames[pos:pos + c]
        if len(part) == 0:
            break
        tr.feed(part, d.decode(part))
        print("decode of %d frames with track: %.3f ms on the device" % (len(part), d.stats()[1]))
        pos += len(part)
    for now in (None, 300.0, ts[-1] - 59.5):
        got = d.aircraft(now)
        to.assert_rows_equal(got, tr.snapshot_array(now), now)
        assert len(got) >= 100, now
    d.close()


def test_iq_to_aircraft_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device -> aircraft_device, with local_cpr and track on: the rows
    equal the checker's on the drained frames and the host path's snapshot."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 22
    rng = np.random.default_rng(29)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    while start < n - 2000:
        aa = (0xA1B2C3, 0x3C6444, 0x4840D6)[sent % 3]
        odd = (sent // 3) % 2
        kind = (sent // 3) % 4
        if kind < 2:
            la, lo_ = dc.cpr_encode(49.9 + 0.1 * (sent % 3), 8.2 + 1e-4 * sent, odd, False)
            frame, _ = dc.df17(aa, dc.me_airborne(11, dc.enc_alt12(20000), odd, la, lo_))
        elif kind == 2:
            frame, _ = dc.df17(aa, dc.me_ident(4, 3, "IQ%06X" % aa))
        else:
            frame, _ = dc.df17(aa, dc.Bits(56).put(1, 5, 19).put(6, 3, 1).put(15, 10, 300).put(26, 10, 200).put(38, 9, 10).v)
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
    d = decode.batch_decoder([50.0, 8.5], local_cpr=10, track=30)
    recs_dev = d.decode_device(fr)
    rows = d.aircraft_device()
    assert rows.is_cuda and rows.numel() == 3 * 128
    got = rows.cpu().numpy().view(decode.AIRCRAFT_DTYPE)
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the checker only
    recs = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    to.assert_rows_equal(got, to.replay(frames, recs, 30), "iq")
    h = decode.batch_decoder([50.0, 8.5], local_cpr=10, track=30)
    h.decode(frames)
    assert h.aircraft().tobytes() == got.tobytes()
    h.close()
    assert sorted(got["icao"].tolist()) == [0x3C6444, 0x4840D6, 0xA1B2C3]
    assert np.all(got["flags"] & decode.AC_HAS_POS) and np.all(got["flags"] & decode.AC_HAS_IDENT)
    assert not math.isnan(float(got["speed"][0]))
