"""Decoder option "commb" on the GPU (amb_decode_commb.cuh after the decode and the local CPR stage, before the track
stage): records byte for byte equal to the sequential checker tests/commb_oracle.py fed with the decoder's own
option-off records, on every scene of tests/commb_cases.py with local_cpr and track on and off; random batch splits;
off = a fresh decoder byte for byte with the same launch count, on = six launches more; only eligible records change,
and only in aux and pad_ bytes 1..4; the track snapshot is the same with the option on and off; reset forgets the
velocities; 60k messages from 300 aircraft; IQ -> rx_path -> drain_device -> decode_device. Need an H100."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import commb_cases as cc  # noqa: E402
import commb_oracle as co  # noqa: E402
import decode_cases as dc  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _changed_only_where_allowed(frames, off, on):
    """Records differ only when eligible, and only in aux and pad_ bytes 1..4."""
    b_off = off.view(np.uint8).reshape(len(off), 144)
    b_on = on.view(np.uint8).reshape(len(on), 144)
    allowed = np.zeros(144, dtype=bool)
    aux = off.dtype.fields["aux"][1]
    pad = off.dtype.fields["pad_"][1]
    allowed[aux:aux + 16] = True
    allowed[pad + 1:pad + 5] = True
    diff = b_off != b_on
    assert not np.any(diff[:, ~allowed])
    rows = np.flatnonzero(diff.any(axis=1))
    for k in rows:
        assert co.eligible(frames[k], off[k]), k
    assert np.all(co.outcome_of(on)[[k for k in range(len(on)) if not co.eligible(frames[k], off[k])]] == co.NOT_TRIED)


def test_scenes_equal_the_checker(decode):
    counts = {}
    for name, msgs, S in cc.scenes():
        frames = tc.frames_of(msgs)
        for local in (0, 10):
            for track in (0, 60):
                plain = decode.batch_decoder(None, local_cpr=local, track=track)
                off = plain.decode(frames)
                k_off = plain.stats()[0]
                snap_off = plain.aircraft() if track else None
                plain.close()
                d = decode.batch_decoder(None, local_cpr=local, track=track, commb=S)
                assert d.get_commb() == S
                on = d.decode(frames)
                assert d.stats()[0] == k_off + 6
                co.assert_records_equal(on, co.replay(frames, off, S), (name, local, track))
                _changed_only_where_allowed(frames, off, on)
                if track:
                    assert d.aircraft().tobytes() == snap_off.tobytes(), name
                d.close()
        o = co.outcome_of(on)
        counts[name] = {v: int(np.sum(o == v)) for v in range(5)}
    print("outcomes per scene:", counts)
    assert counts["reference"][co.RESOLVED] >= 10 and counts["unique"][co.DECODED] >= 50


def test_random_batch_splits(decode):
    msgs = cc.bucket_scene() + []
    frames = tc.frames_of(msgs)
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    want = co.replay(frames, off, 30)
    rng = np.random.default_rng(8)
    for plan in ("ones", "steps", "random"):
        d = decode.batch_decoder(None, commb=30)
        got, pos = [], 0
        while pos < len(frames):
            c = 1 if plan == "ones" and pos < 200 else (int(rng.choice([31, 32, 33])) if plan == "steps" else int(rng.integers(1, 300)))
            got.append(d.decode(frames[pos:pos + c]))
            pos += c
        co.assert_records_equal(np.concatenate(got), want, plan)
        d.close()


def test_off_is_a_fresh_decoder(decode):
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    frames = tc.frames_of(msgs)
    fresh = decode.batch_decoder(loc)
    want = fresh.decode(frames)
    assert fresh.stats()[0] == 7
    fresh.close()
    d = decode.batch_decoder(loc, commb=0)
    assert d.get_commb() == 0 and d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 7
    d.set_commb(30)
    d.set_commb(0)
    assert d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 14
    d.set_commb(600)
    k = d.stats()[0]
    d.decode(frames)
    assert d.stats()[0] - k == 13
    for bad in (-1, 601):
        with pytest.raises(ValueError):
            d.set_commb(bad)
        assert d._lib.amb_decoder_set_option(d._h, b"commb", bad) == -1
    d.close()


def test_reset_forgets_the_velocities(decode):
    msgs = cc.reference_scene(S=30)
    frames = tc.frames_of(msgs, unqueued_every=0)
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    n = len(frames) // 2
    d = decode.batch_decoder(None, commb=30)
    d.decode(frames[:n])
    d.reset()
    got = d.decode(frames[n:])
    co.assert_records_equal(got, co.replay(frames[n:], off[n:], 30), "after reset")
    d.close()


def test_stress_60k_messages_from_300_aircraft(decode):
    msgs, truth = cc.fleet_scene(n_aircraft=300, seconds=100.0)
    assert len(msgs) >= 60000
    frames = tc.frames_of(msgs)
    plain = decode.batch_decoder([10.0, 20.0])
    off = plain.decode(frames)
    plain.close()
    chk = co.Checker(30)
    d = decode.batch_decoder([10.0, 20.0], commb=30)
    pos = 0
    got = []
    for c in (1, 4095, 30000, len(frames)):
        part = slice(pos, pos + c)
        if pos >= len(frames):
            break
        got.append(d.decode(frames[part]))
        co.assert_records_equal(got[-1], chk.feed(frames[part], off[part]), ("batch at", pos))
        print("decode of %d frames with commb: %.3f ms on the device" % (len(got[-1]), d.stats()[1]))
        pos += c
    d.close()
    o = co.outcome_of(np.concatenate(got))
    assert np.sum(o == co.DECODED) > 1000 and np.sum(o == co.RESOLVED) > 100


def test_iq_to_records_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device with the option on: records equal the checker's on the
    drained frames and the host path's."""
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
        if (sent // 3) % 2 == 0:
            frame, _ = cc.velocity(aa, 400, south=bool(sent % 2))
        else:
            frame, _ = cc.reply(20, aa, cc.ambiguous_word(rng, gs=200, trk=int(rng.choice([0, -1024]))), rng)
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
    d = decode.batch_decoder(None, commb=30)
    recs_dev = d.decode_device(fr)
    assert recs_dev.is_cuda
    got = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the checker only
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    co.assert_records_equal(got, co.replay(frames, off, 30), "iq")
    h = decode.batch_decoder(None, commb=30)
    assert h.decode(frames).tobytes() == got.tobytes()
    h.close()
    o = co.outcome_of(got)
    assert np.sum(o == co.RESOLVED) >= 5
