"""Decoder option "opstatus" on the GPU (amb_decode_opstatus.cuh after the Comm-B stage, before the track stage): records
byte for byte equal to the sequential checker tests/opstatus_oracle.py fed with the decoder's own option-off records, on
every scene of tests/opstatus_cases.py with local_cpr, commb and track on and off; random batch splits; off = a fresh
decoder byte for byte with the same launch count, on = six launches more; only eligible records change, and only in aux
and pad_ bytes 5..7; the track snapshot and the Comm-B bytes are the same with the option on and off; reset forgets the
op status; about 10^5 messages from 300 aircraft; IQ -> rx_path -> drain_device -> decode_device. Need an H100."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import commb_cases as cc  # noqa: E402
import decode_cases as dc  # noqa: E402
import opstatus_cases as oc  # noqa: E402
import opstatus_oracle as oo  # noqa: E402
import track_cases as tc  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _changed_only_where_allowed(frames, off, on):
    """Records differ only when eligible, and only in aux and pad_ bytes 5..7; every other DF17 record has aux = 0 and
    every record pad_ bytes 5..7 = 0 with the option off."""
    b_off = off.view(np.uint8).reshape(len(off), 144)
    b_on = on.view(np.uint8).reshape(len(on), 144)
    allowed = np.zeros(144, dtype=bool)
    aux = off.dtype.fields["aux"][1]
    pad = off.dtype.fields["pad_"][1]
    allowed[aux:aux + 16] = True
    allowed[pad + 5:pad + 8] = True
    assert not np.any(b_off[:, pad + 5:pad + 8])
    assert not np.any(off["aux"][off["df"] == 17])
    diff = b_off != b_on
    assert not np.any(diff[:, ~allowed])
    elig = np.array([oo.eligible(frames[k], off[k]) for k in range(len(off))], dtype=bool)
    assert not np.any(diff[~elig])
    assert np.all(oo.outcome_of(on)[~elig] == oo.NOT_TRIED)


def _commb_scene():
    """Comm-B replies and velocities mixed into an op-status scene, for the "Comm-B bytes unchanged" check."""
    ops = oc.table_scene()
    com = cc.reference_scene(S=30)
    return sorted(ops + com, key=lambda m: m[2] + m[3])


def test_scenes_equal_the_checker(decode):
    counts = {}
    scenes = list(oc.scenes()) + [("with_commb", _commb_scene(), 30)]
    for name, msgs, S in scenes:
        frames = tc.frames_of(msgs)
        for local in (0, 10):
            for commb in (0, 30):
                for track in (0, 60):
                    plain = decode.batch_decoder(None, local_cpr=local, commb=commb, track=track)
                    off = plain.decode(frames)
                    k_off = plain.stats()[0]
                    snap_off = plain.aircraft() if track else None
                    plain.close()
                    d = decode.batch_decoder(None, local_cpr=local, commb=commb, track=track, opstatus=S)
                    assert d.get_opstatus() == S
                    on = d.decode(frames)
                    assert d.stats()[0] == k_off + 6
                    oo.assert_records_equal(on, oo.replay(frames, off, S), (name, local, commb, track))
                    _changed_only_where_allowed(frames, off, on)
                    if commb:                                   # the Comm-B bytes: pad_ 1..4 and the DF20/21 aux
                        assert np.array_equal(decode.commb_outcome(on), decode.commb_outcome(off))
                        df2021 = np.isin(off["df"], (20, 21))
                        assert on[df2021].tobytes() == off[df2021].tobytes()
                    if track:
                        assert d.aircraft().tobytes() == snap_off.tobytes(), name
                    d.close()
        o = oo.outcome_of(on)
        counts[name] = {v: int(np.sum(o == v)) for v in range(6)}
    print("outcomes per scene:", counts)
    assert counts["table"][oo.NIC] >= 100 and counts["fields"][oo.TARGET_STATE] >= 20


def test_random_batch_splits(decode):
    msgs = oc.bucket_scene()
    frames = tc.frames_of(msgs)
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    want = oo.replay(frames, off, 5)
    rng = np.random.default_rng(8)
    for plan in ("ones", "steps", "random"):
        d = decode.batch_decoder(None, opstatus=5)
        got, pos = [], 0
        while pos < len(frames):
            c = 1 if plan == "ones" and pos < 200 else (int(rng.choice([31, 32, 33])) if plan == "steps" else int(rng.integers(1, 300)))
            got.append(d.decode(frames[pos:pos + c]))
            pos += c
        oo.assert_records_equal(np.concatenate(got), want, plan)
        d.close()


def test_off_is_a_fresh_decoder(decode):
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    msgs = sorted(msgs + oc.table_scene(), key=lambda m: m[2] + m[3])
    frames = tc.frames_of(msgs)
    fresh = decode.batch_decoder(loc)
    want = fresh.decode(frames)
    assert fresh.stats()[0] == 7
    fresh.close()
    d = decode.batch_decoder(loc, opstatus=0)
    assert d.get_opstatus() == 0 and d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 7
    d.set_opstatus(30)
    d.set_opstatus(0)
    assert d.decode(frames).tobytes() == want.tobytes() and d.stats()[0] == 14
    d.set_opstatus(600)
    k = d.stats()[0]
    d.decode(frames)
    assert d.stats()[0] - k == 13
    for bad in (-1, 601):
        with pytest.raises(ValueError):
            d.set_opstatus(bad)
        assert d._lib.amb_decoder_set_option(d._h, b"opstatus", bad) == -1
    d.close()
    for local, commb, track in ((10, 0, 0), (0, 30, 0), (0, 0, 60), (10, 30, 60)):   # every stage on, off the option
        a = decode.batch_decoder(loc, local_cpr=local, commb=commb, track=track)
        b = decode.batch_decoder(loc, local_cpr=local, commb=commb, track=track, opstatus=0)
        assert a.decode(frames).tobytes() == b.decode(frames).tobytes() and a.stats()[0] == b.stats()[0]
        a.close()
        b.close()


def test_reset_forgets_the_op_status(decode):
    msgs = oc.table_scene()
    frames = tc.frames_of(msgs, unqueued_every=0)
    n = len(frames) // 2
    plain = decode.batch_decoder(None)                  # option-off records of the second half after a reset too
    plain.decode(frames[:n])
    plain.reset()
    off = np.concatenate([np.zeros(n, dtype=decode.FIELDS_DTYPE), plain.decode(frames[n:])])
    plain.close()
    d = decode.batch_decoder(None, opstatus=30)
    d.decode(frames[:n])
    d.reset()
    got = d.decode(frames[n:])
    oo.assert_records_equal(got, oo.replay(frames[n:], off[n:], 30), "after reset")
    d.close()


def test_stress_1e5_messages_from_300_aircraft(decode):
    msgs, truth = oc.fleet_scene(n_aircraft=300, seconds=70.0)
    assert len(msgs) >= 90000
    frames = tc.frames_of(msgs)
    plain = decode.batch_decoder([10.0, 20.0])
    off = plain.decode(frames)
    plain.close()
    chk = oo.Checker(30)
    d = decode.batch_decoder([10.0, 20.0], opstatus=30)
    pos = 0
    got = []
    for c in (1, 4095, 30000, len(frames)):
        part = slice(pos, pos + c)
        if pos >= len(frames):
            break
        got.append(d.decode(frames[part]))
        oo.assert_records_equal(got[-1], chk.feed(frames[part], off[part]), ("batch at", pos))
        print("decode of %d frames with opstatus: %.3f ms on the device" % (len(got[-1]), d.stats()[1]))
        pos += c
    d.close()
    o = oo.outcome_of(np.concatenate(got))
    assert np.sum(o == oo.NIC) > 10000 and np.sum(o == oo.NUC) > 1000 and np.sum(o == oo.TARGET_STATE) > 1000


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
        kind = (sent // 3) % 3
        if kind == 0:
            frame, _ = dc.df17(aa, oc.opstatus_me(sent % 2, 2, nica=1, nicc=1, nacp=10))
        elif kind == 1:
            frame, _ = dc.df17(aa, oc.target_state_me(alt=1001, baro=267, hdg_status=1, hdg=100, modes=0xC6))
        else:
            frame, _ = oc.position(aa, int(rng.choice([7, 8, 11, 13, 16])), int(rng.integers(0, 2)), rng)
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
    d = decode.batch_decoder(None, opstatus=30)
    recs_dev = d.decode_device(fr)
    assert recs_dev.is_cuda
    got = recs_dev.cpu().numpy().view(decode.FIELDS_DTYPE)
    d.close()
    frames = fr.cpu().numpy().view(decode.FRAME_DTYPE)                  # for the checker only
    plain = decode.batch_decoder(None)
    off = plain.decode(frames)
    plain.close()
    oo.assert_records_equal(got, oo.replay(frames, off, 30), "iq")
    h = decode.batch_decoder(None, opstatus=30)
    assert h.decode(frames).tobytes() == got.tobytes()
    h.close()
    o = oo.outcome_of(got)
    assert np.sum(o == oo.NIC) >= 5 and np.sum(o == oo.OPSTATUS) >= 5 and np.sum(o == oo.TARGET_STATE) >= 5
