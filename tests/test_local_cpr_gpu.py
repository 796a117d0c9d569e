"""Decoder option "local_cpr" on the GPU (amb_decode_local.cuh after the seven kernels of the decode): record for record
against the brute-force checker tests/local_cpr_oracle.py on the decode_cases scenes and weak-signal trajectories,
batching invariance, option off = the reference's decoder byte for byte with seven launches per decode, reset, the
"only records without a global fix change" invariant, a 60 k-message stress of 300 aircraft, and IQ -> rx_path ->
drain_device -> decode_device with the option on. Tolerances: integers, flags and the outcome byte exact; lat/lon bit
for bit (IEEE +,-,*,/, floor, fmod with -fmad=false, pinned to cpr_resolve_local by the golden); velocity/heading and
range/bearing 1e-12 relative (CUDA's and glibc's libm differ in the last place). Need an H100."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_cases as dc  # noqa: E402
import local_cpr_cases as lc  # noqa: E402
import local_cpr_oracle as lo  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture()
def decode():
    from gr_air_modes_b200 import decode
    return decode


def _scenes():
    for kw, S in zip(dc.CASES, (10, 60, 600, 60)):
        loc, msgs = dc.make_case(**kw)
        yield "case%d" % kw["seed"], loc, msgs, S
    for seed, drop, loc in ((3, 0.9, None), (4, 0.8, (48.0, 11.0)), (5, 0.95, (48.5, 10.0))):
        msgs, _ = lc.trajectory_scene(seed, n_aircraft=60, seconds=120.0, drop=drop, location=(48.0, 11.0), surface_share=0.2)
        yield "traj%d" % seed, (list(loc) if loc else None), msgs, 30


def test_records_equal_the_checker(decode):
    total = {}
    for name, loc, msgs, S in _scenes():
        d = decode.batch_decoder(loc, local_cpr=S)
        got = d.decode_messages(msgs)
        assert d.stats()[0] == 13                       # seven + keys, four partition kernels, walk
        d.close()
        want = lo.decode_local(msgs, loc, S)
        lc.assert_records_match(got, want, name)
        for r in want:
            total[r["local"]] = total.get(r["local"], 0) + 1
    print("local outcomes over the scenes:", total)
    assert total[lo.LOCAL_DECODED] >= 500 and total[lo.LOCAL_NO_REF] >= 100
    assert total.get(lo.LOCAL_STALE, 0) >= 1 and total.get(lo.LOCAL_REJECTED, 0) >= 1


def test_batching_does_not_change_results(decode):
    msgs, _ = lc.trajectory_scene(6, n_aircraft=50, seconds=90.0, drop=0.85, surface_share=0.3)
    loc = [48.0, 11.0]
    d = decode.batch_decoder(loc, local_cpr=20)
    one = d.decode_messages(msgs)
    assert (decode.local_outcome(one) == decode.LOCAL_DECODED).sum() >= 100
    rng = np.random.default_rng(2)
    for plan in ("ones", "steps", "random"):
        d.reset()
        parts, pos = [], 0
        while pos < len(msgs):
            c = 1 if plan == "ones" and pos < 300 else (int(rng.choice([31, 32, 33])) if plan == "steps" else int(rng.integers(1, 500)))
            parts.append(d.decode_messages(msgs[pos:pos + c]))
            pos += c
        assert np.concatenate(parts).tobytes() == one.tobytes(), plan
    d.close()


def test_off_is_the_plain_decoder(decode):
    loc, msgs = dc.make_case(14, location=(51.5, -0.1), seconds=70.0, n_aircraft=10, n_random=400)
    fresh = decode.batch_decoder(loc)
    want = fresh.decode_messages(msgs)
    assert fresh.stats()[0] == 7
    fresh.close()
    d = decode.batch_decoder(loc, local_cpr=0)
    assert d.get_local_cpr() == 0 and d.decode_messages(msgs).tobytes() == want.tobytes() and d.stats()[0] == 7
    d.close()
    d = decode.batch_decoder(loc)
    d.set_local_cpr(60)
    d.set_local_cpr(0)
    got = d.decode_messages(msgs)
    assert got.tobytes() == want.tobytes() and d.stats()[0] == 7 and not np.any(got["pad_"])
    for bad in (-1, 601):
        with pytest.raises(ValueError):
            d.set_local_cpr(bad)
    for name, v in ((b"local_cpr", 601), (b"local_cpr", -1), (b"no_such_option", 1)):
        assert d._lib.amb_decoder_set_option(d._h, name, v) == -1
    d.close()


def test_only_records_without_a_global_fix_change(decode):
    for name, loc, msgs, S in _scenes():
        off = decode.batch_decoder(loc)
        a = off.decode_messages(msgs)
        off.close()
        on = decode.batch_decoder(loc, local_cpr=S)
        b = on.decode_messages(msgs)
        on.close()
        had = (a["status"] & decode.FS_HAS_POS) != 0
        assert a[had].tobytes() == b[had].tobytes(), name
        changed = np.array([x.tobytes() != y.tobytes() for x, y in zip(a, b)])
        gained = (~had) & ((b["status"] & decode.FS_HAS_POS) != 0)
        assert np.all(b["status"][changed] & ~a["status"][changed] & ~np.uint8(decode.FS_HAS_POS | decode.FS_HAS_RANGE) == 0)
        for f in decode.FIELDS_DTYPE.names:
            if f not in ("lat", "lon", "range", "bearing", "status", "pad_"):
                assert a[f].tobytes() == b[f].tobytes(), (name, f)
        assert np.all(decode.local_outcome(b)[gained] == decode.LOCAL_DECODED)
        assert np.all(decode.local_outcome(b)[had] == 0)


def test_reset_clears_the_reference_positions(decode):
    msgs = lc.chain_scene(n_local=60)
    d = decode.batch_decoder(None, local_cpr=5)
    first = d.decode_messages(msgs[:2])                       # the airborne pair: a global fix
    assert first["status"][1] & decode.FS_HAS_POS
    rest = d.decode_messages(msgs[2:])
    assert decode.local_outcome(rest)[0] == decode.LOCAL_DECODED
    d.reset()
    again = d.decode_messages(msgs[2:])
    assert d.get_local_cpr() == 5
    out = lo.decode_local(msgs[2:], None, 5)
    lc.assert_records_match(again, out, "after reset")
    assert all(r["local"] == lo.LOCAL_NO_REF for r in out if r["icao"] == 0x1234)
    # a decode with the option off does not write the table: the reference is still the one from before
    d.reset()
    d.decode_messages(msgs[:2])
    d.set_local_cpr(0)
    d.decode_messages(msgs[2:10])
    d.set_local_cpr(5)
    nxt = d.decode_messages(msgs[10:11])
    want = lo.apply_local(lo.do.decode_batch(msgs[:2] + msgs[10:11], None), [float(s) + float(f) for _, _, s, f in msgs[:2] + msgs[10:11]], None, 5)
    lc.assert_records_match(nxt, want[2:], "table untouched while off")
    d.close()


def test_stress_60k_messages_of_300_aircraft(decode):
    rng = np.random.default_rng(17)
    fleet = [(int(a), float(rng.uniform(-70, 70)), float(rng.uniform(-180, 180)), bool(rng.random() < 0.2))
             for a in rng.choice(1 << 24, 300, replace=False)]
    msgs, t = [], 0.0
    for k in range(60000):
        aa, lat, lon, surface = fleet[int(rng.integers(0, len(fleet)))]
        odd = int(rng.integers(0, 2))
        la, lo_ = dc.cpr_encode(lat + 1e-3 * rng.standard_normal(), lon + 1e-3 * rng.standard_normal(), odd, surface)
        me = dc.me_surface(6, 10, 1, 5, odd, la, lo_) if surface else dc.me_airborne(12, dc.enc_alt12(12000), odd, la, lo_)
        fr, ecc = dc.df17(aa, me)
        t += float(rng.choice([0.0, 2e-4, 2e-3, 0.3]))
        msgs.append((fr.hex(), ecc, int(t), t - int(t)))
    loc = [10.0, 20.0]
    off = lo.do.decode_batch(msgs, loc)                       # the O(n^2) scan is too slow here: its linear form
    want = _linear_local(off, msgs, loc, 15)
    d = decode.batch_decoder(loc, local_cpr=15)
    arr, n = decode.frames_from_messages(msgs)
    got = d.decode(arr, n)
    print("decode of %d frames with local_cpr: %.3f ms on the device" % (n, d.stats()[1]))
    d.close()
    lc.assert_records_match(got, want, "stress")
    assert sum(r["local"] == lo.LOCAL_DECODED for r in want) >= 1000


def _linear_local(recs, msgs, loc, S):
    """The checker's semantics with a dict of the latest position per ICAO instead of the backwards scan (the same
    answer: the latest earlier message of the aircraft with a position), for sizes where O(n^2) is too slow. Its
    equality with lo.apply_local is checked on the small scenes below."""
    out, last = [], {}
    times = [float(s) + float(f) for _, _, s, f in msgs]
    for k, r0 in enumerate(recs):
        one = lo.apply_local([dict(last[r0["icao"]][0]), r0], [last[r0["icao"]][1], times[k]], loc, S)[1] \
            if lo.is_position(r0) and r0["icao"] in last else lo.apply_local([r0], [times[k]], loc, S)[0]
        out.append(one)
        if lo.is_position(one) and one["status"] & lo.do.FS_HAS_POS:
            last[one["icao"]] = (one, times[k])
    return out


def test_linear_form_equals_the_checker():
    loc, msgs = dc.make_case(**dc.CASES[3])
    recs = lo.do.decode_batch(msgs, loc)
    assert _linear_local(recs, msgs, loc, 60) == lo.decode_local(msgs, loc, 60)


def test_iq_to_local_positions_without_leaving_the_device(decode):
    """IQ (device) -> rx_path -> drain_device -> decode_device with local_cpr: one aircraft's airborne even/odd pair,
    then its surface reports (no receiver location: the global decode never resolves them), beside a second aircraft.
    Records equal the checker's on the messages the slicer queued, and the host path's."""
    import torch
    import gr_air_modes_b200 as am
    from gr_air_modes_b200 import synth
    rate, n = 4e6, 1 << 22
    rng = np.random.default_rng(23)
    iq = (rng.standard_normal((n, 2)) * 0.005).astype(np.float32)
    c = iq.view(np.complex64).reshape(n)
    start, sent = 3000.0, 0
    while start < n - 2000:
        odd = sent % 2
        if sent % 3 == 2:
            la, lo_ = dc.cpr_encode(49.9, 8.2 + 1e-4 * sent, odd, False)
            frame, _ = dc.df17(0xA1B2C3, dc.me_airborne(11, dc.enc_alt12(20000), odd, la, lo_))
        elif sent < 2:
            la, lo_ = dc.cpr_encode(50.03, 8.57, odd, False)
            frame, _ = dc.df17(0x3C6444, dc.me_airborne(11, dc.enc_alt12(1000), odd, la, lo_))
        else:
            la, lo_ = dc.cpr_encode(50.03 + 1e-5 * sent, 8.57 + 1e-5 * sent, odd, True)
            frame, _ = dc.df17(0x3C6444, dc.me_surface(7, 10, 1, 33, odd, la, lo_))
        n0, w = synth.burst_waveform(synth.Burst(start, frame, 0.3, float(rng.uniform(0, 6.28))), rate / 2e6)
        c[n0:n0 + w.size] += w
        start += 20000 + float(rng.uniform(0, 3000))
        sent += 1
    iq = iq.reshape(-1)
    q = am.msg_queue()
    rx = am.rx_path(rate, 7.0, q, use_pmf=True)
    rx.process(iq, flush=True)
    frames, msgs = list(rx.frames), q.strings()
    rx.close()
    d1 = decode.batch_decoder(None, local_cpr=10)
    want_host = d1.decode(frames)
    d1.close()
    rx2 = am.rx_path(rate, 7.0, am.msg_queue(), use_pmf=True)
    dev = torch.from_numpy(iq).cuda()
    for a, b in ((0, 1_000_000), (1_000_000, 2_500_001), (2_500_001, n)):
        rx2.process(dev[2 * a: 2 * b], flush=(b == n), collect=False)
    fr = rx2.drain_device()
    rx2.close()
    assert fr.cpu().numpy().tobytes() == b"".join(bytes(f) for f in frames)
    d2 = decode.batch_decoder(None, local_cpr=10)
    out = d2.decode_device(fr).cpu().numpy().view(decode.FIELDS_DTYPE)
    d2.close()
    assert out.tobytes() == want_host.tobytes()
    queued = out[np.array([bool(f.passed) for f in frames])]
    want = lo.decode_local([(m.split()[0], int(m.split()[1], 16), int(m.split()[3]), float(m.split()[4])) for m in msgs], None, 10)
    lc.assert_records_match(queued, want, "iq")
    assert sum(r["local"] == lo.LOCAL_DECODED for r in want) >= sent // 2
