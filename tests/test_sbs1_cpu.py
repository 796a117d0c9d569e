"""Decoder option "sbs1" without a GPU: the line formatting (gr_air_modes_b200/csrc/amb_sbs1_format.h, compiled for
the host by tests/sbs1_host_shim.cc) against Python's % and datetime over whole input domains; option validation in
Python and through the C ABI of the emulated library (tests/simt/library_emul.cc: the library's own sources on the
SIMT emulator), and a stream through that C ABI against the checker; sbs1_server on loopback; the CLI's -P rules."""
import ctypes as C
import datetime
import math
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import emul_build  # noqa: E402
import sbs1_cases as sc  # noqa: E402
import sbs1_oracle as so  # noqa: E402
import track_cases as tc  # noqa: E402

ERR_INVALID, ERR_OVERFLOW, ERR_STATE = -1, -5, -8


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "sbs1_host_shim.cc")))
    lib.shim_fixed.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_void_p]
    lib.shim_trunc.argtypes = [C.c_void_p, C.c_long, C.c_void_p]
    lib.shim_stamp.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p]
    lib.shim_line.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_double, C.c_int, C.c_char_p]
    return lib


def _strings(buf):
    return [bytes(b).split(b"\0", 1)[0].decode() for b in buf]


def _fixed(shim, x, prec):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.zeros((len(x), 32), dtype=np.uint8)
    shim.shim_fixed(C.c_void_p(x.ctypes.data), len(x), prec, C.c_void_p(out.ctypes.data))
    return _strings(out)


def _check_fixed(shim, x, prec):
    got = _fixed(shim, x, prec)
    fmt = "%%.%df" % prec
    bad = [(v, g) for v, g in zip(x.tolist(), got) if g != fmt % v]
    assert not bad, bad[:5]


def _bds09_values():
    """Velocity and heading of every BDS0,9 subtype 0 and 1 (both sub-2 scalings) word as parse.py computes them."""
    out_v, out_h = [], []
    for vew in range(1024):
        for dew in (0, 1):
            vns = np.arange(1024)
            for dns in (0, 1):
                # subtype 0 (parseBDS09_0): velocity from the -1 words, heading atan2 of the signed ones
                ns, ew = vns - 1.0, float(vew - 1)
                out_v.append(np.hypot(ns, ew))
                h = np.degrees(np.arctan2(-ew if dew else ew, -ns if dns else ns))
                out_h.append(np.where(h < 0, h + 360, h))
                for scale in (1.0, 4.0):                  # parseBDS09_1 subtypes 1 and 2
                    ns1, ew1 = vns * scale, float(vew) * scale
                    out_v.append(np.hypot(ns1, ew1))
                    ews = -ew1 if dew else ew1
                    with np.errstate(divide="ignore", invalid="ignore"):
                        h = np.where(ns1 == 0, 0.0, np.degrees(np.arctan(ews / np.where(ns1 == 0, 1, ns1))))
                    h = 180 - h if dns else h
                    out_h.append(np.where(h < 0, h + 360, h))
    return np.unique(np.concatenate(out_v)), np.unique(np.concatenate(out_h))


def test_every_bds09_velocity_and_heading(shim):
    v, h = _bds09_values()
    _check_fixed(shim, v, 1)
    _check_fixed(shim, h, 1)


def test_every_vertical_rate(shim):
    vr = np.arange(512)
    vals = np.concatenate([vr * 32.0, -(vr * 32.0), (vr - 1) * 64.0, -((vr - 1) * 64.0), [-0.0, 0.5, -0.5, -0.9999, 1e18,
                                                                                           -2.0 ** 62]])
    out = np.zeros((len(vals), 32), dtype=np.uint8)
    shim.shim_trunc(C.c_void_p(vals.ctypes.data), len(vals), C.c_void_p(out.ctypes.data))
    assert _strings(out) == ["%i" % x for x in vals.tolist()]


def _edge_doubles():
    xs = [0.0, -0.0, 5e-324, -5e-324, 1e-300, -1e-7, -4e-6, -5e-6, -6e-6, 4e-6, 5e-6, 6e-6, 90.0, -90.0, 180.0, -180.0,
          179.999995, -179.999995, 89.999995, 0.05, 0.15, 0.25, 0.35, 1e15, -1e15, 2.0 ** 62]
    for m in range(1, 40):                               # exact binary ties k / 2^m and their neighbours
        for k in (1, 3, 5, 7, 9, 11, 13, 101, 1023):
            t = k / 2.0 ** m
            xs += [t, -t, np.nextafter(t, 0), np.nextafter(t, 1e9), 48.0 + t, -180.0 + t]
    for base in (0.0, 90.0, -90.0, 180.0, -180.0):
        for d in range(-50, 51):
            xs.append(base + d * 1e-6)
            xs.append(base + d * 5e-7)
    return np.array(xs, dtype=np.float64)


@pytest.mark.parametrize("prec", [1, 5])
def test_fixed_at_ties_signs_and_range_ends(shim, prec):
    _check_fixed(shim, _edge_doubles(), prec)


def test_fixed_on_a_million_random_doubles(shim):
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.uniform(-200, 200, 400_000), rng.uniform(-1e-3, 1e-3, 100_000),
                        np.ldexp(rng.uniform(-1, 1, 500_000), rng.integers(-60, 40, 500_000))])
    _check_fixed(shim, x, 5)
    _check_fixed(shim, x[:300_000], 1)


def _stamps(shim, secs, frac, tz):
    secs = np.ascontiguousarray(secs, dtype=np.uint64)
    frac = np.ascontiguousarray(frac, dtype=np.float64)
    out = np.zeros((len(secs), 32), dtype=np.uint8)
    shim.shim_stamp(C.c_void_p(secs.ctypes.data), C.c_void_p(frac.ctypes.data), len(secs), tz, C.c_void_p(out.ctypes.data))
    return _strings(out)


def test_date_and_time_against_datetime(shim):
    days = [datetime.datetime(y, m, d) for y, m, d in ((1970, 1, 1), (1972, 2, 28), (1972, 2, 29), (1972, 3, 1),
                                                       (1999, 12, 31), (2000, 2, 29), (2000, 12, 31), (2100, 2, 28),
                                                       (2100, 3, 1), (2400, 2, 29), (9999, 12, 31))]
    secs = []
    for d in days:
        s = int((d - so.EPOCH).total_seconds())
        secs += [s, s + 86399, s + 43200, s - 1]
    secs += [0, so.LAST_SEC, so.LAST_SEC + 1, so.LAST_SEC - 86400, 1_700_000_000, 2 ** 40]
    secs = [x for x in secs if x >= 0]                   # a frame's secs is unsigned
    fracs = [0.0, 0.5, float(np.nextafter(1.0, 0.0)), 0.9995, 1.5, 2.25, 0.001, 0.999]
    for k in range(0, 1000, 37):
        fracs += [float(np.nextafter(k / 1000, 0)), k / 1000, float(np.nextafter(k / 1000, 1))]
    s_all = np.repeat(secs, len(fracs))
    f_all = np.tile(fracs, len(secs))
    for tz in (0, -720, 840, -330, 60):
        got = _stamps(shim, s_all, f_all, tz)
        want = [" ".join(so.stamp(s, f, tz)).strip() for s, f in zip(s_all.tolist(), f_all.tolist())]
        assert got == want


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    from gr_air_modes_b200 import _lib
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def test_stamps_with_negative_huge_or_non_finite_frac(shim):
    """The normalisation secs += int(frac) is exact for any finite frac, a negative frac counts as 0 ms, and a frac that
    is not finite leaves the fields empty, as the checker (and the header) say."""
    cases = [(1_700_000_000, -0.5), (1_700_000_000, -1.5), (1_700_000_000, -0.0004), (0, -0.25), (5, 1e9 + 0.25),
             (2 ** 40, -(2.0 ** 40) + 1e9 + 0.5), (2 ** 63, -(2.0 ** 63)), (2 ** 64 - 1, -(2.0 ** 64) + 2.0 ** 12),
             (so.LAST_SEC + 1, -1.0), (so.LAST_SEC + 10 ** 9, -1e9), (7, 2.0 ** 70), (7, -(2.0 ** 70)),
             (7, math.nan), (7, math.inf), (7, -math.inf)]
    secs = [s for s, _ in cases]
    fracs = [f for _, f in cases]
    for tz in (0, 840, -720):
        got = _stamps(shim, secs, fracs, tz)
        want = [" ".join(so.stamp(s, f, tz)).strip() for s, f in cases]
        assert got == want, tz
    assert got[-1] == got[-2] == got[-3] == ""


def test_lines_of_the_mix_scene_through_the_shim(shim, emulated):
    """amb_sbs1_line on the records of an emulated decode, against the checker's line, record by record."""
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(sc.mix_scene())
    d = decode.batch_decoder(None)
    recs = d.decode(frames)
    d.close()
    out = C.create_string_buffer(256)
    n = 0
    for k, (f, r) in enumerate(zip(frames, recs)):
        rb = np.ascontiguousarray(recs[k:k + 1])
        shim.shim_line(C.c_void_p(rb.ctypes.data), k + 1, int(f["secs"]), float(f["frac"]), 0, out)
        want = so.line(r, k + 1, *so.stamp(int(f["secs"]), float(f["frac"]))) if so.published(r) else None
        assert out.value.decode() == (want or ""), k
        n += want is not None
    assert n > 100


def test_option_validation_in_python():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, True, False):
        assert decode.check_sbs1(ok) == int(ok)
    for bad in (2, -1, "1", 1.0, None):
        with pytest.raises(ValueError):
            decode.check_sbs1(bad)
    for ok in (-720, 0, 840, 330):
        assert decode.check_sbs1_tz(ok) == ok
    for bad in (-721, 841, 1.5, True, "0", None):
        with pytest.raises(ValueError):
            decode.check_sbs1_tz(bad)
    assert (_lib.SBS1_TZ_MIN, _lib.SBS1_TZ_MAX) == (-720, 840)
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    assert "#define AMB_SBS1_TZ_MIN (-720)" in hdr and "#define AMB_SBS1_TZ_MAX 840" in hdr
    for sym in ("amb_decoder_sbs1", "amb_decoder_sbs1_device"):
        assert any(s[0] == sym for s in _lib.SYMBOLS)


def test_option_validation_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    lib = d._lib
    n = C.c_size_t(7)
    assert lib.amb_decoder_sbs1(d._h, None, 0, C.byref(n)) == ERR_STATE and n.value == 0
    for name, v in ((b"sbs1", 2), (b"sbs1", -1), (b"sbs1_tz", 841), (b"sbs1_tz", -721), (b"sbs2", 1)):
        assert lib.amb_decoder_set_option(d._h, name, v) == ERR_INVALID
    with pytest.raises(RuntimeError):
        d.sbs1_text()
    d.set_sbs1(True)
    assert d.get_sbs1() and d.sbs1_text() == b""                          # on, nothing decoded yet
    d.set_sbs1_tz(-330)
    assert d.get_sbs1_tz() == -330
    for bad in (2, 841):
        with pytest.raises(ValueError):
            d.set_sbs1(bad) if bad == 2 else d.set_sbs1_tz(bad)
    d.close()


def test_a_stream_through_the_c_abi(emulated):
    """Records unchanged by the option, ten launches more per decode, the text equal to the checker's across calls and
    a reset, AMB_ERR_OVERFLOW with the size and nothing written."""
    from gr_air_modes_b200 import decode
    frames = tc.frames_of(sc.mix_scene())
    cuts = ((0, 100), (100, 333), (333, len(frames)))
    plain = decode.batch_decoder(None, local_cpr=10)
    want = [plain.decode(frames[a:b]) for a, b in cuts]
    k_plain = plain.stats()[0]
    plain.close()
    d = decode.batch_decoder(None, local_cpr=10, sbs1=True, sbs1_tz=60)
    chk = so.Sbs1Checker(60)
    for (a, b), w in zip(cuts, want):
        recs = d.decode(frames[a:b])
        assert recs.tobytes() == w.tobytes()
        assert d.sbs1_text() == chk.feed(frames[a:b], recs)
    assert d.stats()[0] == k_plain + 10 * len(cuts)
    lib = d._lib
    n = C.c_size_t()
    buf = C.create_string_buffer(b"\x5a" * 64)
    assert lib.amb_decoder_sbs1(d._h, buf, 10, C.byref(n)) == ERR_OVERFLOW
    assert n.value > 10
    assert buf.raw == b"\x5a" * 64 + b"\0"
    d.reset()
    chk.reset()
    recs = d.decode(frames[:50])
    assert d.sbs1_text() == chk.feed(frames[:50], recs)
    d.set_sbs1(False)
    with pytest.raises(RuntimeError):
        d.sbs1_text()
    d.close()


def _recv_all(sock, want, timeout=5.0):
    sock.settimeout(timeout)
    got = b""
    while len(got) < want:
        b = sock.recv(65536)
        if not b:
            break
        got += b
    return got


def test_server_two_clients_one_dropped():
    from gr_air_modes_b200.sbs1 import sbs1_server
    with sbs1_server(0, host="127.0.0.1") as srv:
        a = socket.create_connection(("127.0.0.1", srv.port))
        b = socket.create_connection(("127.0.0.1", srv.port))
        time.sleep(0.05)
        srv.send(b"MSG,8,0,1\r\n")
        assert srv.connections == 2
        assert _recv_all(a, 11) == b"MSG,8,0,1\r\n" and _recv_all(b, 11) == b"MSG,8,0,1\r\n"
        b.close()
        for k in range(50):                              # the closed client fails a send and is dropped
            srv.send(b"MSG,8,0,%d\r\n" % k)
            if srv.connections == 1:
                break
            time.sleep(0.01)
        assert srv.connections == 1
        srv.send(b"last\r\n")
        a.shutdown(socket.SHUT_WR)
        time.sleep(0.05)
        srv.close()
        assert _recv_all(a, 1 << 20).endswith(b"last\r\n")   # the remaining client got every line
        a.close()
    assert srv.connections == 0


def test_server_drops_a_client_that_stops_reading():
    from gr_air_modes_b200.sbs1 import sbs1_server
    with sbs1_server(0, host="127.0.0.1", max_backlog=1 << 18) as srv:
        slow = socket.socket()
        slow.setsockopt(socket.SOL_SOCKET, socket.SO_RCVBUF, 4096)
        slow.connect(("127.0.0.1", srv.port))
        time.sleep(0.05)
        chunk = b"x" * 65536
        for _ in range(200):
            srv.send(chunk)                              # never blocks
            if srv.connections == 0:
                break
        assert srv.connections == 0                      # never read: dropped once its backlog passed the bound
        slow.close()


def test_server_keeps_a_reading_client_through_a_large_send():
    """One chunk's text in one send: a client that reads continuously gets every byte, through later sends and the
    flush at close, and is not dropped."""
    import threading
    from gr_air_modes_b200.sbs1 import sbs1_server
    srv = sbs1_server(0, host="127.0.0.1")
    c = socket.create_connection(("127.0.0.1", srv.port))
    got = []
    t = threading.Thread(target=lambda: got.append(b"".join(iter(lambda: c.recv(65536), b""))))
    t.start()
    time.sleep(0.05)
    big = bytes(range(256)) * (4 << 12)                  # 4 MiB
    srv.send(big)
    assert srv.connections == 1
    for k in range(20):
        srv.send(b"MSG,8,0,%d\r\n" % k)
        time.sleep(0.005)
    assert srv.connections == 1
    srv.close(linger=10.0)
    t.join(timeout=10)
    c.close()
    assert got[0] == big + b"".join(b"MSG,8,0,%d\r\n" % k for k in range(20))


def test_server_waits_for_a_first_client():
    from gr_air_modes_b200.sbs1 import sbs1_server
    with sbs1_server(0, host="127.0.0.1") as srv:
        t0 = time.monotonic()
        assert not srv.wait_for_client(0.2) and time.monotonic() - t0 >= 0.19
        c = socket.create_connection(("127.0.0.1", srv.port))
        assert srv.wait_for_client(5.0) and srv.connections == 1
        c.close()


def test_cli_arguments():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200 as m
    a = m.parse_args(["-s", "x.cfile", "-P"])
    assert a.sbs1 == 30003
    assert m.parse_args(["-s", "x.cfile", "--sbs1", "4000", "-l", "1,2", "--local-cpr", "10"]).sbs1 == 4000
    assert m.parse_args(["-s", "x.cfile"]).sbs1 is None
    assert m.parse_args(["-s", "x.cfile", "-P", "--sbs1-wait", "5"]).sbs1_wait == 5
    for bad in (["-P", "0"], ["-P", "70000"], ["-P", "abc"], ["--sbs1-wait", "5"], ["-P", "--sbs1-wait", "-1"]):
        with pytest.raises(SystemExit):
            m.parse_args(["-s", "x.cfile"] + bad)
    assert -720 <= m.local_utc_offset_minutes() <= 840
    doc = open(os.path.join(ROOT, "tools", "modes_rx_b200.py")).read()
    assert "SBS-1 and FlightGear outputs are the reference's own" not in doc
