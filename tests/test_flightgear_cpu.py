"""The FlightGear checker (tests/flightgear_oracle.py) against the UNMODIFIED reference python/flightgear.py: every
packet of tests/golden/flightgear_golden.json.gz (made by tests/golden/make_flightgear_golden.py from
output_flightgear.output and fg_posmsg.pack), replayed on the records of the decoder's per-message arithmetic compiled
for the host (tests/decode_host_shim.cc), and the packer grid. The decoder's packet math (amb_fg_format.h) compiled for
the host equals the checker byte for byte over the grid and 10^6 random inputs. The option's bounds and message through
the emulated C ABI, fg_sender on loopback, and the CLI's -m rules."""
import ctypes as C
import gzip
import json
import os
import socket
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import emul_build  # noqa: E402
import flightgear_oracle as fo  # noqa: E402
import track_cases as tc  # noqa: E402

MODEL_NAMES = {"HEAVY": 5, "PARACHUTE": fo.SANTA}


def golden():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "flightgear_golden.json.gz")) as f:
        return json.loads(f.read())


@pytest.fixture(scope="module")
def decode_shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "decode_host_shim.cc")))
    lib.shim_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def fg_shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "flightgear_host_shim.cc")))
    lib.shim_fg_packets.argtypes = [C.c_void_p] * 9 + [C.c_long, C.c_void_p, C.c_void_p]
    return lib


def records(shim, msgs, loc):
    from gr_air_modes_b200 import decode
    frames = tc.frames_of([tuple(m) for m in msgs], unqueued_every=0)
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    have, lat, lon = (0, 0.0, 0.0) if loc is None else (1, float(loc[0]), float(loc[1]))
    assert shim.shim_decode(C.c_void_p(frames.ctypes.data), len(frames), have, lat, lon, C.c_void_p(recs.ctypes.data)) == 0
    return frames, recs


def host_packets(shim, rows):
    """amb_fg_packet compiled for the host over rows of (ident, model, lat, lon, alt, t, hdg, vel_ms, turn)."""
    n = len(rows)
    ident = b"".join(r[0] for r in rows)
    cols = list(zip(*[r[1:] for r in rows]))
    model = np.array(cols[0], dtype=np.int32)
    dbl = [np.array(c, dtype=np.float64) for c in cols[1:6]]
    flt = [np.array(c, dtype=np.float32) for c in cols[6:8]]
    out = C.create_string_buffer(fo.PACKET_BYTES * n)
    ok = np.zeros(n, dtype=np.int32)
    shim.shim_fg_packets(ident, model.ctypes.data, *[a.ctypes.data for a in dbl], *[a.ctypes.data for a in flt], n, out,
                         ok.ctypes.data)
    raw = out.raw
    return [raw[i * fo.PACKET_BYTES: (i + 1) * fo.PACKET_BYTES] if ok[i] else None for i in range(n)]


def test_golden_covers_every_rule():
    g = golden()
    errs = [o[1] for sc in g["scenes"] for o in sc["out"]]
    assert "IndexError" in errs
    assert sum(g_[5] == "TypeError" for g_ in g["grid"]) >= 2
    packets = [bytes.fromhex(p) for sc in g["scenes"] for o in sc["out"] for p in o[0]]
    assert len(packets) > 1000 and all(len(p) == fo.PACKET_BYTES and p[:4] == b"FGFS" for p in packets)
    models = {p[32:128].rstrip(b"\0").decode() for p in packets}
    assert len(models) >= 14 and fo.MODELS[fo.SANTA] in models


@pytest.mark.parametrize("name", [sc["name"] for sc in golden()["scenes"]])
def test_checker_reproduces_the_reference_golden(decode_shim, name):
    sc = next(s for s in golden()["scenes"] if s["name"] == name)
    frames, recs = records(decode_shim, sc["msgs"], sc["location"])
    chk = fo.FgChecker()
    for k, (f, r) in enumerate(zip(frames, recs)):
        p = chk.record(f, r)
        want = sc["out"][k][0]
        assert ([p.hex()] if p is not None else []) == want, (name, k, sc["out"][k][1])


def _grid_rows(g):
    callsign, model, vel, turn, t = g["grid_args"]
    m = MODEL_NAMES[model]
    return [(callsign.encode(), m, lat, lon, float(alt), t, hdg, fo.f32(vel * 0.514444444), fo.f32(turn * (np.pi / 180.)))
            for lat, lon, alt, hdg, _, _ in g["grid"]]


def test_checker_and_host_packet_math_reproduce_the_packer_grid(fg_shim):
    g = golden()
    rows = _grid_rows(g)
    host = host_packets(fg_shim, rows)
    for row, (_, _, _, _, want, err), h in zip(rows, g["grid"], host):
        p = fo.packet(*row)
        assert (p.hex() if p is not None else None) == want, (row, err)
        assert h == p, row
        assert (err == "TypeError") == (p is None)


def test_host_packet_math_equals_the_checker_on_random_inputs(fg_shim):
    rng = np.random.default_rng(2024)
    n = 1_000_000
    lat, lon = rng.uniform(-90, 90, n), rng.uniform(-180, 180, n)
    hdg = np.where(rng.random(n) < 0.5, rng.uniform(0, 360, n), rng.integers(0, 1440, n) / 4.0)
    alt = rng.integers(-1000, 50000, n).astype(np.float64)
    t = 1.7e9 + rng.uniform(0, 1e6, n)
    vel = rng.uniform(0, 600, n) * 0.514444444
    turn = rng.uniform(-3, 3, n) * (np.pi / 180.)
    model = rng.integers(0, 16, n)
    rows = [(b"R%07d" % i, int(model[i]), float(lat[i]), float(lon[i]), float(alt[i]), float(t[i]), float(hdg[i]),
             fo.f32(float(vel[i])), fo.f32(float(turn[i]))) for i in range(n)]
    host = host_packets(fg_shim, rows)
    bad = [i for i in range(n) if host[i] != fo.packet(*rows[i])]
    assert not bad, bad[:5]


def test_model_table_is_the_reference_rows(fg_shim):
    for ftc in range(0, 6):
        for cat in range(-1, 9):
            want = fo.model(ftc, cat)
            assert fg_shim.shim_fg_model(ftc, cat) == (-1 if want is None else want), (ftc, cat)


# ---- the option, the sender and the CLI ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    e = C.CDLL(emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL))
    e.amb_decoder_create.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.POINTER(C.c_void_p)]
    e.amb_decoder_destroy.argtypes = [C.c_void_p]
    e.amb_decoder_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    e.amb_decoder_last_error.argtypes = [C.c_void_p]
    e.amb_decoder_last_error.restype = C.c_char_p
    return e


def test_option_bounds_and_message(lib):
    h = C.c_void_p()
    assert lib.amb_decoder_create(0, 0, 0.0, 0.0, C.byref(h)) == 0
    try:
        for v in (0, 1, 0):
            assert lib.amb_decoder_set_option(h, b"flightgear", v) == 0
        for bad in (-1, 2, 1 << 30):
            assert lib.amb_decoder_set_option(h, b"flightgear", bad) == -1
            assert lib.amb_decoder_last_error(h) == b"flightgear: 0 (off) or 1 (on)"
    finally:
        lib.amb_decoder_destroy(h)
    from gr_air_modes_b200 import decode
    assert decode.OPTIONS["flightgear"] == ("switch", 0, 1)
    assert decode.check_flightgear(True) == 1 and decode.check_flightgear(0) == 0
    with pytest.raises(ValueError):
        decode.check_flightgear(2)


def test_fg_sender_on_loopback():
    from gr_air_modes_b200 import flightgear
    rx = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    rx.bind(("127.0.0.1", 0))
    rx.settimeout(5)
    try:
        pk = [fo.packet(b"ABC     ", 3, 47.9, 11.1, 1000.0, 1.7e9 + i, 90.0 * i, 100.0, 0.0) for i in range(4)]
        with flightgear.fg_sender("127.0.0.1", rx.getsockname()[1]) as s:
            assert s.send(b"".join(pk)) == 4 and s.sent == 4 and s.dropped == 0
            assert s.send(b"") == 0
            with pytest.raises(ValueError):
                s.send(pk[0][:-1])
            got = [rx.recvfrom(2048)[0] for _ in range(4)]
        assert got == pk and flightgear.PACKET_BYTES == fo.PACKET_BYTES
        assert struct.unpack("!4sLLL", got[0][:16]) == (b"FGFS", 0x00010001, 7, 232)
    finally:
        rx.close()


def test_fg_sender_drops_instead_of_blocking():
    """A closed port: the kernel reports ICMP port unreachable on a later send; it is counted, never raised."""
    from gr_air_modes_b200 import flightgear
    probe = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    probe.bind(("127.0.0.1", 0))
    port = probe.getsockname()[1]
    probe.close()
    pk = fo.packet(b"ABC     ", 3, 47.9, 11.1, 1000.0, 1.7e9, 45.0, 100.0, 0.0)
    with flightgear.fg_sender("127.0.0.1", port) as s:
        for _ in range(5):
            s.send(pk * 3)
        assert s.sent + s.dropped == 15


def test_cli_multiplayer_rules():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200 as m
    assert m.parse_args(["-s", "x.cfile", "-m", "127.0.0.1:5000"]).multiplayer == ("127.0.0.1", 5000)
    assert m.parse_args(["-s", "x.cfile", "--multiplayer", "fg.example:5002", "-l", "1,2"]).multiplayer == ("fg.example", 5002)
    assert m.parse_args(["-s", "x.cfile"]).multiplayer is None
    assert m.parse_args(["--input", "beast", "-s", "feed.bin", "-m", "localhost:5000"]).multiplayer == ("localhost", 5000)
    for bad in ("localhost", "localhost:0", "localhost:70000", ":5000", "host:port"):
        with pytest.raises(SystemExit):
            m.parse_args(["-s", "x.cfile", "-m", bad])
    doc = m.__doc__
    assert "KML and FlightGear outputs are the reference's" not in doc and "-m HOST:PORT" in doc
