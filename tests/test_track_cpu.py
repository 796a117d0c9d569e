"""Decoder option "track" without a GPU: option validation in Python and through the C ABI of the emulated library
(tests/simt/library_emul.cc: the library's own sources on the SIMT emulator), a small stream through that C ABI against
the checker, the AIRCRAFT_DTYPE layout against the header's struct amb_aircraft (compiled on the host), aircraft_to_dict,
and the CLI's --track / --aircraft with a stand-in decoder."""
import ctypes as C
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import track_cases as tc  # noqa: E402
import track_oracle as to  # noqa: E402

FIELDS = ("icao", "messages", "first_seen", "seen", "ref_level", "flags", "ftc", "cat", "ident", "altitude", "squawk",
          "lat", "lon", "range", "bearing", "pos_t", "speed", "heading", "vertical", "eps", "pad_")
LAYOUT_SHIM = r"""
#include <stddef.h>
#include "airmodes_b200.h"
#define F(name) offsetof(amb_aircraft, name), sizeof(((amb_aircraft*)0)->name)
static const size_t table[] = {%s};
int shim_aircraft_layout(size_t* out) { for (size_t k = 0; k < sizeof table / sizeof table[0]; k++) out[k] = table[k];
                                        return (int)sizeof(amb_aircraft); }
"""


def test_option_validation_in_python():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, 3600, 60.0):
        assert decode.check_track(ok) == int(ok)
    for bad in (-1, 3601, 1.5, True, None, "x"):
        with pytest.raises(ValueError):
            decode.check_track(bad)
    assert _lib.TRACK_MAX == decode.TRACK_MAX == 3600
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    assert re.search(r"#define AMB_TRACK_MAX 3600\b", hdr)
    for name in ("HAS_ALT", "HAS_SQUAWK", "HAS_IDENT", "HAS_POS", "HAS_RANGE", "HAS_VELOCITY", "HAS_HEADING", "HAS_EPS",
                 "ON_GROUND"):
        v = int(re.search(r"#define AMB_AC_%s (0x[0-9a-fA-F]+)" % name, hdr).group(1), 16)
        assert getattr(decode, "AC_" + name) == getattr(to, "AC_" + name) == v, name
    for sym in ("amb_decoder_aircraft", "amb_decoder_aircraft_device"):
        assert (sym, C.c_int, [C.c_void_p, C.c_double, C.c_void_p, C.c_int]) in _lib.SYMBOLS


def test_aircraft_layout_matches_the_header(tmp_path):
    from gr_air_modes_b200 import decode
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_SHIM % ", ".join("F(%s)" % f for f in FIELDS))
    lib = str(tmp_path / "liblayout.so")
    subprocess.run(["gcc", "-std=c99", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-o", lib, str(src)],
                   check=True)
    s = C.CDLL(lib)
    out = (C.c_size_t * (2 * len(FIELDS)))()
    assert s.shim_aircraft_layout(out) == 128 == decode.AIRCRAFT_DTYPE.itemsize
    assert decode.AIRCRAFT_DTYPE.names == FIELDS
    for k, f in enumerate(FIELDS):
        dt, off = decode.AIRCRAFT_DTYPE.fields[f][:2]
        assert (out[2 * k], out[2 * k + 1]) == (off, dt.itemsize), f


def test_aircraft_to_dict():
    from gr_air_modes_b200 import decode
    row = to.pack([to._blank(0xABCDEF, 12.5)])[0]
    row["messages"], row["ref_level"] = 3, np.float32(1e-10)
    d = decode.aircraft_to_dict(row)
    assert d["icao"] == 0xABCDEF and d["messages"] == 3 and d["first_seen"] == 12.5 and d["rssi"] == -80.0
    for k in ("altitude", "squawk", "ident", "ftc", "cat", "lat", "lon", "pos_t", "range", "bearing", "speed", "heading",
              "vertical", "eps"):
        assert d[k] is None, k
    assert d["on_ground"] is False
    row["flags"] = to.AC_HAS_IDENT | to.AC_HAS_POS | to.AC_ON_GROUND | to.AC_HAS_ALT
    row["ident"] = np.frombuffer(b"KLM1234 ", dtype="S1")
    row["lat"], row["lon"], row["altitude"], row["ref_level"] = 52.25, 4.5, 0, np.float32(0.5)
    d = decode.aircraft_to_dict(row)
    assert d["ident"] == "KLM1234 " and d["lat"] == 52.25 and d["altitude"] == 0 and d["on_ground"] is True
    assert d["range"] is None and d["speed"] is None and abs(d["rssi"] - 10 * math.log10(0.5)) < 1e-12
    json.dumps(d)


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    from gr_air_modes_b200 import _lib
    out = str(tmp_path_factory.mktemp("libsimt_track") / "libairmodes_b200_emulated.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas",
                    "-Wno-psabi", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "simt", "library_emul.cc")],
                   check=True)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        yield out
    finally:
        _lib.LIB_PATH, _lib._lib = saved


def test_option_validation_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    lib = d._lib
    for name, v in ((b"track", 3601), (b"track", -1), (b"tracks", 5)):
        assert lib.amb_decoder_set_option(d._h, name, v) == -1
    assert d.get_track() == 0
    assert lib.amb_decoder_aircraft(d._h, math.nan, None, 0) == -8          # AMB_ERR_STATE: the option is off
    with pytest.raises(RuntimeError):
        d.aircraft()
    for bad in (-1, 3601):
        with pytest.raises(ValueError):
            d.set_track(bad)
    d.set_track(3600)
    assert d.get_track() == 3600 and len(d.aircraft()) == 0                # on, nothing decoded yet
    d.close()


def test_a_stream_through_the_c_abi(emulated):
    """The burst scene (one address, rows expiring and recreated inside a 32-record step) through the emulated
    library's decoder: records unchanged by the option, launches counted, snapshots equal to the checker's."""
    from gr_air_modes_b200 import decode
    msgs = tc.burst_scene()[:120]
    frames = tc.frames_of(msgs)
    off = decode.batch_decoder(None)
    want = off.decode(frames)
    off.close()
    d = decode.batch_decoder(None, track=3)
    tr = to.Tracker(3)
    got = []
    for a, b in ((0, 33), (33, 120)):
        got.append(d.decode(frames[a:b]))
        tr.feed(frames[a:b], got[-1])
    assert np.concatenate(got).tobytes() == want.tobytes()
    k0 = d.stats()[0]
    assert k0 == 2 * 13
    snap = d.aircraft()
    assert d.stats()[0] == k0 + 2 + 3                      # aircraft(): a count, then count + scan + gather
    to.assert_rows_equal(snap, tr.snapshot_array(), "emulated C ABI")
    assert len(snap) == 2 and snap["messages"][0] < 100
    n = d._lib.amb_decoder_aircraft(d._h, math.nan, None, 0)
    buf = np.zeros(n, dtype=decode.AIRCRAFT_DTYPE)
    assert d._lib.amb_decoder_aircraft(d._h, math.nan, C.c_void_p(buf.ctypes.data), n - 1) == -5   # AMB_ERR_OVERFLOW
    assert not buf.view(np.uint8).any()
    d.reset()
    assert len(d.aircraft()) == 0 and d.get_track() == 3
    d.close()


class _FakeDecoder:
    def __init__(self):
        self.batches = []

    def decode_messages(self, texts):
        from gr_air_modes_b200 import decode
        self.batches.append(list(texts))
        return np.zeros(len(texts), dtype=decode.FIELDS_DTYPE)

    def aircraft(self):
        rows = [to._blank(0x4840D6, 1.0), to._blank(0x3C6444, 2.0)]
        rows[0]["flags"], rows[0]["altitude"] = to.AC_HAS_ALT, 37000
        return to.pack(rows)


class _Msg:
    def __init__(self, text):
        self.text = text

    def to_string(self):
        return self.text


def _cli():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import modes_rx_b200
    return modes_rx_b200


def test_cli_parsing():
    cli = _cli()
    a = cli.parse_args(["-s", "x.cfile", "--track", "60", "--aircraft", "out.json"])
    assert a.track == 60 and a.aircraft == "out.json"
    assert cli.parse_args(["-s", "x.cfile"]).track == 0
    for bad in (["--aircraft", "out.json"], ["--track", "0", "--aircraft", "o.json"], ["--track", "3601"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["-s", "x.cfile"] + bad)


def test_cli_writes_the_table_after_every_batch(tmp_path):
    cli = _cli()
    path = str(tmp_path / "aircraft.json")
    fake = _FakeDecoder()
    q = cli.report_queue(None, 0, out=None, aircraft=path, decoder=fake)
    q.handle(_Msg("8d4840d6202cc371c32ce0576098 000000 0.5 1 0.25"))
    q.flush()
    assert len(fake.batches) == 1
    rows = json.load(open(path))
    assert [r["icao"] for r in rows] == [0x4840D6, 0x3C6444]
    assert rows[0]["altitude"] == 37000 and rows[1]["altitude"] is None and rows[0]["lat"] is None
    q.flush()                                                  # nothing queued: no decode, the file is written again
    assert len(fake.batches) == 1 and json.load(open(path)) == rows
    assert sorted(os.listdir(str(tmp_path))) == ["aircraft.json"]
