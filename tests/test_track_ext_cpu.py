"""Decoder option "track_ext" without a GPU: the AIRCRAFT_EXT_DTYPE layout against the header's struct amb_aircraft_ext
(compiled on the host), option validation in Python and through the C ABI of the emulated library
(tests/simt/library_emul.cc: the library's own sources on the SIMT emulator), a stream through that C ABI against the
checker, aircraft_ext_to_dict against opstatus_values / commb_values of the records that wrote the groups, and the CLI's
--track-ext with a stand-in decoder."""
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

import emul_build  # noqa: E402
import track_cases as tc  # noqa: E402
import track_ext_cases as xc  # noqa: E402
import track_ext_oracle as xo  # noqa: E402
import track_oracle as to  # noqa: E402

FIELDS = ("icao", "shown", "ops_version", "integ_es", "integ_version", "t", "ops", "ts", "integ", "integ_nic",
          "commb_mask", "commb_outcome", "pad0_", "commb", "pad_")
LAYOUT_SHIM = r"""
#include <stddef.h>
#include "airmodes_b200.h"
#define F(name) offsetof(amb_aircraft_ext, name), sizeof(((amb_aircraft_ext*)0)->name)
static const size_t table[] = {%s};
int shim_ext_layout(size_t* out) { for (size_t k = 0; k < sizeof table / sizeof table[0]; k++) out[k] = table[k];
                                   return (int)sizeof(amb_aircraft_ext); }
"""
ERR_INVALID, ERR_OVERFLOW, ERR_STATE = -1, -5, -8


def test_ext_layout_matches_the_header(tmp_path):
    from gr_air_modes_b200 import decode
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_SHIM % ", ".join("F(%s)" % f for f in FIELDS))
    lib = str(tmp_path / "liblayout.so")
    subprocess.run(["gcc", "-std=c99", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-o", lib, str(src)],
                   check=True)
    s = C.CDLL(lib)
    out = (C.c_size_t * (2 * len(FIELDS)))()
    assert s.shim_ext_layout(out) == 144 == decode.AIRCRAFT_EXT_DTYPE.itemsize
    assert decode.AIRCRAFT_EXT_DTYPE.names == FIELDS
    for k, f in enumerate(FIELDS):
        dt, off = decode.AIRCRAFT_EXT_DTYPE.fields[f][:2]
        assert (out[2 * k], out[2 * k + 1]) == (off, dt.itemsize), f


def test_option_validation_in_python():
    from gr_air_modes_b200 import _lib, decode
    for ok in (0, 1, 3600, 60.0):
        assert decode.check_option("track_ext", ok) == int(ok)
    for bad in (-1, 3601, 1.5, True, None, "x"):
        with pytest.raises(ValueError):
            decode.check_option("track_ext", bad)
    assert _lib.TRACK_EXT_MAX == decode.TRACK_EXT_MAX == decode.OPTION_MAX["track_ext"] == 3600
    hdr = open(os.path.join(ROOT, "include", "airmodes_b200.h")).read()
    assert re.search(r"#define AMB_TRACK_EXT_MAX 3600\b", hdr)
    for k, name in enumerate(("OPS", "TS", "INTEG", "B40", "B50", "B60")):
        v = int(re.search(r"#define AMB_AXG_%s (0x[0-9a-fA-F]+)" % name, hdr).group(1), 16)
        assert getattr(decode, "AXG_" + name) == v == 1 << k, name
    for sym in ("amb_decoder_aircraft_ext", "amb_decoder_aircraft_ext_device"):
        assert (sym, C.c_int, [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_int]) in _lib.SYMBOLS


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


def test_option_validation_through_the_c_abi(emulated):
    from gr_air_modes_b200 import decode
    d = decode.batch_decoder(None)
    lib = d._lib
    for name, v in ((b"track_ext", 3601), (b"track_ext", -1), (b"track_exts", 5)):
        assert lib.amb_decoder_set_option(d._h, name, v) == ERR_INVALID
    assert d.get_track_ext() == 0
    assert lib.amb_decoder_aircraft_ext(d._h, math.nan, None, None, 0) == ERR_STATE      # track off
    d.set_track_ext(60)
    assert d.get_track_ext() == 60
    assert lib.amb_decoder_aircraft_ext(d._h, math.nan, None, None, 0) == ERR_STATE      # track still off
    with pytest.raises(RuntimeError):
        d.aircraft_ext()
    d.set_track(60)
    d.set_track_ext(0)
    assert lib.amb_decoder_aircraft_ext(d._h, math.nan, None, None, 0) == ERR_STATE      # track_ext off
    for bad in (-1, 3601):
        with pytest.raises(ValueError):
            d.set_track_ext(bad)
    d.set_track_ext(3600)
    rows, ext = d.aircraft_ext()
    assert len(rows) == len(ext) == 0                                                   # on, nothing decoded yet
    d.close()


def _stream(decode, track_ext, S=20, S2=30):
    """The absence scene through the emulated library's decoder in two calls: (decoder, records, checker)."""
    frames = tc.frames_of(xc.absence_scene(S=10))
    d = decode.batch_decoder(None, opstatus=30, commb=30, track=S, track_ext=track_ext)
    chk = xo.ExtTracker(S, S2)
    recs = []
    for a, b in ((0, 33), (33, len(frames))):
        recs.append(d.decode(frames[a:b]))
        chk.feed(frames[a:b], recs[-1])
    return d, np.concatenate(recs), chk


def test_a_stream_through_the_c_abi(emulated):
    """Records and base snapshot unchanged by the option, six launches more per decode, three per snapshot, the
    snapshot equal to the checker's, AMB_ERR_OVERFLOW without a write, reset."""
    from gr_air_modes_b200 import decode
    plain, want, _ = _stream(decode, 0)
    k_plain = plain.stats()[0]
    base = plain.aircraft()
    plain.close()
    d, got, chk = _stream(decode, 30)
    assert got.tobytes() == want.tobytes()
    k0 = d.stats()[0]
    assert k0 == k_plain + 2 * 6
    rows, ext = d.aircraft_ext()
    assert d.stats()[0] == k0 + 2 + 3                       # a count, then count + scan + gather
    assert rows.tobytes() == base.tobytes() == d.aircraft().tobytes()
    xo.assert_snapshots_equal((rows, ext), chk.snapshot_arrays(), "emulated C ABI")
    assert len(rows) == 3 and np.all(ext["shown"] & decode.AXG_INTEG)
    n = len(rows)
    buf, xbuf = np.zeros(n, dtype=decode.AIRCRAFT_DTYPE), np.zeros(n, dtype=decode.AIRCRAFT_EXT_DTYPE)
    assert d._lib.amb_decoder_aircraft_ext(d._h, math.nan, C.c_void_p(buf.ctypes.data), C.c_void_p(xbuf.ctypes.data),
                                           n - 1) == ERR_OVERFLOW
    assert not buf.view(np.uint8).any() and not xbuf.view(np.uint8).any()
    assert d._lib.amb_decoder_aircraft_ext(d._h, math.nan, C.c_void_p(buf.ctypes.data), None, n) == ERR_INVALID
    d.reset()
    assert len(d.aircraft_ext()[0]) == 0 and d.get_track_ext() == 30
    d.close()


def test_aircraft_ext_to_dict_equals_the_writing_records(emulated):
    from gr_air_modes_b200 import decode
    d, recs, chk = _stream(decode, 30)
    rows, ext = d.aircraft_ext()
    d.close()
    frames = tc.frames_of(xc.absence_scene(S=10))
    t = frames["secs"].astype(float) + frames["frac"]
    keys = ("opstatus", "target_state", "integrity", "bds40", "bds50", "bds60")
    seen = set()
    for row, x in zip(rows, ext):
        got = decode.aircraft_ext_to_dict(row, x)
        assert {k: v for k, v in got.items() if k not in keys} == decode.aircraft_to_dict(row)
        for g, key in enumerate(keys):
            if not x["shown"] & (1 << g):
                assert got[key] is None
                continue
            k = max(i for i in range(len(recs)) if xo.group_of(recs[i]) == g and recs[i]["icao"] == row["icao"])
            want = decode.opstatus_values(recs[k]) if g < 3 else decode.commb_values(recs[k])
            assert got[key] == {"t": float(t[k]), **want}, key
            seen.add(g)
        json.dumps(got)
    assert seen == set(range(6))


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

    def aircraft_ext(self):
        from gr_air_modes_b200 import decode
        ext = np.zeros(2, dtype=decode.AIRCRAFT_EXT_DTYPE)
        ext["icao"] = (0x4840D6, 0x3C6444)
        ext["t"] = math.nan
        ext[0]["shown"] = decode.AXG_B50
        ext[0]["t"][4] = 1.5
        ext[0]["commb_outcome"][1], ext[0]["commb_mask"][1] = 1, 0x04
        ext[0]["commb"][1][2] = 200
        return self.aircraft(), ext


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
    a = cli.parse_args(["-s", "x.cfile", "--track", "60", "--track-ext", "120", "--aircraft", "out.json",
                        "--opstatus", "30", "--commb", "30"])
    assert a.track_ext == 120 and a.opstatus == 30 and a.commb == 30
    assert cli.parse_args(["-s", "x.cfile"]).track_ext == 0
    for bad in (["--track-ext", "60"], ["--track", "60", "--track-ext", "3601"], ["--track", "60", "--track-ext", "-1"],
                ["--track", "60", "--opstatus", "30", "--aircraft", "o.json"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["-s", "x.cfile"] + bad)


def _write(cli, tmp_path, track_ext):
    path = str(tmp_path / ("aircraft%d.json" % track_ext))
    q = cli.report_queue(None, 0, out=None, aircraft=path, decoder=_FakeDecoder(), track_ext=track_ext)
    q.handle(_Msg("8d4840d6202cc371c32ce0576098 000000 0.5 1 0.25"))
    q.flush()
    return open(path).read()


def test_cli_json_with_and_without_track_ext(tmp_path):
    cli = _cli()
    from gr_air_modes_b200 import decode
    plain = _write(cli, tmp_path, 0)
    assert plain == json.dumps([decode.aircraft_to_dict(r) for r in _FakeDecoder().aircraft()])
    rows = json.loads(_write(cli, tmp_path, 60))
    assert [r["icao"] for r in rows] == [0x4840D6, 0x3C6444]
    base = json.loads(plain)
    for r, b in zip(rows, base):
        assert {k: v for k, v in r.items() if k in b} == b
    assert rows[0]["bds50"]["t"] == 1.5 and rows[0]["bds50"]["gs"] == 400.0 and rows[0]["bds50"]["roll"] is None
    assert rows[0]["opstatus"] is None and rows[1]["bds50"] is None
