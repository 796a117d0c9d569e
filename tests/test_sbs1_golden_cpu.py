"""The SBS-1 checker (tests/sbs1_oracle.py) against the UNMODIFIED reference python/sbs1.py: every line and every
aircraft id of tests/golden/sbs1_golden.json.gz (made by tests/golden/make_sbs1_golden.py from output_sbs1.parse),
replayed on the records of the decoder's per-message arithmetic compiled for the host (tests/decode_host_shim.cc), and
the same on fresh seeds against the live reference modules where the reference tree is present. The GPU twin,
tests/test_sbs1_gpu.py::test_golden_scenes_on_the_device, compares the device's text with the same golden."""
import ctypes as C
import gzip
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import emul_build  # noqa: E402
import sbs1_oracle as so  # noqa: E402
import track_cases as tc  # noqa: E402

REF = os.path.join(os.environ.get("AMB_REFERENCE_TREE", "/root/reference"), "python")


def golden():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "sbs1_golden.json.gz")) as f:
        return json.loads(f.read())["scenes"]


def golden_text(scene) -> bytes:
    return "".join(line for _, _, line, _ in scene["out"] if line is not None).encode("ascii")


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(ROOT, "tests", "decode_host_shim.cc")))
    lib.shim_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    return lib


def _records(shim, msgs, loc):
    from gr_air_modes_b200 import decode
    frames = tc.frames_of([tuple(m) for m in msgs], unqueued_every=0)
    recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
    have, lat, lon = (0, 0.0, 0.0) if loc is None else (1, float(loc[0]), float(loc[1]))
    assert shim.shim_decode(C.c_void_p(frames.ctypes.data), len(frames), have, lat, lon, C.c_void_p(recs.ctypes.data)) == 0
    return frames, recs


def _check(shim, msgs, loc, out, name):
    frames, recs = _records(shim, msgs, loc)
    ids = []
    text = so.Sbs1Checker().feed(frames, recs, ids)
    assert [bool(so.published(r)) for r in recs] == [bool(o[0]) for o in out], name
    assert ids == [o[1] for o in out if o[0]], name
    want = "".join(o[2] for o in out if o[2] is not None).encode("ascii")
    assert text == want, name


def test_golden_covers_every_line_kind_and_both_escaping_errors():
    kinds, errors = set(), set()
    for sc in golden():
        for _, _, line, err in sc["out"]:
            if line is not None:
                kinds.add(line.split(",")[1])
            if err is not None:
                errors.add(err)
    assert kinds == {"1", "2", "3", "4", "5", "6", "7", "8"}
    assert errors == {"ValueError", "IndexError"}


@pytest.mark.parametrize("name", [sc["name"] for sc in golden()])
def test_checker_reproduces_the_reference_golden(shim, name):
    sc = next(s for s in golden() if s["name"] == name)
    _check(shim, sc["msgs"], sc["location"], sc["out"], name)


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "sbs1.py")), reason="the reference's Python sources are not present")
def test_checker_against_the_live_reference_on_fresh_seeds(shim):
    import decode_cases as dc
    import make_sbs1_golden as mk
    import sbs1_cases as sc
    mods = mk.load_reference()
    try:
        for seed in (101, 102, 103):
            msgs = sc.mix_scene(seed=seed)
            _check(shim, msgs, mk.SBS1_LOCATION, mk.run_reference(mk.SBS1_LOCATION, msgs, mods), ("mix", seed))
            loc, msgs = dc.make_case(seed=seed, location=(45.0, 7.0) if seed % 2 else None)
            _check(shim, msgs, loc, mk.run_reference(loc, msgs, mods), ("decode", seed))
    finally:
        import make_decode_golden as mdg
        mdg.unload_reference()
