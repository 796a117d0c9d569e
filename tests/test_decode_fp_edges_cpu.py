"""nl() of the batch decoder at every latitude where the decoder evaluates it.

The decoder never computes cpr.py:48-51's libm expression on the device: amb_nl() compares |lat| with a transition
table that amb_build_nl_table() bisects once on the host (gr_air_modes_b200/csrc/amb_decode_core.h). The two agree
wherever the expression is monotone in the last bit, and a latitude inside a window where it is not would get a
different zone count than the reference: another longitude, or a straddle where the reference has none.

nl() only ever sees the latitudes of the CPR lattices, d * (j + y / 2^17) with y = 0..2^17-1:
  * the global decode (amb_cpr_global): d = 360/60 and 360/59 with j = 0..59 / 0..58 and the "> 270 -> -360" shift;
    d = 90/60 and 90/59 for surface reports, as they are and with the -90 of a receiver south of the equator;
  * the local decode (amb_cpr_local): d = span / (60 - ctype) with j = floor(my_lat / d) + {-1, 0, 1}, so
    j = floor(-90 / d) - 1 .. floor(90 / d) + 1 for a reference latitude in [-90, 90].
At |lat| >= 87 both return 1 by rule (cpr.py:47), so the global decode's latitudes above 90 need no lattice of their
own. tests/decode_host_shim.cc walks each lattice in C with the decoder's own double expressions: about 9e7 latitudes,
each one compared with the direct formula; every one must agree. The table itself must be the formula's transitions
to the last bit, and CPython's nl() (oracle/decode_oracle.py) must equal the C formula at the lattice latitudes
nearest each transition.
"""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402

NL_MAX = 64


def _lattices():
    """(name, span, div, j_lo, j_hi, post) of every lattice the decoder evaluates nl() on."""
    out = []
    for div, fmt in ((60, "even"), (59, "odd")):
        out.append(("global airborne %s" % fmt, 360.0, div, 0, div - 1, 1))
        out.append(("global surface %s" % fmt, 90.0, div, 0, div - 1, 0))
        out.append(("global surface %s, receiver south" % fmt, 90.0, div, 0, div - 1, 2))
    for span, kind in ((360.0, "airborne"), (90.0, "surface")):
        for ctype in (0, 1):
            d = span / (60 - ctype)
            out.append(("local %s ctype %d" % (kind, ctype), span, 60 - ctype, math.floor(-90 / d) - 1,
                        math.floor(90 / d) + 1, 0))
    return out


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    lib = C.CDLL(emul_build.build(tmp_path_factory, os.path.join(emul_build.ROOT, "tests", "decode_host_shim.cc")))
    lib.shim_nl.restype = C.c_int
    lib.shim_nl.argtypes = [C.c_double]
    lib.shim_nl_table.restype = None
    lib.shim_nl_table.argtypes = [C.c_void_p]
    lib.shim_nl_lattice.restype = C.c_longlong
    lib.shim_nl_lattice.argtypes = [C.c_double, C.c_int, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p, C.c_int,
                                    C.POINTER(C.c_longlong), C.c_void_p]
    return lib


def _table(shim):
    T = np.zeros(NL_MAX)
    shim.shim_nl_table(C.c_void_p(T.ctypes.data))
    return T


def test_nl_table_is_the_formulas_transitions_to_the_last_bit(shim):
    """T[k] is the smallest double at which cpr.py's nl() drops below k, and the double just below it still gives k:
    a table entry one ulp off either way fails here."""
    from oracle import decode_oracle as do
    T = _table(shim)
    assert T[0] == 59
    for k in range(3, 60):
        below = float(np.nextafter(T[k], 0.0))
        assert do.nl(T[k]) == k - 1 and do.nl(below) == k, (k, T[k])
        assert shim.shim_nl(T[k]) == k - 1 and shim.shim_nl(below) == k, (k, T[k])


@pytest.mark.parametrize("name,span,div,j_lo,j_hi,post", _lattices(), ids=[x[0] for x in _lattices()])
def test_nl_at_every_lattice_latitude(shim, name, span, div, j_lo, j_hi, post):
    from oracle import decode_oracle as do
    bad = np.zeros(64)
    n_bad = C.c_longlong()
    near = np.full(2 * NL_MAX, np.nan)
    n = shim.shim_nl_lattice(span, div, j_lo, j_hi, post, C.c_void_p(bad.ctypes.data), len(bad), C.byref(n_bad),
                             C.c_void_p(near.ctypes.data))
    assert n == (j_hi - j_lo + 1) << 17
    T = _table(shim)
    gaps = [abs(abs(x) - T[k // 2]) / math.ulp(T[k // 2]) for k, x in enumerate(near) if k >= 6 and not math.isnan(x)]
    print("%s: %d latitudes checked, %d disagree; nearest to a transition: %.3g ulp" % (name, n, n_bad.value, min(gaps)))
    assert n_bad.value == 0, bad[:min(n_bad.value, len(bad))].tolist()
    # the lattice latitudes nearest each transition: CPython's nl() (the reference's expression) equals the C one there
    pts = [float(x) for x in near if not math.isnan(x)]
    assert len(pts) >= 2 * 57 - 2                  # both sides of every transition below 87 (a surface lattice reaches
    for x in pts:                                  # only its own span, so it may lack one side of one transition)
        assert int(do.nl(x)) == shim.shim_nl(x), x


def test_commb_ties_under_the_emulated_decoder(tmp_path_factory):
    """The Comm-B stage's kernel source under the SIMT emulator (tests/simt/decode_emul.cc) on every 7th velocity of
    commb_cases.tie_scene: RESOLVED as 5,0 exactly at 2 GS - speed = +-20 and not at +-22, and exactly on the near side
    of the 10 deg track rule; records equal to the checker fed with CPython's velocities (oracle/decode_oracle.py)."""
    import commb_cases as cc
    import commb_oracle as co
    import track_cases as tc
    from test_decode_fp_edges_gpu import cpython_velocities, tie_outcomes, with_val_of
    from gr_air_modes_b200 import decode
    e = emul_build.decode_emul(tmp_path_factory)
    msgs, cases = cc.tie_scene(every=7)
    frames = tc.frames_of(msgs, unqueued_every=0)
    out = {}
    for S in (0, 30):
        h = e.emul_new(17)
        recs = np.zeros(len(frames), dtype=decode.FIELDS_DTYPE)
        emul_build.opts(e, h, commb=S)
        assert e.emul_decode(h, C.c_void_p(frames.ctypes.data), len(frames), C.c_void_p(recs.ctypes.data)) == 0
        e.emul_free(h)
        out[S] = recs
    py, _ = cpython_velocities(msgs, out[0])
    co.assert_records_equal(out[30], with_val_of(co.replay(frames, py, 30), out[0]), "ties, CPython velocities")
    counts, bad = tie_outcomes(out[30], cases)
    print("Comm-B ties under the emulator: replies per case %s" % dict(sorted(counts.items(), key=str)))
    assert not bad, bad[:10]
    assert all(counts.get(("speed", x), 0) > 20 for x in (-22, -20, 20, 22))
