"""amb_decoder_set_option through the C ABI of the emulated library (tests/simt/library_emul.cc): for each of the nine
decoder options, both bounds are taken and one value past each bound is refused with the option's own message; an
unknown name is refused with "amb_decoder_set_option: unknown option". This pins the option table's names, ranges and
messages."""
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402

AMB_OK, AMB_ERR_INVALID = 0, -1

# name, lowest and highest value taken, message for a value past either
OPTIONS = [
    ("local_cpr", 0, 600, "local_cpr: 0 (off) .. 600 seconds"),
    ("commb", 0, 600, "commb: 0 (off) .. 600 seconds"),
    ("opstatus", 0, 600, "opstatus: 0 (off) .. 600 seconds"),
    ("track", 0, 3600, "track: 0 (off) .. 3600 seconds"),
    ("track_ext", 0, 3600, "track_ext: 0 (off) .. 3600 seconds"),
    ("sbs1", 0, 1, "sbs1: 0 (off) or 1 (on)"),
    ("coverage", 0, 1, "coverage: 0 (off) or 1 (on)"),
    ("reports", 0, 1, "reports: 0 (off) or 1 (on)"),
    ("sbs1_tz", -720, 840, "sbs1_tz: -720 .. 840 minutes"),
]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    e = C.CDLL(emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL))
    e.amb_decoder_create.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.POINTER(C.c_void_p)]
    e.amb_decoder_destroy.argtypes = [C.c_void_p]
    e.amb_decoder_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    e.amb_decoder_last_error.argtypes = [C.c_void_p]
    e.amb_decoder_last_error.restype = C.c_char_p
    return e


@pytest.fixture(scope="module")
def decoder(lib):
    h = C.c_void_p()
    assert lib.amb_decoder_create(0, 0, 0.0, 0.0, C.byref(h)) == AMB_OK
    yield h
    lib.amb_decoder_destroy(h)


@pytest.mark.parametrize("name,lo,hi,message", OPTIONS, ids=[o[0] for o in OPTIONS])
def test_bounds_taken_and_values_past_them_refused(lib, decoder, name, lo, hi, message):
    for bad in (lo - 1, hi + 1):
        assert lib.amb_decoder_set_option(decoder, b"nope", 0) == AMB_ERR_INVALID     # another message before
        assert lib.amb_decoder_set_option(decoder, name.encode(), bad) == AMB_ERR_INVALID
        assert lib.amb_decoder_last_error(decoder).decode() == message
    for ok in (lo, hi, lo):
        assert lib.amb_decoder_set_option(decoder, name.encode(), ok) == AMB_OK


def test_unknown_and_missing_names_refused(lib, decoder):
    for name in (b"nope", b"", b"sbs1 ", b"Track", b"seconds"):
        assert lib.amb_decoder_set_option(decoder, name, 0) == AMB_ERR_INVALID
        assert lib.amb_decoder_last_error(decoder).decode() == "amb_decoder_set_option: unknown option"
    assert lib.amb_decoder_set_option(decoder, None, 0) == AMB_ERR_INVALID
    assert lib.amb_decoder_set_option(None, b"track", 0) == AMB_ERR_INVALID
