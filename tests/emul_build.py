"""The one g++ recipe of the CPU test tier: the emulated library (tests/simt/library_emul.cc), the kernel harnesses under
tests/simt and the host shims of the decode core, each compiled once per pytest session."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY_EMUL = os.path.join(ROOT, "tests", "simt", "library_emul.cc")
DECODE_EMUL = os.path.join(ROOT, "tests", "simt", "decode_emul.cc")

# -U_FORTIFY_SOURCE: the SIMT emulator's fibers switch stacks with _longjmp, which the fortified longjmp refuses.
# -ffp-contract=off: no fused multiply-add, as nvcc -fmad=false builds the decoder; the shims' arithmetic must match it.
FLAGS = ["-std=c++17", "-O1", "-U_FORTIFY_SOURCE", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-psabi", "-shared",
         "-fPIC"]

_built = {}


def build(tmp_path_factory, src) -> str:
    """Compile the C++ file `src` into a shared library under the session's base temp directory, once per session and
    source path (so that a patched copy of a source builds on its own); returns the library's path."""
    src = os.path.abspath(str(src))
    if src not in _built:
        name = "%s_%s.so" % (os.path.splitext(os.path.basename(src))[0], hashlib.sha1(src.encode()).hexdigest()[:12])
        out = str(tmp_path_factory.getbasetemp() / name)
        subprocess.run(["g++"] + FLAGS + ["-o", out, src], check=True)
        _built[src] = out
    return _built[src]


class EmulOpts(C.Structure):
    """The options of one emulated decode (struct EmulOpts of tests/simt/decode_emul.cc): the receiver location and
    every stage's S, 0 = off."""
    _fields_ = [("have_loc", C.c_int), ("lat", C.c_double), ("lon", C.c_double), ("local_cpr", C.c_int),
                ("commb", C.c_int), ("opstatus", C.c_int), ("track", C.c_int), ("track_ext", C.c_int), ("sbs1", C.c_int),
                ("sbs1_tz", C.c_int)]


def opts(loc=None, **stages):
    """EmulOpts with the receiver at loc = (lat, lon) (None: no location) and the given stages on, e.g. commb=30."""
    return EmulOpts(0, 0.0, 0.0, **stages) if loc is None else EmulOpts(1, loc[0], loc[1], **stages)


def decode_emul(tmp_path_factory, src=DECODE_EMUL):
    """The decoder harness tests/simt/decode_emul.cc (or a patched copy at `src`), built and bound."""
    e = C.CDLL(build(tmp_path_factory, src))
    e.emul_new.restype = C.c_void_p
    e.emul_new.argtypes = [C.c_int]
    e.emul_free.argtypes = [C.c_void_p]
    e.emul_reset.argtypes = [C.c_void_p]
    e.emul_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(EmulOpts), C.c_void_p]
    e.emul_snapshot.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_int]
    e.emul_sbs1_text.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    e.emul_sbs1_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return e


def mutant(tmp_path, tmp_path_factory, rel, old, new):
    """The harness built from a copy of the sources under tmp_path in which the text `old`, which must occur exactly
    once in the file `rel` (relative to the repository), reads `new`. old and new may also be tuples of such texts,
    patched in turn."""
    for sub in ("gr_air_modes_b200/csrc", "include", "tests/simt"):
        shutil.copytree(os.path.join(ROOT, sub), str(tmp_path / sub))
    p = tmp_path / rel
    src = p.read_text()
    for a, b in zip(*((old, new) if isinstance(old, tuple) else ((old,), (new,)))):
        assert src.count(a) == 1, a
        src = src.replace(a, b)
    p.write_text(src)
    return decode_emul(tmp_path_factory, tmp_path / "tests/simt/decode_emul.cc")
