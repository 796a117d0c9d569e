"""The one g++ recipe of the CPU test tier: the emulated library (tests/simt/library_emul.cc), the kernel harnesses under
tests/simt and the host shims of the decode core, each compiled once per pytest session."""
import ctypes as C
import hashlib
import os
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


def decode_emul(tmp_path_factory, src=DECODE_EMUL):
    """The decoder harness tests/simt/decode_emul.cc (or a patched copy at `src`), built and bound."""
    e = C.CDLL(build(tmp_path_factory, src))
    e.emul_new.restype = C.c_void_p
    e.emul_new.argtypes = [C.c_int]
    e.emul_free.argtypes = [C.c_void_p]
    e.emul_reset.argtypes = [C.c_void_p]
    e.emul_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int,
                              C.c_void_p]
    e.emul_snapshot.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_uint, C.c_void_p, C.c_int]
    return e
