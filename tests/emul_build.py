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


def opts(e, h, loc=None, **stages):
    """Set every option of the harness's decoder `h` (e: the bound harness), as amb_decoder_set_location and
    amb_decoder_set_option would: the receiver at loc = (lat, lon) (None: no location), the options named in `stages` to
    their values (e.g. commb=30, coverage=1) and every other option of decode.OPTIONS to 0."""
    from gr_air_modes_b200 import decode
    assert set(stages) <= set(decode.OPTIONS), stages
    e.emul_set_location(h, *((0, 0.0, 0.0) if loc is None else (1, loc[0], loc[1])))
    for name in decode.OPTIONS:
        assert e.emul_set_option(h, name.encode(), int(stages.get(name, 0))) == 0, name


def decode_emul(tmp_path_factory, src=DECODE_EMUL):
    """The decoder harness tests/simt/decode_emul.cc (or a patched copy at `src`), built and bound."""
    e = C.CDLL(build(tmp_path_factory, src))
    e.emul_new.restype = C.c_void_p
    e.emul_new.argtypes = [C.c_int]
    e.emul_free.argtypes = [C.c_void_p]
    e.emul_reset.argtypes = [C.c_void_p]
    e.emul_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    e.emul_set_location.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double]
    e.emul_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    e.emul_snapshot.argtypes = [C.c_void_p, C.c_double, C.c_uint, C.c_void_p, C.c_void_p, C.c_int]
    e.emul_text.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    e.emul_sbs1_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    e.emul_coverage.argtypes = [C.c_void_p, C.c_void_p]
    e.emul_coverage_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    e.emul_reports_state.argtypes = [C.c_void_p]
    e.simt_launch_count.restype = C.c_ulonglong
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
