"""In-tree build of libairmodes_b200.so (nvcc, sm_90a only). Cross-compiles without a GPU."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libairmodes_b200.so")
SOURCES = ["amb_kernels.cu", "amb_api.cu", "amb_decode.cu"]
HEADERS = ["amb_internal.h", "amb_launch.h", "amb_params.h", "amb_decode_core.h", "amb_decode_kernels.cuh", "amb_decode_v3.cuh", "amb_decode_local.cuh", "amb_decode_commb.cuh", "amb_decode_track.cuh", "amb_order_kernels.cuh", os.path.join("..", "..", "include", "airmodes_b200.h")]
# amb_decode.cu follows cpr.py operation by operation in IEEE double: no fused multiply-add contraction there
EXTRA_FLAGS = {"amb_decode.cu": ["-fmad=false"]}
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--compiler-options", "-fPIC,-fvisibility=hidden", "-Xcompiler", "-Wall"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libairmodes_b200.so cannot be built")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build_native(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    env = dict(os.environ)
    host = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc, "-ccbin", host, *NVCC_FLAGS, *EXTRA_FLAGS.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((cmd, subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s" % (" ".join(cmd), out.decode()))
        if verbose:
            print(out.decode())
    cmd = [nvcc, "-ccbin", host, "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB, *objs, "-cudart", "shared"]
    subprocess.run(cmd, check=True, env=env)
    return LIB


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))


def build_c_example(force: bool = False) -> str:
    """Compile examples/modes_rx_c.c against the C ABI with plain gcc (proves the boundary has no C++/torch types)."""
    root = os.path.dirname(HERE)
    src = os.path.join(root, "examples", "modes_rx_c.c")
    out = os.path.join(root, "examples", "modes_rx_c")
    if not force and os.path.exists(out) and os.path.getmtime(out) > max(os.path.getmtime(src), os.path.getmtime(LIB)):
        return out
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.run([cc, "-std=c99", "-O2", "-Wall", "-I" + os.path.join(root, "include"), src, "-L" + HERE,
                    "-lairmodes_b200", "-Wl,-rpath," + HERE, "-o", out], check=True)
    return out
