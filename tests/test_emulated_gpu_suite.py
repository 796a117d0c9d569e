"""Runs the GPU parity tests themselves - tests/test_gpu_parity.py, tests/test_decision_edges_gpu.py and
tests/test_zz_decode_gpu.py, unchanged, at their real sizes (up to 4 M samples per scene, the 16.7 M-sample gap of the
float-rounding test, dense traffic, time-sharding with cuts inside packets, DC blocker bit-exactness, every kernel
instantiation at threshold knife edges ...) - on the CPU box against the EMULATED build of the library
(tests/simt/library_emul.cc: the library's own sources on a SIMT emulator, see tests/test_library_simt.py), in a child
pytest spread over a few worker processes. What cannot run there is excluded by name: the 2^28-sample property test
and the 60 M-sample configs[0] scene (hours of emulation), tests that start other processes which load the real
library (CLI, C example, stress tool), and the threaded speculative-resolution test (one emulated device, not
thread-safe; tests/test_library_simt.py has its sequential form).

This is the CPU tier's rehearsal of the GPU tier, not a substitute: `pytest -m gpu` still has to run on an H100.
"""
import os
import subprocess
import sys

import emul_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXCLUDE = ("full_size or config0 or c_abi_example or cli_ or randomised_stress or time_sharded_speculative or "
           "host_ingest_paths or sc16_input or torch_input or device_resident_decode or device_side_drain or "
           "without_leaving_the_device")   # the last six need pinned / CUDA tensors; test_library_simt.py has their emulated twins


def test_gpu_parity_tests_pass_against_the_emulated_library(tmp_path_factory):
    lib = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    env = dict(os.environ, AMB_TEST_EMULATED_LIB=lib)
    workers = str(max(1, min(6, (os.cpu_count() or 2) - 1)))
    cmd = [sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_parity.py"),
           os.path.join(ROOT, "tests", "test_decision_edges_gpu.py"),
           os.path.join(ROOT, "tests", "test_zz_decode_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
           "-n", workers, "-k", "not (%s)" % EXCLUDE]
    out = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    tail = "\n".join(out.stdout.splitlines()[-25:])
    assert out.returncode == 0, tail + "\n" + out.stderr[-2000:]
    assert " passed" in tail and "failed" not in tail, tail
    passed = int(tail.split(" passed")[0].split()[-1])
    assert passed >= 138, tail
