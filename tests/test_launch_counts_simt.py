"""amb_stats.kernel_launches is the number of kernels the library launched: for every entry point that launches, its
growth equals the growth of the SIMT emulator's own count of AMB_LAUNCH (simt_launch_count), with the library's
sources compiled for the host (tests/simt/library_emul.cc)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import gr_air_modes_b200 as am
from gr_air_modes_b200 import _lib, synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_build  # noqa: E402

RATE = 4e6


@pytest.fixture(scope="module")
def launches(tmp_path_factory):
    out = emul_build.build(tmp_path_factory, emul_build.LIBRARY_EMUL)
    saved = (_lib.LIB_PATH, _lib._lib)
    _lib.LIB_PATH, _lib._lib = out, None
    try:
        lib = C.CDLL(out)
        lib.simt_launch_count.restype = C.c_ulonglong
        yield lib.simt_launch_count
    finally:
        _lib.LIB_PATH, _lib._lib = saved


@pytest.fixture(scope="module")
def iq():
    return synth.make_scene(RATE, 24_000, 4, 17).iq


def counted(launches, ctx, fn):
    """(kernel_launches growth, AMB_LAUNCH growth) over fn(), with everything fn enqueued dispatched."""
    s0, c0 = ctx.stats().kernel_launches, launches()
    fn()
    s1 = ctx.stats().kernel_launches
    return s1 - s0, launches() - c0


def same(launches, ctx, fn, what):
    got, want = counted(launches, ctx, fn)
    assert want > 0 and got == want, (what, got, want)


@pytest.mark.parametrize("opts", [dict(resolver=0), dict(resolver=1), dict(ec=2), dict(ec_any=2), dict(ap_filter=10),
                                  dict(dcblock=True), dict(resolver=1, dcblock=True, ec=1)])
def test_process_counts_every_launch(launches, iq, opts):
    opts = dict(opts)
    dcblock = opts.pop("dcblock", False)
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True, use_dcblock=dcblock)
    for k, v in opts.items():
        rx.set_option(k, v)
    n = iq.size // 2
    same(launches, rx._ctx, lambda: rx.process(iq, flush=True), "one-shot")
    for chunks in ([5_000, 1, 511, 7_777, 513], [3, 17, 239]):       # ragged chunks, then tiny calls only
        rx.reset()
        rx._slicer._first = True

        def stream():
            pos = 0
            for c in chunks:
                rx.process(iq[2 * pos: 2 * (pos + c)])
                pos += c
            rx.process(iq[2 * pos: 2 * (pos + (n - pos if chunks[0] > 100 else 100))], flush=True)
        same(launches, rx._ctx, stream, chunks)
    rx.reset()
    same(launches, rx._ctx, lambda: rx.process(iq[:2 * 40], flush=True), "tiny flush")
    rx.close()


@pytest.mark.parametrize("resolver", [0, 1])
def test_time_shard_entry_points_count_every_launch(launches, iq, resolver):
    n = iq.size // 2
    rx = am.rx_path(RATE, 7.0, am.msg_queue(), use_pmf=True)
    rx.set_option("resolver", resolver)
    rx.defer_resolve(True)
    same(launches, rx._ctx, lambda: rx.seek(0, 0, (0, 0)), "seek")
    same(launches, rx._ctx, lambda: rx.process(iq[:2 * (n // 2)], collect=False), "deferred")
    same(launches, rx._ctx, lambda: rx.resolve(), "resolve")
    same(launches, rx._ctx, lambda: rx.resolve((0, 0)), "re-resolution")
    entry = np.zeros(2, np.int64)
    same(launches, rx._ctx, lambda: rx.resolve_device(entry.ctypes.data), "resolve_device")
    rx.drain()
    same(launches, rx._ctx, lambda: rx.seek(1000, 5000), "seek into the stream")
    same(launches, rx._ctx, lambda: rx.process(iq[2000: 2 * n], flush=True, collect=False), "deferred flush")
    same(launches, rx._ctx, lambda: rx.resolve((5000, 5000)), "resolve with an entry state")
    rx.drain()
    same(launches, rx._ctx, lambda: rx.seek(0, 0), "seek")
    same(launches, rx._ctx, lambda: rx.process(iq[:2 * 40], flush=True, collect=False), "deferred tiny flush")
    same(launches, rx._ctx, lambda: rx.resolve_device(entry.ctypes.data), "resolve_device of a tiny flush")
    rx.close()


@pytest.mark.parametrize("resolver", [0, 1])
def test_split_form_and_tools_count_every_launch(launches, port, iq, resolver):
    from oracle import cpu_oracle as co
    bb, avg = port.frontend(iq, RATE, True, co.MA_CANONICAL)
    pre = am.preamble(RATE, 7.0)
    pre._ctx.call("amb_set_option", b"resolver", resolver)
    out = []
    same(launches, pre._ctx, lambda: out.append(pre.process(bb[:9_000], avg[:9_000], flush=False)), "preamble")
    same(launches, pre._ctx, lambda: out.append(pre.process(bb[9_000:], avg[9_000:], flush=True)), "preamble flush")
    chips = np.concatenate([o[0] for o in out])
    assert chips.shape[0] > 0
    q = am.msg_queue()
    for ec in (0, 2):
        sl = am.slicer(q, ec=ec)
        same(launches, sl._ctx, lambda: sl.process(chips, [(0, 0.0)] * chips.shape[0]), ("slicer", ec))
    rx = am.rx_path(RATE, 7.0, q, use_pmf=True)
    for stage in ("m2", "bb", "avg", "dc"):
        same(launches, rx._ctx, lambda: rx.dump_stage(stage, iq[:4000]), stage)
    crc = (C.c_uint32 * 2)()
    same(launches, rx._ctx, lambda: rx._ctx.call("amb_device_crc", bytes.fromhex("8D4840D6202CC371C32CE0") * 2, 2, 11, crc),
         "crc")
    rx.close()
