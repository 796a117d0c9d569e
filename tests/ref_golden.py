"""What the unmodified reference returned for every call the tests make of it, so that the comparisons with the
reference run where its sources are absent: its C++ objects (oracle/_ref) in tests/golden/ref_calls.json.gz, its
Python modules in tests/golden/ref_python.json.gz.

The `ref` and `ref_py` fixtures (tests/conftest.py) answer from these records. With AMB_RECORD_REF=1 they call the
live reference instead and rewrite the records at the end of the session (the C++ objects must have been built into
oracle/_ref, the Python modules are read from AMB_REFERENCE_TREE, default /root/reference):

    AMB_RECORD_REF=1 python -m pytest tests -m "not gpu" -p no:xdist
    AMB_RECORD_REF=1 python -m pytest tests/test_gpu_parity.py -k live_reference      (no GPU needed for the record)

A call whose input is not in the record fails: the test's inputs changed and the record must be made again.
"""
from __future__ import annotations

import gzip
import hashlib
import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_calls.json.gz")


class RecordedChips:
    """The 240-chip packets of a recorded call, kept as their digest (chips_sha256)."""

    def __init__(self, sha256: str, n: int):
        self.sha256, self.n = sha256, n

    def __len__(self):
        return self.n


def chips_sha256(chips) -> str:
    """sha256 of float32 packets with every NaN made the same NaN (the equal_nan comparison, as a digest)."""
    if isinstance(chips, RecordedChips):
        return chips.sha256
    a = np.ascontiguousarray(chips, dtype=np.float32)
    a = np.where(np.isnan(a), np.float32(np.nan), a).astype(np.float32)
    return hashlib.sha256(a.tobytes()).hexdigest()


def same_chips(a, b) -> bool:
    return chips_sha256(a) == chips_sha256(b)


def _key(name, *args) -> str:
    h = hashlib.sha256(name.encode())
    for x in args:
        if isinstance(x, np.ndarray):
            h.update(str((x.dtype.str, x.shape)).encode())
            h.update(np.ascontiguousarray(x).tobytes())
        else:
            h.update(repr(x).encode())
        h.update(b"|")
    return h.hexdigest()


def _result_to_json(r) -> dict:
    return {"index": [int(x) for x in r.index], "secs": [int(x) for x in r.secs],
            "frac": [float(x).hex() for x in r.frac], "chips_sha256": chips_sha256(r.chips), "msgs": list(r.msgs),
            "calls": int(r.calls)}


def _result_from_json(d):
    from oracle.cpu_oracle import Result
    return Result(np.array(d["index"], np.uint64), np.array(d["secs"], np.uint64),
                  np.array([float.fromhex(x) for x in d["frac"]], np.float64),
                  RecordedChips(d["chips_sha256"], len(d["index"])), list(d["msgs"]), None, d["calls"])


def _args(name, a):
    """Canonical arguments of one call, as the reference sees them."""
    if name in ("run_streams",):
        bb, avg, rate, thr, slice_, start = a
        bb = np.ascontiguousarray(bb, np.float32)
        return (bb, np.ascontiguousarray(avg, np.float32), float(rate), float(thr), bool(slice_),
                None if start is None else (int(start[0]), float(start[1])))
    if name == "run_slicer":
        chips, secs, frac = a
        return (np.ascontiguousarray(chips, np.float32), np.ascontiguousarray(secs, np.uint64),
                np.ascontiguousarray(frac, np.float64))
    if name == "crc24":
        return (bytes(a[0]),)
    return tuple(float(x) for x in a)          # preamble_params(rate, threshold_db)


class GoldenRef:
    """Same methods as oracle.cpu_oracle.Ref; answers from the record, or (live=Ref()) calls it and records."""

    def __init__(self, live=None):
        self.live = live
        self.table = {}
        if live is None:
            with gzip.open(PATH, "rt") as f:
                self.table = json.load(f)

    def _call(self, name, *a):
        key = _key(name, *_args(name, a))
        if self.live is None:
            if key not in self.table:
                raise KeyError("no recorded reference result for this %s call: remake %s (see tests/ref_golden.py)"
                               % (name, os.path.relpath(PATH)))
            return self._decode(name, self.table[key])
        if name in ("run_streams",):
            bb, avg, rate, thr, slice_, start = a
            r = self.live.run_streams(bb, avg, rate, thr, slice_=slice_, start_time=start)
        else:
            r = getattr(self.live, name)(*a)
        self.table[key] = self._encode(name, r)
        return self._decode(name, self.table[key]) if name in ("run_streams", "run_slicer") else r

    @staticmethod
    def _encode(name, r):
        if name in ("run_streams", "run_slicer"):
            return _result_to_json(r)
        return list(r) if isinstance(r, tuple) else r

    @staticmethod
    def _decode(name, d):
        if name in ("run_streams", "run_slicer"):
            return _result_from_json(d)
        return tuple(d) if isinstance(d, list) else d

    def crc24(self, data: bytes) -> int:
        return self._call("crc24", data)

    def preamble_params(self, rate, threshold_db):
        return self._call("preamble_params", rate, threshold_db)

    def run_streams(self, bb, avg, rate, threshold_db, slice_=True, start_time=None):
        return self._call("run_streams", bb, avg, rate, threshold_db, slice_, start_time)

    def run_slicer(self, chips, secs, frac):
        return self._call("run_slicer", chips, secs, frac)

    def save(self, merge=True):
        """Write the record (merged into the existing one, so that separate sessions can add to it)."""
        table = {}
        if merge and os.path.exists(PATH):
            with gzip.open(PATH, "rt") as f:
                table = json.load(f)
        table.update(self.table)
        with gzip.GzipFile(PATH, "wb", mtime=0) as f:
            f.write(json.dumps(table, sort_keys=True, separators=(",", ":")).encode())


PY_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_python.json.gz")


def _plain(o):
    """JSON-safe copy: tuples as lists, NaN / Inf as None (as tests/golden/make_decode_golden.py stores them)."""
    if isinstance(o, float) and (o != o or o in (float("inf"), float("-inf"))):
        return None
    if isinstance(o, dict):
        return {k: _plain(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return [_plain(v) for v in o]
    if isinstance(o, np.integer):
        return int(o)
    if isinstance(o, np.floating):
        return _plain(float(o))
    return o


class PythonRecord:
    """What the reference's unmodified Python modules (parse.py, altitude.py, cpr.py, msprint.py) returned for the
    tests' inputs, stored in tests/golden/ref_python.json.gz. get(name, inputs, compute) answers from the record; with
    live=True (AMB_RECORD_REF=1) it runs compute() - which loads the reference modules - and records the answer. Either
    way the answer is the stored JSON form, so both modes compare the same values. The key includes a digest of the
    inputs, so a test whose inputs changed fails instead of comparing against a stale answer."""

    def __init__(self, live=False):
        self.live = live
        self.table = {}
        if not live:
            with gzip.open(PY_PATH, "rt") as f:
                self.table = json.load(f)

    def get(self, name, inputs, compute):
        key = name + "/" + hashlib.sha256(json.dumps(_plain(inputs), sort_keys=True).encode()).hexdigest()[:16]
        if self.live:
            self.table[key] = json.loads(json.dumps(_plain(compute())))
        elif key not in self.table:
            raise KeyError("no recorded reference answer for %s with these inputs: remake %s (see tests/ref_golden.py)"
                           % (name, os.path.relpath(PY_PATH)))
        return self.table[key]

    def save(self):
        table = {}
        if os.path.exists(PY_PATH):
            with gzip.open(PY_PATH, "rt") as f:
                table = json.load(f)
        table.update(self.table)
        with gzip.GzipFile(PY_PATH, "wb", mtime=0) as f:
            f.write(json.dumps(table, sort_keys=True, separators=(",", ":")).encode())
