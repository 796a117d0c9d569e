"""Shared by the text-report tests (decoder option reports): the slicer's message text of a frame, as
amb_format_message writes it, and the report lines report.py forms from that text and the frame's record."""
import numpy as np


def slicer_text(frame, first: bool) -> str:
    """slicer_impl.cc:186-192 for one frame (a FRAME_DTYPE record or a ctypes Frame): hex payload, "%06x" crc,
    "%.*g" of the float32 level (precision 6 for the stream's first message, 10 after), secs, "%.10g" of frac."""
    nbits, data = int(frame["nbits"] if isinstance(frame, np.void) else frame.nbits), \
        bytes(frame["data"] if isinstance(frame, np.void) else frame.data)
    crc = int(frame["crc"] if isinstance(frame, np.void) else frame.crc)
    lev = float(np.float32(frame["ref_level"] if isinstance(frame, np.void) else frame.ref_level))
    secs = int(frame["secs"] if isinstance(frame, np.void) else frame.secs)
    frac = float(frame["frac"] if isinstance(frame, np.void) else frame.frac)
    return "%s %06x %.*g %d %.10g" % (data[: min(nbits // 8, 14)].hex(), crc, 6 if first else 10, lev, secs, frac)


def expected_text(frames, records, first: bool = True) -> bytes:
    """What the option writes for one call: report.format_report(text, record) + "\\n" for every queued frame, the
    first queued frame at precision 6 when `first`."""
    from gr_air_modes_b200 import decode, report
    out = []
    for f, r in zip(frames, records):
        if int(r["status"]) & decode.FS_NOT_QUEUED:
            continue
        line = report.format_report(slicer_text(f, first), r)
        first = False
        if line is not None:
            out.append(line + "\n")
    return "".join(out).encode("latin-1")


def frames_with_levels(arr, n, seed):
    """The frames of a ctypes Frame array as a FRAME_DTYPE array, with float32 levels spread over the receiver's range
    (1e-9 .. 10, a few exact powers of ten) and the stamps kept."""
    from gr_air_modes_b200 import decode
    a = np.frombuffer(bytes(arr), dtype=decode.FRAME_DTYPE, count=n).copy()
    rng = np.random.default_rng(seed)
    lev = (10.0 ** rng.uniform(-9, 1, n)).astype(np.float32)
    lev[rng.random(n) < 0.05] = np.float32(0.001)
    a["ref_level"] = lev
    return a


def text_option_scenes(small=False):
    """(name, frames, stages) of the scenes that exercise the lines options commb and opstatus write: every scene of
    tests/opstatus_cases.py with opstatus = its S, every scene of tests/commb_cases.py with commb = its S. small: only
    the frames whose position squitters' addresses fit the SIMT harness's pairing table (below 2^15)."""
    import commb_cases as cc
    import opstatus_cases as oc
    import track_cases as tc
    for prefix, scenes, option in (("opstatus", oc.scenes(), "opstatus"), ("commb", cc.scenes(), "commb")):
        for name, msgs, S in scenes:
            fr = tc.frames_of(msgs)
            if small:
                icao = np.array([int.from_bytes(bytes(f["data"][1:4]), "big") for f in fr])
                fr = np.ascontiguousarray(fr[(fr["df"] != 17) | (icao < (1 << 15))])
            yield "%s_%s" % (prefix, name), fr, {option: S}


# every kind of line the options commb and opstatus add, and every optional part of a target-state line
OPTION_LINE_KINDS = {"BDS4,0", "BDS5,0", "BDS6,0", "BDS6,5 airborne v0", "BDS6,5 airborne v1+", "BDS6,5 surface v0",
                     "BDS6,5 surface v1+", "BDS6,2 +alt", "BDS6,2 -alt", "BDS6,2 +baro", "BDS6,2 -baro",
                     "BDS6,2 +heading", "BDS6,2 -heading", "BDS6,2 +modes", "BDS6,2 -modes"}


def line_kinds(text: bytes) -> set:
    """The OPTION_LINE_KINDS present in a call's text."""
    out = set()
    for line in text.decode("latin-1").splitlines():
        body = line.split(") ", 1)[1]
        for reg in ("BDS4,0", "BDS5,0", "BDS6,0"):
            if body.startswith("Type 2") and (" %s " % reg) in body:
                out.add(reg)
        if "BDS6,5 (operational status)" in body:
            out.add("BDS6,5 %s %s" % ("surface" if " surface " in body else "airborne",
                                       "v0" if " version 0 " in body else "v1+"))
        if "BDS6,2 (target state)" in body:
            for part, key in ((" selected alt ", "alt"), (" baro ", "baro"), (" heading ", "heading"),
                              (" modes ", "modes")):
                out.add("BDS6,2 %s%s" % ("+" if part in body else "-", key))
    return out
