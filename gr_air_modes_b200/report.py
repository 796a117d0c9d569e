"""Text reports in the format of the reference's stdout printer, from GPU-decoded records.

    air_modes.output_print(cpr_dec, publisher)      python/msprint.py:30-260   (what apps/modes_rx prints by default)

The reference formats one line per parsed message inside its pubsub handlers; here the numbers come from
`decode.batch_decoder` (struct amb_fields) and only the string formatting happens on the host - line for line the
reference's, including its quirks: no line for DF4/5/20/21 replies whose flight status is 0, 6 or 7 (fs_text raises,
msprint.py:86-98), no line for DF0 with ri in (1, 5, 6, 7, 8) (:76-77), no DF16 line (printTCAS asks for a field DF16
does not have, :196-199, and make_parser swallows the ADSBError, parse.py:426-434), BDS6,1 printed as "FTC=28 not
implemented" (:163-167), and the DF21 squawk printed with %x (:257).
"""
from __future__ import annotations

import math

from . import decode as _d

_CATEGORIES = [["NO INFO", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED"],
               ["NO INFO", "SURFACE EMERGENCY VEHICLE", "SURFACE SERVICE VEHICLE", "FIXED OBSTRUCTION", "CLUSTER OBSTRUCTION",
                "LINE OBSTRUCTION", "RESERVED"],
               ["NO INFO", "GLIDER", "BALLOON/BLIMP", "PARACHUTE", "ULTRALIGHT", "RESERVED", "UAV", "SPACECRAFT"],
               ["NO INFO", "LIGHT", "SMALL", "LARGE", "LARGE HIGH VORTEX", "HEAVY", "HIGH PERFORMANCE", "ROTORCRAFT"]]   # parse.py:263-266
_ARA = ["CLIMB", "DON'T DESCEND", "DON'T DESCEND >500FPM", "DON'T DESCEND >1000FPM", "DON'T DESCEND >2000FPM", "DESCEND",
        "DON'T CLIMB", "DON'T CLIMB >500FPM", "DON'T CLIMB >1000FPM", "DON'T CLIMB >2000FPM", "TURN LEFT", "TURN RIGHT",
        "DON'T TURN LEFT", "DON'T TURN RIGHT"]                                      # parse.py:382-385, bits 41..54
_RAC = ["DON'T DESCEND", "DON'T CLIMB", "DON'T TURN LEFT", "DON'T TURN RIGHT"]      # parse.py:386, bits 55..58
_HANDLED = (0, 4, 5, 11, 16, 17, 20, 21)                                            # msprint.py:35 "handle%i"


def _fs_text(fs):                                   # msprint.py:86-98
    return {1: " (aircraft is on the ground)", 2: " (AIRBORNE ALERT)", 3: " (GROUND ALERT)", 4: " (SPI ALERT)",
            5: " (SPI)"}.get(fs)


def _resolutions(ara, rac):                         # parse.py:380-397
    res = "".join(" " + t for k, t in enumerate(_ARA) if ara & (1 << (13 - k)))
    comp = "".join(" " + t for k, t in enumerate(_RAC) if rac & (1 << (3 - k)))
    return res, comp


def prefix(reference: float, secs: int, frac: float) -> str:
    """output_print.prefix (msprint.py:44-46) with rssi and stamp as make_parser builds them (parse.py:427-430)."""
    rssi = 10.0 * math.log10(max(1e-8, float(reference)))
    secs, frac = int(secs), float(frac)
    secs += int(frac)                               # modes_types.stamp.__init__ (modes_types.py:29-33)
    frac -= int(frac)
    return "(%i %.8f) " % (rssi, secs + frac)


# Comm-B inference (decoder option commb): per register, its title and (name, format) of the fields that are present
_COMMB_TEXT = {
    0x40: ("BDS4,0 selected vertical intention", (("mcp_alt", "MCP alt %ift"), ("fms_alt", "FMS alt %ift"),
                                                  ("baro", "baro %.1fmb"), ("modes", "modes %i"),
                                                  ("alt_source", "alt source %i"))),
    0x50: ("BDS5,0 track and turn report", (("roll", "roll %.1f"), ("track", "track %.1f"), ("gs", "GS %ikt"),
                                            ("track_rate", "track rate %.2f"), ("tas", "TAS %ikt"))),
    0x60: ("BDS6,0 heading and speed report", (("heading", "heading %.1f"), ("ias", "IAS %ikt"), ("mach", "Mach %.3f"),
                                               ("baro_rate", "baro rate %ift/min"),
                                               ("inertial_rate", "inertial rate %ift/min"))),
}


def _commb_text(df, ecc, v):
    title, fields = _COMMB_TEXT[v["bds"]]
    parts = [fmt % v[name] for name, fmt in fields if v[name] is not None]
    return "Type %i %s from %x: %s" % (df, title, ecc, " ".join(parts))


def _opstatus_text(icao, v):
    """Decoder option opstatus: one line for a decoded TC 31 (BDS6,5) or TC 29 subtype 1 (BDS6,2) squitter."""
    if v["kind"] == "opstatus":
        out = "Type 17 BDS6,5 (operational status) from %x version %i %s capability %04x mode %04x" % (
            icao, v["version"], "surface" if v["subtype"] else "airborne", v["capability"], v["op_mode"])
        if v["version"]:
            out += " NIC-A %i NACp %i SIL %i" % (v["nic_a"], v["nacp"], v["sil"])
            if v["subtype"]:
                out += " NIC-C %i TRK/HDG %i L/W %i" % (v["nic_c"], v["trk_hdg"], v["length_width"])
            else:
                out += " GVA %i NICbaro %i" % (v["gva"], v["nic_baro"])
            out += " HRD %i SIL supp %i" % (v["hrd"], v["sil_supplement"])
        return out
    out = "Type 17 BDS6,2 (target state) from %x" % icao
    if v["selected_alt"] is not None:
        out += " selected alt %ift (%s)" % (v["selected_alt"], v["alt_source"])
    if v["baro"] is not None:
        out += " baro %.1fmb" % v["baro"]
    if v["heading"] is not None:
        out += " heading %.1f" % v["heading"]
    modes = [name for name, key in (("AP", "autopilot"), ("VNAV", "vnav"), ("ALT", "alt_hold"), ("APP", "approach"),
                                    ("LNAV", "lnav"), ("TCAS", "tcas")) if v[key]]
    if modes:
        out += " modes " + " ".join(modes)
    return out + " NACp %i NICbaro %i SIL %i" % (v["nacp"], v["nic_baro"], v["sil"])


def format_report(message: str, r) -> str | None:
    """One slicer message string + its decoded record -> the line output_print would print, or None where the
    reference prints nothing. `r`: a FIELDS_DTYPE record or the dict from decode.record_to_dict()."""
    if not isinstance(r, dict):
        r = _d.record_to_dict(r)
    _, _, ref, secs, frac = message.split()
    st, df, ecc = r["status"], r["df"], r["ecc"]
    if st == _d.FS_NO_HANDLER and df in (20, 21):
        v = _d.commb_values(r)                      # decoder option commb: an inferred BDS 4,0 / 5,0 / 6,0 register
        if v is not None:
            return prefix(float(ref), int(secs), float(frac)) + _commb_text(df, ecc, v)
    if st == _d.FS_NO_HANDLER and df == 17:
        v = _d.opstatus_values(r)                   # decoder option opstatus: a decoded TC 31 / TC 29 squitter
        if v is not None:
            return prefix(float(ref), int(secs), float(frac)) + _opstatus_text(r["icao"], v)
    if st & (_d.FS_NO_HANDLER | _d.FS_NOT_QUEUED):
        return None                                 # the parser raised: nothing is published (parse.py:431-434)
    out = prefix(float(ref), int(secs), float(frac))
    if df not in _HANDLED:                          # catch_nohandler (msprint.py:54-62); only DF24 gets this far
        return out + "No handler for message type %i from %.6x" % (df, ecc)
    metric = bool(st & _d.FS_METRIC_ALT)
    if df == 0:                                     # handle0 (msprint.py:64-84)
        if metric:
            return None
        out += "Type 0 (short A-A surveillance) from %x at %ift" % (ecc, r["altitude"])
        ri = r["ri"]
        if ri == 0:
            out += " (No TCAS)"
        elif ri == 2:
            out += " (TCAS resolution inhibited)"
        elif ri == 3:
            out += " (Vertical TCAS resolution only)"
        elif ri == 4:
            out += " (Full TCAS resolution)"
        elif ri == 9:
            out += " (speed <75kt)"
        elif ri > 9:
            out += " (speed %i-%ikt)" % (75 * (1 << (ri - 10)), 75 * (1 << (ri - 9)))
        else:
            return None
        if r["vs"] == 1:
            out += " (aircraft is on the ground)"
        return out
    if df == 4:                                     # handle4 (:100-107)
        if metric or _fs_text(r["fs"]) is None:
            return None
        return out + "Type 4 (short surveillance altitude reply) from %x at %ift" % (ecc, r["altitude"]) + _fs_text(r["fs"])
    if df == 5:                                     # handle5 (:109-116)
        if _fs_text(r["fs"]) is None:
            return None
        return out + "Type 5 (short surveillance ident reply) from %x with ident %i" % (ecc, r["squawk"]) + _fs_text(r["fs"])
    if df == 11:                                    # handle11 (:118-124)
        return out + "Type 11 (all call reply) from %x in reply to interrogator %i with capability level %i" % (
            r["icao"], ecc & 0xF, r["ca"] + 1)
    if df == 17:                                    # handle17 (:127-172)
        icao, bds = r["icao"], r["bds"]
        if bds == 0x08:
            row = _CATEGORIES[r["ftc"] - 1]
            if r["cat"] >= len(row):
                return None                         # the reference dies with an IndexError here (parse.py:268)
            return out + "Type 17 BDS0,8 (ident) from %x type %s ident %s" % (icao, row[r["cat"]], r["ident"])
        if bds in (0x05, 0x06):
            if not (st & _d.FS_HAS_POS):
                return None                         # CPRNoPositionError / CPRBoundaryStraddleError (:170-171)
            if bds == 0x06:
                out += "Type 17 BDS0,6 (surface report) from %x at (%.6f, %.6f) ground track %i" % (icao, r["lat"], r["lon"], r["val"][0])
                if st & _d.FS_HAS_RANGE:
                    out += " (%.2f @ %.0f)" % (r["range"], r["bearing"])
                return out
            out += "Type 17 BDS0,5 (position report) from %x at (%.6f, %.6f)" % (icao, r["lat"], r["lon"])
            if st & _d.FS_HAS_RANGE:
                out += " (" + "%.2f" % r["range"] + " @ " + "%.0f" % r["bearing"] + ")"
            return out + " at " + str(r["altitude"]) + "ft"
        if bds == 0x09:
            sub, v = r["subtype"], r["val"]
            if sub == 0:
                return out + "Type 17 BDS0,9-%i (track report) from %x with velocity %.0fkt heading %.0f VS %.0f turn rate %.0f" % (
                    sub, icao, v[0], v[1], v[2], v[3])
            if sub == 1:
                return out + "Type 17 BDS0,9-%i (track report) from %x with velocity %.0fkt heading %.0f VS %.0f" % (sub, icao, v[0], v[1], v[2])
            return out + ("Type 17 BDS0,9-%i (air course report) from %x with %s %.0fkt magnetic heading %.0f VS %.0f geo. diff. "
                          "from baro. alt. %.0fft") % (sub, icao, "TAS" if r["ast"] == 1 else "IAS", v[1], v[0], v[2], v[3])
        return out + "Type 17 with FTC=%i from %x not implemented" % (r["ftc"], icao)
    if df == 16:
        return None                                 # printTCAS reads msg.data["vds1"]: FieldNotInPacket, swallowed (see module doc)
    # DF20 / DF21: printTCAS (:174-258)
    bds1 = r["bds"]
    if bds1 == 0:
        out += "No handler in type %i for BDS1 == 0 from %x" % (df, ecc)
    elif bds1 == 1:
        a = r["aux"]
        out += "Type %i link capability report from %x: ACS: 0x%x, BCS: 0x%x, ECS: 0x%x, continues %i" % (df, ecc, a[0], a[1], a[2], a[3])
    elif bds1 == 2:
        out += "Type %i identification from %x with text %s" % (df, ecc, r["ident"])
    else:
        out += "Type %i TCAS report from %x: " % (df, ecc)
        a, tti = r["aux"], r["tti"]
        res, comp = _resolutions(a[0], a[1])
        rat, mte = a[2] & 1, (a[2] >> 1) & 1
        if tti == 1:
            out += "threat ID: %x advised: %s complement: %s" % (a[3], res, comp)
        elif tti == 2:
            if r["threat_alt"] == _d.NO_ALTITUDE:
                return None                         # MetricAltError out of parseMB_TCAS_threatloc (parse.py:407)
            out += "range: %i bearing: %i alt: %i advised: %s complement: %s" % (a[3] & 0x7F, a[3] >> 8, r["threat_alt"], res, comp)
        else:
            rat = mte = 0
            out += " (no handler for TTI=%i)" % tti
        if mte == 1:
            out += " (multiple threats)"
        if rat == 1:
            out += " (resolved)"
    if df == 20:
        if r["altitude"] == _d.NO_ALTITUDE:
            return None                             # MetricAltError (:251)
        return out + " at %ift" % r["altitude"]
    return out + " ident %x" % r["squawk"]


def report_lines(messages, records):
    """All printable lines of a batch, in order."""
    out = []
    for m, r in zip(messages, records):
        line = format_report(m, r)
        if line is not None:
            out.append(line)
    return out
