#!/usr/bin/env python
"""modes_rx-style front end for the H100 receive chain (SURVEY.md 8 row f1).

The receiver half of apps/modes_rx + python/radio.py: the same "Receiver setup options" where they make sense
without a radio (radio.py:89-121), the same two offline sources (radio.py:221-232: a cfile or a UDP stream of
gr_complex), and the same two outlets for the slicer's messages: printed to stdout one per line
("<hex> <crc> <ref> <secs> <frac>", what lands on the gr.msg_queue) and published as ZMQ "dl_data"
(radio.py:79-87) on tcp://*:PORT with -t. With --reports / -l LAT,LON stdout carries what apps/modes_rx prints by
default instead: the text reports of python/msprint.py, decoded on the GPU (gr_air_modes_b200.decode: parse.py,
altitude.py, cpr.py for whole batches). With -P [PORT] the SBS-1 (BaseStation) feed of apps/modes_rx -P is served on
TCP port PORT (default 30003): the lines are formed on the GPU by the decoder (gr_air_modes_b200.decode, option sbs1)
with the date and time of each message's stamp in the host's local time, and sent by gr_air_modes_b200.sbs1. With
-l LAT,LON --coverage PATH the receiver coverage map of apps/modes_gui's azimuth map (python/az_map.py, the model, not
the widget) - the greatest range heard per 5-degree bearing sector and altitude band, in statute miles - is kept on the
GPU by the decoder (option coverage) and written to PATH as JSON after every chunk. With --beast [PORT] the frames are
served as the Beast binary feed of dump1090 and readsb (default port 30005, what mlat-client and the other consumers of
a receiver's raw frames read), with --avr [PORT] as the AVR raw feed (default port 30002; --avr-mlat for the "@" lines
with the timestamp): the bytes are formed on the GPU by the decoder (options beast and avr) from the receive chain's own
frames, stamps and levels, and sent by gr_air_modes_b200.sbs1's server. With -m HOST:PORT (--multiplayer, as
apps/modes_rx -m) every aircraft heard with a callsign, a velocity and a position is sent to a FlightGear multiplayer
server or instance at HOST:PORT, one UDP position packet per position message: the packets are formed on the GPU by the
decoder (option flightgear) and sent by gr_air_modes_b200.flightgear, stamped with the message's time.

With --input beast the frames come from another receiver instead of the IQ chain: -s FILE replays a recorded Beast
binary byte stream, -s HOST:PORT connects over TCP to a Beast server (dump1090 or readsb on port 30005, or this tool's
own --beast) and ends when the server closes. The bytes are parsed on the GPU (gr_air_modes_b200.beast) and every
chunk's frames go where the receive chain's go: their message lines to stdout, -t, --reports / -l, -P, --track /
--aircraft and --coverage, and the frames themselves to --beast / --avr. The stamps are the feed's 48-bit 12 MHz
counter, not wall-clock time: SBS-1 dates on Beast input follow that counter. Options that only configure the receive
chain (-d, -r, -T, --ec, --ec-any, --ap-filter, --resample, --modeac) are errors with --input beast.

With --modeac the receive chain also finds Mode A/C replies (squawk, altitude, SPI) on the GPU and prints one line per
reply after each chunk's messages (the format is in the option's help).

    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 [-T 7.0] [-d] [-t 5556] [-n] [--reports | -l 37.4,-122.1]
    python tools/modes_rx_b200.py -s 127.0.0.1:12345 -r 4e6 --udp-idle 2.0
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 --track 60 --aircraft aircraft.json
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 --track 60 --track-ext 60 --opstatus 30 --commb 30 \
        --aircraft aircraft.json
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 --reports --commb 30
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 --reports --opstatus 60
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 -l 37.4,-122.1 -P 30003
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 -l 37.4,-122.1 --coverage coverage.json
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 -n --beast 30005 --avr 30002 --avr-mlat
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 -l 37.4,-122.1 -m 127.0.0.1:5000
    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 --modeac
    python tools/modes_rx_b200.py --input beast -s 192.168.1.20:30005 --reports
    python tools/modes_rx_b200.py --input beast -s feed.bin -l 37.4,-122.1 -P 30003

Differences, all on the far side of rx_path:
* live radios (-s uhd / osmocom) need GNU Radio: use gr_air_modes_b200.gr_adapter.rx_path inside modes_radio.
* radio.py:49-53 resamples rates below 4 Msps to 4 Msps with GNU Radio's pfb.arb_resampler_ccf. That filter
  bank is GNU Radio code and cannot be reproduced sample for sample; by default the chain is run at the native rate (it
  supports every rate from 2 Msps, preamble_impl.cc:56-63) and a note is printed; --resample puts a documented
  stand-in (tools/resample_standin.py: rational polyphase resampler on the host, where the reference runs its own)
  in front and runs the chain at 4 Msps like modes_rx does.
"""
import argparse
import json
import os
import re
import socket
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gr_air_modes_b200 as air_modes  # noqa: E402


def file_source(path, chunk):
    """blocks.file_source(gr.sizeof_gr_complex, path) (radio.py:230): yields (float32 view, last?)."""
    n_total = os.path.getsize(path) // 8
    mm = np.memmap(path, dtype=np.float32, mode="r", shape=(2 * n_total,)) if n_total else np.zeros(0, np.float32)
    pos = 0
    while True:
        c = min(chunk, n_total - pos)
        yield np.asarray(mm[2 * pos: 2 * (pos + c)]), pos + c >= n_total
        pos += c
        if pos >= n_total:
            return


def open_udp(ip, port, idle_s):
    sock = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    sock.setsockopt(socket.SOL_SOCKET, socket.SO_RCVBUF, 1 << 24)
    try:
        sock.setsockopt(socket.SOL_SOCKET, getattr(socket, "SO_RCVBUFFORCE", 33), 1 << 24)   # beyond rmem_max when root
    except OSError:
        pass
    sock.bind((ip, port))
    sock.settimeout(idle_s)
    print("UDP receive buffer %d bytes" % sock.getsockopt(socket.SOL_SOCKET, socket.SO_RCVBUF), file=sys.stderr, flush=True)
    return sock


def udp_source(sock, chunk):
    """blocks.udp_source(gr.sizeof_gr_complex, ip, port) (radio.py:227): datagrams of whole gr_complex items.
    The stream ends after the socket's idle timeout without a datagram (a file-like end for offline use)."""
    buf, have, started = [], 0, False
    try:
        while True:
            try:
                d = sock.recv(65536)
            except socket.timeout:
                if not started:
                    continue
                break
            started = True
            d = d[: len(d) // 8 * 8]
            buf.append(np.frombuffer(d, np.float32))
            have += len(d) // 8
            if have >= chunk:
                yield np.concatenate(buf), False
                buf, have = [], 0
    finally:
        sock.close()
    yield (np.concatenate(buf) if buf else np.zeros(0, np.float32)), True


class tee_queue:
    """Fans the slicer's messages out to several msg_queue-like sinks (print + ZMQ)."""

    def __init__(self, sinks):
        self._sinks = sinks

    def handle(self, msg):
        for s in self._sinks:
            s.handle(msg)

    insert_tail = handle


class print_queue:
    def __init__(self, out=sys.stdout):
        self._out, self.count = out, 0

    def handle(self, msg):
        text = msg.to_string()
        self._out.write((text.decode("ascii") if isinstance(text, bytes) else text) + "\n")
        self.count += 1


def write_json(path, obj):
    """obj as JSON, written to a temporary file beside `path` and renamed over it, so that a reader never sees a
    half-written file."""
    tmp = "%s.tmp%d" % (path, os.getpid())
    with open(tmp, "w") as f:
        json.dump(obj, f)
    os.replace(tmp, path)


def write_aircraft(path, rows, ext=None):
    """The aircraft table (AIRCRAFT_DTYPE rows) as a JSON list, one object per aircraft (decode.aircraft_to_dict, or
    decode.aircraft_ext_to_dict with the extension rows `ext`), through write_json."""
    from gr_air_modes_b200 import decode
    if ext is None:
        write_json(path, [decode.aircraft_to_dict(r) for r in rows])
    else:
        write_json(path, [decode.aircraft_ext_to_dict(r, x) for r, x in zip(rows, ext)])


class report_queue:
    """What apps/modes_rx prints by default: air_modes.output_print(cpr_dec, publisher) (apps/modes_rx:77-78,
    python/msprint.py) - one text report per parsed message. The GPU batch decoder (gr_air_modes_b200.decode) forms
    the lines on the device (option reports: gr_air_modes_b200.report's lines). out=None decodes without printing;
    aircraft=PATH writes the decoder's aircraft table (option track) to PATH after every batch, with the extension of
    every row when track_ext is on; sbs1=server (gr_air_modes_b200.sbs1.sbs1_server) sends the batch's SBS-1 lines to
    it, with the date and time shifted by sbs1_tz minutes; flightgear=sender (gr_air_modes_b200.flightgear.fg_sender)
    sends the batch's FlightGear position packets to it; coverage=PATH writes the decoder's coverage map (option
    coverage) to PATH after every batch (decode.coverage_to_dict). A decoder given as `decoder` is used as it is, except
    that option reports is turned on when out is not None."""

    def __init__(self, location, device, out=sys.stdout, local_cpr=0, track=0, aircraft=None, decoder=None, commb=0,
                 opstatus=0, track_ext=0, sbs1=None, sbs1_tz=0, coverage=None, flightgear=None):
        from gr_air_modes_b200 import decode
        self._dec = decoder if decoder is not None else \
            decode.batch_decoder(location, device, local_cpr=local_cpr, track=track, commb=commb,
                                 opstatus=opstatus, track_ext=track_ext, sbs1=sbs1 is not None,
                                 sbs1_tz=sbs1_tz, coverage=coverage is not None,
                                 flightgear=flightgear is not None, reports=out is not None)   # = cpr_decoder(my_position), apps/modes_rx:68
        if decoder is not None and out is not None:
            decoder.set_reports(True)                   # flush() prints the decoder's text reports
        self._out, self._texts, self.count, self._aircraft = out, [], 0, aircraft
        self._coverage, self._location = coverage, location
        self._ext = track_ext > 0
        self._sbs1 = sbs1
        self._fg = flightgear

    def handle(self, msg):
        text = msg.to_string()
        self._texts.append(text.decode("ascii") if isinstance(text, bytes) else text)

    insert_tail = handle

    def flush(self):
        """Decode and print everything queued since the last call (one GPU batch)."""
        if self._texts:
            self._dec.decode_messages(self._texts)
            if self._sbs1 is not None:
                self._sbs1.send(self._dec.sbs1_text())
            if self._fg is not None:
                self._fg.send(self._dec.flightgear_bytes())
            if self._out is not None:
                text = self._dec.report_text()
                self._out.write(text.decode("latin-1"))
                self.count += text.count(b"\n")
            self._texts = []
        if self._out is not None:
            self._out.flush()
        if self._aircraft and self._ext:
            write_aircraft(self._aircraft, *self._dec.aircraft_ext())
        elif self._aircraft:
            write_aircraft(self._aircraft, self._dec.aircraft())
        if self._coverage:
            from gr_air_modes_b200 import decode
            write_json(self._coverage, decode.coverage_to_dict(self._dec.coverage(), self._location))

    def close(self):
        self._dec.close()
        if self._sbs1 is not None:
            self._sbs1.close()
        if self._fg is not None:
            self._fg.close()


class raw_feed:
    """The Beast binary and AVR raw feeds: every chunk's frames as the receive chain drained them (rx_path.frames, with
    their own stamps and levels, not parsed back from the message text) through a batch decoder with option beast and
    / or avr, and its bytes sent to the clients of `beast` / `avr` (gr_air_modes_b200.sbs1.sbs1_server each, or None).
    avr_form: 1 for "*" lines, 2 for "@" lines with the timestamp."""

    def __init__(self, device, beast=None, avr=None, avr_form=1):
        from gr_air_modes_b200 import decode
        self._dec = decode.batch_decoder(None, device, beast=beast is not None, avr=avr_form if avr is not None else 0)
        self._beast, self._avr = beast, avr

    def flush(self, frames):
        if len(frames) == 0:
            return
        self._dec.decode(frames)
        if self._beast is not None:
            self._beast.send(self._dec.beast_bytes())
        if self._avr is not None:
            self._avr.send(self._dec.avr_text())

    def close(self):
        self._dec.close()
        for server in (self._beast, self._avr):
            if server is not None:
                server.close()


def beast_file_source(path, chunk):
    """A recorded Beast byte stream: yields (bytes, last?), chunk bytes at a time."""
    with open(path, "rb") as f:
        data = f.read(chunk)
        while True:
            nxt = f.read(chunk)
            yield data, not nxt
            if not nxt:
                return
            data = nxt


def beast_tcp_source(host, port, chunk):
    """A Beast server's byte stream over TCP (dump1090 / readsb port 30005): yields (bytes, last?) as they arrive,
    at most chunk bytes at a time; the stream ends when the server closes the connection."""
    sock = socket.create_connection((host, port))
    try:
        while True:
            d = sock.recv(min(chunk, 1 << 20))
            yield d, not d
            if not d:
                return
    finally:
        sock.close()


class beast_input:
    """--input beast: the Beast bytes of another receiver parsed on the GPU (gr_air_modes_b200.beast.beast_reader) into
    frames, and the message line of every passed frame (amb_format_messages, what the slicer queues) handed to `queue`
    as rx_path hands its own."""

    def __init__(self, queue, device):
        from gr_air_modes_b200 import beast
        self._reader = beast.beast_reader(device)
        self._queue, self._first, self.messages = queue, True, 0

    def process(self, data, last):
        import ctypes as C
        from gr_air_modes_b200 import _lib
        fr = self._reader.process(data, flush=last)
        if len(fr):
            cap = 128 * len(fr) + 16
            buf = C.create_string_buffer(cap)
            k = _lib.check(_lib.load().amb_format_messages(C.c_void_p(fr.ctypes.data), len(fr), int(self._first), buf, cap))
            if k:
                for text in buf.value.decode("ascii").split("\n"):
                    self._queue.handle(air_modes.message(text))
                self._first = False
                self.messages += k
        return fr

    def stats(self):
        return self._reader.stats()

    def close(self):
        self._reader.close()


def local_utc_offset_minutes() -> int:
    """The host's current UTC offset in minutes, as datetime.now() writes local time in the reference's lines
    (sbs1.py:113-115), within the decoder's -720 .. 840."""
    import datetime
    off = datetime.datetime.now().astimezone().utcoffset()
    return max(-720, min(840, int(off.total_seconds() // 60)))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("-s", "--source", required=True,
                    help="<filename> (cfile) or <ip:port> (UDP of gr_complex); with --input beast a recorded Beast byte "
                         "stream or <host:port> of a Beast TCP server")                                              # radio.py:94-95
    ap.add_argument("--input", choices=("iq", "beast"), default="iq",
                    help="iq (default): samples through the GPU receive chain; beast: another receiver's Beast binary "
                         "frames (dump1090 / readsb port 30005), parsed on the GPU; their stamps are the feed's 12 MHz "
                         "counter, so SBS-1 dates follow that counter, not the wall clock")
    ap.add_argument("-t", "--tcp", type=int, default=None, metavar="PORT",
                    help="publish messages as ZMQ dl_data on tcp://*:PORT")                                        # radio.py:96-97,80-82
    ap.add_argument("-r", "--rate", type=float, default=None, help="default 4e6")                                 # radio.py:112
    ap.add_argument("-T", "--threshold", type=float, default=None, help="default 7.0")                            # radio.py:114
    ap.add_argument("-p", "--pmf", action="store_true", default=True, help="pulse matched filter (default on)")    # radio.py:116
    ap.add_argument("--no-pmf", dest="pmf", action="store_false")
    ap.add_argument("-d", "--dcblock", action="store_true", default=False)                                         # radio.py:118
    ap.add_argument("-n", "--no-print", action="store_true", default=False)                                        # apps/modes_rx:42
    ap.add_argument("--reports", action="store_true", default=False,
                    help="print decoded text reports (what apps/modes_rx prints by default) instead of the raw message lines")
    ap.add_argument("-l", "--location", type=str, default=None,
                    help="GPS coordinates of receiving station in format xx.xxxxx,xx.xxxxx (implies --reports)")   # apps/modes_rx:36-37
    ap.add_argument("--resample", action="store_true", default=False,
                    help="rates below 4 Msps: resample to 4 Msps in front of the chain like radio.py:49-53 "
                         "(stand-in for GNU Radio's pfb.arb_resampler_ccf, tools/resample_standin.py)")
    ap.add_argument("--chunk", type=int, default=1 << 24,
                    help="complex samples per amb_process call (with --input beast: bytes per call at most)")
    ap.add_argument("--udp-idle", type=float, default=2.0, help="end a UDP stream after this many idle seconds")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--ec", type=int, default=0, metavar="K",
                    help="correct DF11/DF17 frames over at most K (1..23) low-confidence bits; 0 = off, as the reference")
    ap.add_argument("--ec-any", type=int, default=0, metavar="M",
                    help="correct DF17 frames by at most M (1, 2) flipped bits anywhere, after --ec; 0 = off, as the reference")
    ap.add_argument("--modeac", action="store_true", default=False,
                    help="also find Mode A/C replies (needs the PMF and -r >= 4e6) and print one line per reply after "
                         "each chunk's messages, in stream order: 'modeac SQUAWK ALT SPI PEAK FLOOR SECS FRAC' with SQUAWK "
                         "the four octal digits, ALT the Gillham altitude in feet or '-', SPI 0 or 1, PEAK and FLOOR the "
                         "reply's linear levels (%%.6e) and SECS FRAC its time stamp (%%d %%.9f)")
    ap.add_argument("--ap-filter", type=int, default=0, metavar="S",
                    help="drop address/parity replies from aircraft not confirmed by a clean DF11/DF17 in the last S "
                         "seconds, and accept DF11 replies with an II/SI code from confirmed ones; 0 = off, as the reference")
    ap.add_argument("--commb", type=int, default=0, metavar="S",
                    help="text reports: infer the register (BDS 4,0 / 5,0 / 6,0) of DF20/21 replies the parser does not "
                         "handle, with the aircraft's ADS-B velocity of at most S (1..600) seconds before; 0 = off")
    ap.add_argument("--opstatus", type=int, default=0, metavar="S",
                    help="text reports: decode ADS-B operational status (TC 31) and target state (TC 29) squitters, and "
                         "rate positions by the aircraft's op status of at most S (1..600) seconds before; 0 = off")
    ap.add_argument("--local-cpr", type=int, default=0, metavar="S",
                    help="position reports: decode a message that has no global fix relative to the aircraft's last "
                         "position of at most S (1..600) seconds before; 0 = off, as the reference")
    ap.add_argument("--track", type=int, default=0, metavar="S",
                    help="keep a per-aircraft table on the GPU; an aircraft is dropped S (1..3600) seconds after its "
                         "last message; 0 = off")
    ap.add_argument("--aircraft", type=str, default=None, metavar="PATH",
                    help="after every chunk, write the aircraft table to PATH as JSON, one object per aircraft "
                         "(needs --track; decodes the messages even without --reports)")
    ap.add_argument("--track-ext", type=int, default=0, metavar="S",
                    help="keep beside every aircraft the latest op status, target state, position integrity (with "
                         "--opstatus) and Comm-B 4,0 / 5,0 / 6,0 (with --commb), each shown for S (1..3600) seconds, and "
                         "write them with --aircraft (needs --track); 0 = off")
    ap.add_argument("-P", "--sbs1", type=int, nargs="?", const=30003, default=None, metavar="PORT",
                    help="serve the SBS-1 (BaseStation) feed on TCP port PORT (default 30003), as apps/modes_rx -P; "
                         "decodes the messages even without --reports")                                          # apps/modes_rx:48,84-85
    ap.add_argument("--sbs1-wait", type=float, default=0.0, metavar="S",
                    help="with -P: wait up to S seconds for the first SBS-1 client before reading the source (for "
                         "replaying a recording); 0 = start at once, as modes_rx")
    ap.add_argument("-m", "--multiplayer", type=str, default=None, metavar="HOST:PORT",
                    help="FlightGear multiplayer feed: UDP position packets to HOST:PORT")                      # apps/modes_rx:50-51
    ap.add_argument("--coverage", type=str, default=None, metavar="PATH",
                    help="after every chunk, write the receiver coverage map to PATH as JSON: the greatest range "
                         "(statute miles) heard per 5-degree bearing sector and altitude band, as modes_gui's azimuth "
                         "map keeps it (needs -l; decodes the messages even without --reports)")
    ap.add_argument("--beast", type=int, nargs="?", const=30005, default=None, metavar="PORT",
                    help="serve the frames as the Beast binary feed (dump1090's) on TCP port PORT (default 30005)")
    ap.add_argument("--avr", type=int, nargs="?", const=30002, default=None, metavar="PORT",
                    help="serve the frames as the AVR raw feed (\"*<hex>;\" lines) on TCP port PORT (default 30002)")
    ap.add_argument("--avr-mlat", action="store_true", default=False,
                    help="with --avr: \"@<timestamp><hex>;\" lines, the 48-bit 12 MHz timestamp of each frame")
    ap.add_argument("--feed-wait", type=float, default=0.0, metavar="S",
                    help="with --beast / --avr: wait up to S seconds for the first client of each feed before reading "
                         "the source (for replaying a recording); 0 = start at once")
    args = ap.parse_args(argv)
    if args.input == "beast":
        given = [name for name, on in (("-d", args.dcblock), ("-r", args.rate is not None), ("-T", args.threshold is not None),
                                        ("--ec", args.ec), ("--ec-any", args.ec_any), ("--ap-filter", args.ap_filter),
                                        ("--resample", args.resample), ("--modeac", args.modeac)) if on]
        if given:
            ap.error("%s configure%s the receive chain, which --input beast does not run" %
                     (", ".join(given), "s" if len(given) == 1 else ""))
    args.rate = 4e6 if args.rate is None else args.rate
    args.threshold = 7.0 if args.threshold is None else args.threshold
    if args.modeac and (not args.pmf or (int(args.rate) < 4e6 and not args.resample)):
        ap.error("--modeac needs the PMF and a chain rate of at least 4 Msps")
    if args.coverage and args.location is None:
        ap.error("--coverage needs -l LAT,LON")
    if args.sbs1 is not None and not 0 < args.sbs1 < 65536:
        ap.error("--sbs1: a TCP port 1 .. 65535")
    if not 0 <= args.sbs1_wait <= 3600:
        ap.error("--sbs1-wait: 0 .. 3600 seconds")
    if args.sbs1_wait and args.sbs1 is None:
        ap.error("--sbs1-wait needs -P")
    for name, port in (("--beast", args.beast), ("--avr", args.avr)):
        if port is not None and not 0 < port < 65536:
            ap.error("%s: a TCP port 1 .. 65535" % name)
    if args.avr_mlat and args.avr is None:
        ap.error("--avr-mlat needs --avr")
    if not 0 <= args.feed_wait <= 3600:
        ap.error("--feed-wait: 0 .. 3600 seconds")
    if args.feed_wait and args.beast is None and args.avr is None:
        ap.error("--feed-wait needs --beast or --avr")
    if args.multiplayer is not None:
        m = re.fullmatch(r"(.+):(\d{1,5})", args.multiplayer)                                                    # apps/modes_rx:80-82
        if not m or not 0 < int(m.group(2)) < 65536:
            ap.error("--multiplayer: HOST:PORT with a UDP port 1 .. 65535")
        args.multiplayer = (m.group(1), int(m.group(2)))
    if not 0 <= args.track <= 3600:
        ap.error("--track: 0 (off) .. 3600 seconds")
    if args.aircraft and args.track <= 0:
        ap.error("--aircraft needs --track S")
    if not 0 <= args.track_ext <= 3600:
        ap.error("--track-ext: 0 (off) .. 3600 seconds")
    if args.track_ext and args.track <= 0:
        ap.error("--track-ext needs --track S")
    with_table = bool(args.aircraft and args.track_ext)     # the extension shows what --commb / --opstatus decode
    if not 0 <= args.commb <= 600:
        ap.error("--commb: 0 (off) .. 600 seconds")
    if args.commb and not (args.reports or args.location is not None or with_table):
        ap.error("--commb needs --reports or -l")
    if not 0 <= args.opstatus <= 600:
        ap.error("--opstatus: 0 (off) .. 600 seconds")
    if args.opstatus and not (args.reports or args.location is not None or with_table):
        ap.error("--opstatus needs --reports or -l")
    return args


def format_modeac(r) -> str:
    """One --modeac line: 'modeac SQUAWK ALT SPI PEAK FLOOR SECS FRAC' (see the option's help)."""
    alt = "-" if int(r["altitude"]) == air_modes.blocks.NO_ALTITUDE else "%d" % int(r["altitude"])
    return "modeac %04d %s %d %.6e %.6e %d %.9f" % (int(r["squawk"]), alt, int(r["spi"]), float(r["peak"]), float(r["floor"]),
                                                   int(r["secs"]), float(r["frac"]))


def main(argv=None):
    args = parse_args(argv)

    if args.input == "beast":
        return main_beast(args)
    if args.source in ("uhd", "osmocom"):
        raise SystemExit("live radios need GNU Radio: use gr_air_modes_b200.gr_adapter.rx_path in modes_radio (INTEGRATION.md)")
    rate = int(args.rate)                                                                                          # radio.py:44
    resampler = None
    rx_rate = rate
    if rate < 4e6 and args.resample:                                                                               # radio.py:49-51
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from resample_standin import StreamResampler
        resampler = StreamResampler(rate, 4e6)
        rx_rate = 4000000
        print("# rate %d < 4 Msps: resampling %d/%d to 4 Msps in front of the chain (stand-in for GNU Radio's "
              "pfb.arb_resampler_ccf, radio.py:49-53)" % (rate, resampler.up, resampler.down), file=sys.stderr)
    elif rate < 4e6:
        print("# rate %d < 4 Msps: the reference would resample to 4 Msps (radio.py:49-53, GNU Radio PFB, not "
              "reproduced; --resample runs a stand-in); running the chain at the native rate" % rate, file=sys.stderr)
    sinks, printer, reporter, raw, pub = make_outputs(args)
    rx = air_modes.rx_path(rx_rate, args.threshold, tee_queue(sinks), args.pmf, args.dcblock, device=args.device,
                           ec=args.ec, ec_any=args.ec_any, ap_filter=args.ap_filter, modeac=args.modeac)   # radio.py:55-56

    if ":" in args.source and not os.path.exists(args.source):
        m = re.search(r"(.*)\:(\d{1,5})$", args.source)                                                           # radio.py:223-226
        if not m:
            raise SystemExit("Please input UDP source e.g. 192.168.10.1:12345")
        print("Using UDP source %s:%s" % m.groups(), file=sys.stderr)
        src = udp_source(open_udp(m.group(1), int(m.group(2)), args.udp_idle), args.chunk)
    else:
        print("Using file source %s" % args.source, file=sys.stderr)
        src = file_source(args.source, args.chunk)
    print("Rate is %i" % rate, file=sys.stderr)

    total = 0
    for block, last in src:
        if resampler is not None:
            block = resampler.push(block, last)
        total += rx.process(block, flush=last)
        if printer:
            sys.stdout.flush()
        if reporter:
            reporter.flush()
        if raw:
            raw.flush(rx.frames)
        if args.modeac:
            for r in rx.modeac():
                print(format_modeac(r))
            sys.stdout.flush()
    st = rx.stats()
    print("# %d samples in, %d messages" % (st.samples_in, total), file=sys.stderr)
    close_outputs(reporter, raw, pub)
    rx.close()
    return 0


def main_beast(args):
    """--input beast: the outputs of main(), fed by another receiver's Beast frames instead of the receive chain."""
    sinks, printer, reporter, raw, pub = make_outputs(args)
    src_in = beast_input(tee_queue(sinks), args.device)
    if ":" in args.source and not os.path.exists(args.source):
        m = re.search(r"(.*)\:(\d{1,5})$", args.source)
        if not m:
            raise SystemExit("Please input a Beast server as host:port, e.g. 127.0.0.1:30005")
        print("Using Beast TCP source %s:%s" % m.groups(), file=sys.stderr)
        src = beast_tcp_source(m.group(1), int(m.group(2)), args.chunk)
    else:
        print("Using Beast file source %s" % args.source, file=sys.stderr)
        src = beast_file_source(args.source, args.chunk)
    for data, last in src:
        frames = src_in.process(data, last)
        if printer:
            sys.stdout.flush()
        if reporter:
            reporter.flush()
        if raw:
            raw.flush(frames)
    st = src_in.stats()
    print("# %d bytes in, %d Mode S frames, %d messages" % (st["bytes_in"], st["modes"], src_in.messages), file=sys.stderr)
    close_outputs(reporter, raw, pub)
    src_in.close()
    return 0


def make_outputs(args):
    """The sinks of the messages (printer, reporter, ZMQ publisher) and the raw feeds, as the options ask."""
    sinks = []
    printer = None
    reporter = None
    my_position = [float(x) for x in args.location.split(",")] if args.location is not None else None   # apps/modes_rx:64-65
    server = None
    if args.sbs1 is not None:
        from gr_air_modes_b200.sbs1 import sbs1_server
        server = sbs1_server(args.sbs1)                                                                            # apps/modes_rx:84-85
        if args.sbs1_wait and not server.wait_for_client(args.sbs1_wait):
            print("# no SBS-1 client within %g s, starting anyway" % args.sbs1_wait, file=sys.stderr)
    feed = {"sbs1": server, "sbs1_tz": local_utc_offset_minutes()} if server is not None else {}
    if args.coverage:
        feed["coverage"] = args.coverage
    if args.multiplayer is not None:
        from gr_air_modes_b200.flightgear import fg_sender
        feed["flightgear"] = fg_sender(*args.multiplayer)                                                         # apps/modes_rx:80-82
    if not args.no_print:
        if args.reports or args.location is not None:
            reporter = report_queue(my_position, args.device, local_cpr=args.local_cpr, track=args.track, commb=args.commb,
                                    opstatus=args.opstatus, aircraft=args.aircraft, track_ext=args.track_ext, **feed)
            sinks.append(reporter)
        else:
            printer = print_queue()
            sinks.append(printer)
    if (args.aircraft or server is not None or args.coverage or args.multiplayer) and reporter is None:   # no printed reports
        reporter = report_queue(my_position, args.device, out=None, local_cpr=args.local_cpr, track=args.track,
                                aircraft=args.aircraft, **({"commb": args.commb, "opstatus": args.opstatus,
                                                            "track_ext": args.track_ext} if args.track_ext else {}),
                                **feed)
        sinks.append(reporter)
    raw = None
    if args.beast is not None or args.avr is not None:
        from gr_air_modes_b200.sbs1 import sbs1_server
        servers = [sbs1_server(p) if p is not None else None for p in (args.beast, args.avr)]
        for name, srv in zip(("Beast", "AVR"), servers):
            if srv is not None and args.feed_wait and not srv.wait_for_client(args.feed_wait):
                print("# no %s client within %g s, starting anyway" % (name, args.feed_wait), file=sys.stderr)
        raw = raw_feed(args.device, *servers, avr_form=2 if args.avr_mlat else 1)
    pub = None
    if args.tcp is not None:
        from gr_air_modes_b200.zmq_pub import zmq_queue
        pub = zmq_queue(["tcp://*:%i" % args.tcp])
        sinks.append(pub)
    return sinks, printer, reporter, raw, pub


def close_outputs(reporter, raw, pub):
    if pub:
        import time
        time.sleep(0.2)                                                                                           # apps/modes_rx:88-91
        pub.close()
    if reporter:
        reporter.close()
    if raw:
        raw.close()


if __name__ == "__main__":
    sys.exit(main())
