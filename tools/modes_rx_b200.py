#!/usr/bin/env python
"""modes_rx-style front end for the H100 receive chain (SURVEY.md 8 row f1).

The receiver half of apps/modes_rx + python/radio.py: the same "Receiver setup options" where they make sense
without a radio (radio.py:89-121), the same two offline sources (radio.py:221-232: a cfile or a UDP stream of
gr_complex), and the same two outlets for the slicer's messages: printed to stdout one per line
("<hex> <crc> <ref> <secs> <frac>", what lands on the gr.msg_queue) and published as ZMQ "dl_data"
(radio.py:79-87) on tcp://*:PORT with -t. With --reports / -l LAT,LON stdout carries what apps/modes_rx prints by
default instead: the text reports of python/msprint.py, decoded on the GPU (gr_air_modes_b200.decode: parse.py,
altitude.py, cpr.py for whole batches). KML, SBS-1 and FlightGear outputs are the reference's own pure-Python consumers
of the dl_data feed and are not re-implemented.

    python tools/modes_rx_b200.py -s capture.cfile -r 4e6 [-T 7.0] [-d] [-t 5556] [-n] [--reports | -l 37.4,-122.1]
    python tools/modes_rx_b200.py -s 127.0.0.1:12345 -r 4e6 --udp-idle 2.0

Differences, all on the far side of rx_path:
* live radios (-s uhd / osmocom) need GNU Radio: use gr_air_modes_b200.gr_adapter.rx_path inside modes_radio.
* radio.py:49-53 resamples rates below 4 Msps to 4 Msps with GNU Radio's pfb.arb_resampler_ccf. That filter
  bank is GNU Radio code and cannot be reproduced sample for sample; by default the chain is run at the native rate (it
  supports every rate from 2 Msps, preamble_impl.cc:56-63) and a note is printed; --resample puts a documented
  stand-in (tools/resample_standin.py: rational polyphase resampler on the host, where the reference runs its own)
  in front and runs the chain at 4 Msps like modes_rx does.
"""
import argparse
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


class report_queue:
    """What apps/modes_rx prints by default: air_modes.output_print(cpr_dec, publisher) (apps/modes_rx:77-78,
    python/msprint.py) - one text report per parsed message. The numbers come from the GPU batch decoder
    (gr_air_modes_b200.decode), the line format from gr_air_modes_b200.report."""

    def __init__(self, location, device, out=sys.stdout):
        from gr_air_modes_b200 import decode
        self._dec = decode.batch_decoder(location, device)      # = cpr_decoder(my_position), apps/modes_rx:68
        self._out, self._texts, self.count = out, [], 0

    def handle(self, msg):
        text = msg.to_string()
        self._texts.append(text.decode("ascii") if isinstance(text, bytes) else text)

    insert_tail = handle

    def flush(self):
        """Decode and print everything queued since the last call (one GPU batch)."""
        from gr_air_modes_b200 import report
        if self._texts:
            for line in report.report_lines(self._texts, self._dec.decode_messages(self._texts)):
                self._out.write(line + "\n")
                self.count += 1
            self._texts = []
        self._out.flush()

    def close(self):
        self._dec.close()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("-s", "--source", required=True, help="<filename> (cfile) or <ip:port> (UDP of gr_complex)")   # radio.py:94-95
    ap.add_argument("-t", "--tcp", type=int, default=None, metavar="PORT",
                    help="publish messages as ZMQ dl_data on tcp://*:PORT")                                        # radio.py:96-97,80-82
    ap.add_argument("-r", "--rate", type=float, default=4e6)                                                       # radio.py:112
    ap.add_argument("-T", "--threshold", type=float, default=7.0)                                                  # radio.py:114
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
    ap.add_argument("--chunk", type=int, default=1 << 24, help="complex samples per amb_process call")
    ap.add_argument("--udp-idle", type=float, default=2.0, help="end a UDP stream after this many idle seconds")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args(argv)

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
    sinks = []
    printer = None
    reporter = None
    if not args.no_print:
        if args.reports or args.location is not None:
            my_position = [float(x) for x in args.location.split(",")] if args.location is not None else None   # apps/modes_rx:64-65
            reporter = report_queue(my_position, args.device)
            sinks.append(reporter)
        else:
            printer = print_queue()
            sinks.append(printer)
    pub = None
    if args.tcp is not None:
        from gr_air_modes_b200.zmq_pub import zmq_queue
        pub = zmq_queue(["tcp://*:%i" % args.tcp])
        sinks.append(pub)
    rx = air_modes.rx_path(rx_rate, args.threshold, tee_queue(sinks), args.pmf, args.dcblock, device=args.device)   # radio.py:55-56

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
    st = rx.stats()
    print("# %d samples in, %d messages" % (st.samples_in, total), file=sys.stderr)
    if pub:
        import time
        time.sleep(0.2)                                                                                           # apps/modes_rx:88-91
        pub.close()
    if reporter:
        reporter.close()
    rx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
