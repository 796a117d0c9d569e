"""FlightGear multiplayer feed sender: the UDP side of the reference's output_flightgear (python/flightgear.py:17-83,
modes_rx -m HOST:PORT), for the position packets the batch decoder writes on the GPU
(batch_decoder(flightgear=True).flightgear_bytes()).

Like the reference it sends each 232-byte packet as one datagram to (host, port), where a FlightGear instance started
with --multiplay=in,... (or any listener) picks it up. Unlike it, the socket is non-blocking: a datagram the kernel
will not take at once (a full send buffer, an unreachable port reported back by ICMP) is dropped and counted, never
waited for, so the receiver never stalls on its output. Nothing runs in the background."""
from __future__ import annotations

import socket

PACKET_BYTES = 232               # '!4sLLLLL8s0L' header + '!96sdd3d3f3f3f3f3fI' position message (flightgear.py:97, 190)


class fg_sender:
    """send(packets) sends every PACKET_BYTES-byte packet of `packets` (the concatenation flightgear_bytes() returns)
    to (host, port) as its own datagram; .sent and .dropped count the datagrams; close() closes the socket."""

    def __init__(self, host: str, port: int):
        self.addr = (socket.gethostbyname(host), int(port))
        self._s = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        self._s.setblocking(False)
        self.sent = 0
        self.dropped = 0

    def send(self, packets: bytes) -> int:
        """Send the packets; returns how many went out. `packets` must be a whole number of packets."""
        data = memoryview(bytes(packets))
        if len(data) % PACKET_BYTES:
            raise ValueError("fg_sender.send: %d bytes is not a whole number of %d-byte packets" % (len(data), PACKET_BYTES))
        n = 0
        for off in range(0, len(data), PACKET_BYTES):
            try:
                self._s.sendto(data[off: off + PACKET_BYTES], self.addr)
                n += 1
            except OSError:                     # BlockingIOError, ConnectionRefusedError (ICMP), ...: drop it
                self.dropped += 1
        self.sent += n
        return n

    def close(self):
        self._s.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
