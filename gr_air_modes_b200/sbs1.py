"""SBS-1 (BaseStation) feed server: the TCP side of the reference's output_sbs1 (python/sbs1.py:49-111, modes_rx -P),
for the lines the batch decoder writes on the GPU (batch_decoder(sbs1=True).sbs1_text()).

Like the reference it listens on a port, sends every line to every connected client and drops a client whose socket
fails. Unlike it, no thread polls for new clients: pending connections are accepted with non-blocking calls each time
lines are sent, so nothing is left running. Sends never block the receiver: what a client's socket does not take at
once waits in that client's own buffer and goes out with the next send, and a client whose backlog grows past
`max_backlog` bytes (it stopped reading) is dropped."""
from __future__ import annotations

import select
import socket
import time

MAX_BACKLOG = 16 << 20           # bytes a client may fall behind before it is dropped (several seconds of busy traffic)


class sbs1_server:
    """Listen on (host, port); port 0 picks a free port (see .port). send(data) accepts whoever is waiting, then queues
    data for every client and writes what each socket takes; close() flushes what it can for up to `linger` seconds and
    closes every socket."""

    def __init__(self, port: int, host: str = "", max_backlog: int = MAX_BACKLOG):
        self._s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        self._s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        try:
            self._s.bind((host, int(port)))
            self._s.listen(8)
            self._s.setblocking(False)
        except OSError:
            self._s.close()
            raise
        self._max = int(max_backlog)
        self._conns: dict[socket.socket, bytearray] = {}     # client -> bytes it has not taken yet

    @property
    def port(self) -> int:
        return self._s.getsockname()[1]

    @property
    def connections(self) -> int:
        return len(self._conns)

    def accept_pending(self):
        """Accept every connection waiting on the listening socket, without blocking (add_pending_conns, sbs1.py:105)."""
        while True:
            try:
                conn, _ = self._s.accept()
            except OSError:                             # BlockingIOError: nobody is waiting
                return
            conn.setblocking(False)
            self._conns[conn] = bytearray()

    def wait_for_client(self, timeout: float) -> bool:
        """Block up to `timeout` seconds until at least one client is connected (e.g. before replaying a recording)."""
        deadline = time.monotonic() + timeout
        while True:
            self.accept_pending()
            left = deadline - time.monotonic()
            if self._conns or left <= 0:
                return bool(self._conns)
            select.select([self._s], [], [], left)

    def _drop(self, conn):
        del self._conns[conn]
        try:
            conn.close()
        except OSError:
            pass

    def _flush(self, conn):
        buf = self._conns[conn]
        try:
            while buf:
                del buf[:conn.send(buf)]
        except BlockingIOError:
            pass                                        # the socket is full: the rest goes with the next send
        except OSError:
            self._drop(conn)

    def send(self, data: bytes):
        """Queue data for every client (sbs1.py:92-101) and write what each socket takes now; a client whose send fails,
        or whose backlog would exceed max_backlog bytes, is dropped."""
        self.accept_pending()
        for conn in list(self._conns):
            buf = self._conns[conn]
            if len(buf) + len(data) > self._max:
                self._drop(conn)
                continue
            buf += data
            self._flush(conn)

    def close(self, linger: float = 2.0):
        deadline = time.monotonic() + linger
        while self._conns and time.monotonic() < deadline:
            waiting = [c for c, b in self._conns.items() if b]
            if not waiting:
                break
            _, ready, _ = select.select([], waiting, [], max(0.0, deadline - time.monotonic()))
            for conn in ready:
                self._flush(conn)
        for conn in list(self._conns):
            self._drop(conn)
        self._s.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
