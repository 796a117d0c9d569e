"""GNU Radio adapters: the H100 receive path as drop-ins for the reference's blocks inside a flowgraph.

    air_modes.rx_path(rate, threshold, queue, use_pmf, use_dcblock)   python/rx_path.py:27      -> rx_path (sink of gr_complex)
    air_modes.preamble(channel_rate, threshold_db)                    preamble.h:36-45          -> preamble (2 x float in, float out)
    air_modes.slicer(queue)                                           slicer.h:37-42            -> slicer (sink of float)

Importable only where gnuradio (and its pmt) is installed; radio.py:55-56,73-76 keep working:
`self.connect(source, rx_path(rate, threshold, queue, pmf, dcblock))`, and so does the reference's own wiring of the
two split blocks (rx_path.py:57-65): the preamble adapter emits 240 float items per detection with a `preamble_found`
stream tag whose value is the (uint64 secs, double frac) tuple of preamble_impl.cc:224-232, the slicer adapter reads
exactly that. tests/test_library_simt.py drives all three with a stand-in `gnuradio.gr` (ragged work() calls, restart).

work() hands its items to rx_path.process(collect=False): the library gathers such small calls in its pinned ingest ring
and launches once enough are pending; finished frames are picked up with the non-blocking poll, so a work() call costs a
memcpy and never waits for the GPU.
"""
import numpy as np
from gnuradio import gr  # noqa: F401  (ImportError here is the import guard)
import pmt

from . import blocks


class rx_path(gr.sync_block):
    def __init__(self, rate, threshold, queue, use_pmf=False, use_dcblock=False, device=0):
        gr.sync_block.__init__(self, "modes_rx_path_b200", in_sig=[np.complex64], out_sig=None)
        self._impl = blocks.rx_path(rate, threshold, queue, use_pmf, use_dcblock, device=device)
        for name in ("set_rate", "set_threshold", "set_pmf", "get_pmf", "get_threshold"):
            setattr(self, name, getattr(self._impl, name))
        self._open = False

    def start(self):
        self._impl.reset()                      # a restarted flowgraph is a new stream (sample 0, fresh slicer state)
        self._impl._slicer._first = True
        self._open = True
        return True

    def work(self, input_items, output_items):
        if not self._open:
            self.start()
        x = input_items[0]
        n = len(x)
        # rx_time tags of a UHD source (preamble_impl.cc:164-170): tag at item 0 = start time, later ones = overflows
        for t in self.get_tags_in_range(0, self.nitems_read(0), self.nitems_read(0) + n):
            if pmt.symbol_to_string(t.key) == "rx_time":
                secs = pmt.to_uint64(pmt.tuple_ref(t.value, 0))
                frac = pmt.to_double(pmt.tuple_ref(t.value, 1))
                if t.offset == 0:
                    self._impl.set_start_time(secs, frac)
                else:
                    self._impl.add_time_tag(t.offset, secs, frac)
        self._impl.process(x, collect=False)    # chunking does not change results (DESIGN.md 4)
        self._impl.poll_ready()                 # messages of whatever has completed; never blocks
        return n

    def stop(self):
        if self._open:
            self._impl.process(np.zeros(0, np.complex64), flush=True)   # end-of-stream rules + the remaining messages
            self._open = False
        return True


class preamble(gr.basic_block):
    """in0 = signal, in1 = moving-average reference (preamble_impl.cc:43); out = 240 chips per detection + tag."""

    def __init__(self, channel_rate, threshold_db, device=0):
        gr.basic_block.__init__(self, "modes_preamble_b200", in_sig=[np.float32, np.float32], out_sig=[np.float32])
        self._impl = blocks.preamble(channel_rate, threshold_db, device=device)
        self.set_output_multiple(240)
        self._key = pmt.string_to_symbol("preamble_found")         # preamble_impl.cc:53
        self._me = pmt.string_to_symbol("preamble_b200")
        self._out = []                                             # packets decided but not yet written: (chips, secs, frac)
        for name in ("set_rate", "set_threshold", "get_rate", "get_threshold"):
            setattr(self, name, getattr(self._impl, name))

    def forecast(self, noutput_items, ninput_items_required):
        for k in range(len(ninput_items_required)):
            ninput_items_required[k] = 0 if self._out else 1

    def _emit(self, out):
        room = len(out) // 240
        k = 0
        while self._out and k < room:
            chips, secs, frac = self._out.pop(0)
            out[240 * k: 240 * (k + 1)] = chips
            self.add_item_tag(0, self.nitems_written(0) + 240 * k, self._key,
                              pmt.make_tuple(pmt.from_uint64(int(secs)), pmt.from_double(float(frac))), self._me)
            k += 1
        return 240 * k

    def general_work(self, input_items, output_items):
        n = min(len(input_items[0]), len(input_items[1]))
        if n:
            chips, tags = self._impl.process(input_items[0][:n], input_items[1][:n], flush=False)
            for c, (_, secs, frac) in zip(chips, tags):
                self._out.append((c, secs, frac))
            self.consume_each(n)
        return self._emit(output_items[0])

    def stop(self):
        chips, tags = self._impl.process(np.zeros(0, np.float32), np.zeros(0, np.float32), flush=True)
        for c, (_, secs, frac) in zip(chips, tags):
            self._out.append((c, secs, frac))          # a scheduler that calls stop() will not ask for output again
        return True


class slicer(gr.sync_block):
    """Sink of the preamble block's stream: 240 chips per `preamble_found` tag -> queue messages (slicer_impl.cc:102-198)."""

    def __init__(self, queue, device=0):
        gr.sync_block.__init__(self, "modes_slicer_b200", in_sig=[np.float32], out_sig=None)
        self._impl = blocks.slicer(queue, device=device)
        self.set_output_multiple(240)

    def work(self, input_items, output_items):
        x = input_items[0]
        n = len(x)
        base = self.nitems_read(0)
        chips, tags, used = [], [], n
        for t in self.get_tags_in_range(0, base, base + n):
            if pmt.symbol_to_string(t.key) != "preamble_found":
                continue
            o = int(t.offset - base)
            if o + 240 > n:                 # packet not completely here yet: leave it for the next call (slicer_impl.cc:107-114)
                used = min(used, o)
                break
            chips.append(x[o:o + 240])
            tags.append((pmt.to_uint64(pmt.tuple_ref(t.value, 0)), pmt.to_double(pmt.tuple_ref(t.value, 1))))
        if chips:
            self._impl.process(np.stack(chips), tags)
        return used
