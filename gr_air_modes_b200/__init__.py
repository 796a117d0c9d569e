"""gr-air-modes_b200: the Mode S / ADS-B receive hot path of gr-air-modes as sm_90a CUDA.

Python identifiers cannot contain '-', so the package directory is gr_air_modes_b200. It exports the
reference's names for the path (python/__init__.py:34,44 exports the swig blocks and rx_path):

    import gr_air_modes_b200 as air_modes
    q = air_modes.msg_queue()
    rx = air_modes.rx_path(4e6, 7.0, q, use_pmf=True)
    rx.process(iq, flush=True)

Importing the package does not need a GPU; constructing a block does (no CPU fallback).
"""
from .blocks import (preamble, slicer, rx_path, modes_check_crc, modes_crc, msg_queue, message,
                     message_from_string, format_message, query_geometry)
from ._lib import Frame, Stats

__all__ = ["preamble", "slicer", "rx_path", "modes_check_crc", "modes_crc", "msg_queue", "message",
           "message_from_string", "format_message", "query_geometry", "Frame", "Stats"]
