"""Seeded synthetic 1090 MHz Mode S IQ scenes (SURVEY.md 8d configs).

Tooling for tests and bench.py, not part of the receive path. The waveform model follows what the
reference detector/slicer expect: 0.5 us chips at 2 Mchip/s (preamble_impl.cc:46), preamble pulses
at chips 0, 2, 7, 9 (preamble_impl.cc:88-90, 158-162), PPM data from chip 16 with bit 1 = (on, off)
(slicer_impl.cc:133-151), 56/112 data bits, parity = Mode S CRC with polynomial 0xFFF409
(modes_crc.cc:31).  Output format is interleaved float32 I/Q = gr_complex (rx_path.py:29).
"""
from __future__ import annotations

import dataclasses
import hashlib

import numpy as np

POLY = 0xFFF409


def crc24(data: bytes) -> int:
    """Bitwise Mode S CRC over `data` (same polynomial/init as modes_crc.cc:31-63), tool-local."""
    crc = 0
    for byte in data:
        crc ^= byte << 16
        for _ in range(8):
            crc <<= 1
            if crc & 0x1000000:
                crc ^= 0x1000000 | POLY
    return crc & 0xFFFFFF


def make_frame(df: int, rng: np.random.Generator, garble_bits: int = 0) -> bytes:
    """Random DF11 (56 bit) or DF17-style (112 bit) frame whose last 24 bits are the CRC (II=0)."""
    nbytes = 14 if df in (16, 17, 20, 21) else 7
    body = bytearray(rng.integers(0, 256, nbytes - 3, dtype=np.uint8).tobytes())
    body[0] = ((df & 0x1F) << 3) | (body[0] & 0x07)
    frame = bytearray(body) + crc24(bytes(body)).to_bytes(3, "big")
    for _ in range(garble_bits):
        b = int(rng.integers(0, nbytes * 8))
        frame[b // 8] ^= 0x80 >> (b % 8)
    return bytes(frame)


def frame_chips(frame: bytes) -> np.ndarray:
    """On/off chip pattern (16 preamble chips + 2 per bit)."""
    bits = np.unpackbits(np.frombuffer(frame, dtype=np.uint8))
    chips = np.zeros(16 + 2 * bits.size, dtype=np.float64)
    chips[[0, 2, 7, 9]] = 1.0
    chips[16 + 2 * np.nonzero(bits)[0]] = 1.0
    chips[17 + 2 * np.nonzero(bits == 0)[0]] = 1.0
    return chips


@dataclasses.dataclass
class Burst:
    start: float          # fractional sample index of the leading edge of the first preamble pulse
    frame: bytes
    amplitude: float
    phase: float
    freq: float = 0.0     # carrier offset, cycles/sample


def burst_waveform(b: Burst, spc: float):
    """(first_sample, complex64 samples): box-car integrated rectangular pulses at a fractional offset."""
    chips = frame_chips(b.frame)
    knots = np.arange(chips.size + 1) * spc
    cum = np.concatenate([[0.0], np.cumsum(chips) * spc])
    n0 = int(np.floor(b.start))
    n1 = int(np.ceil(b.start + chips.size * spc)) + 1
    edges = np.arange(n0, n1 + 1, dtype=np.float64) - b.start
    integ = np.interp(edges, knots, cum)
    cover = np.diff(integ)  # fraction of each sample interval covered by "on"
    n = np.arange(n0, n1, dtype=np.float64)
    ph = b.phase + 2 * np.pi * b.freq * (n - b.start)
    w = (b.amplitude * cover) * np.exp(1j * ph)
    return n0, w.astype(np.complex64)


@dataclasses.dataclass
class Scene:
    rate: float
    n: int
    iq: np.ndarray                # float32, shape (2n,), interleaved I/Q
    bursts: list

    def sha256(self) -> str:
        return hashlib.sha256(self.iq.tobytes()).hexdigest()


def make_scene(rate: float, n: int, n_bursts: int, seed: int, *, noise_sigma: float = 0.01,
               snr_db=(6.0, 30.0), df_choices=(11, 17), garble_frac: float = 0.0,
               starts=None, amplitude=None, quantize_bits: int | None = None,
               fruit: int = 0, min_gap: float | None = None) -> Scene:
    """Complex Gaussian noise (sigma per component) + `n_bursts` Mode S bursts.

    SNR = A^2 / (2 sigma^2) drawn uniformly in dB from `snr_db`; start times uniform with fractional
    offsets (or Poisson-like overlap when min_gap is None); random carrier phase per burst.
    `quantize_bits` rounds I/Q to a signed fixed-point grid (exactly representable, for small fixtures).
    `fruit` adds that many isolated 0.45 us Mode A/C-like pulses pairs.
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    iq = np.empty((n, 2), dtype=np.float32)
    step = 1 << 22
    for a in range(0, n, step):  # chunked to bound temporaries
        m = min(step, n - a)
        iq[a:a + m] = rng.standard_normal((m, 2), dtype=np.float32) * np.float32(noise_sigma)
    c = iq.view(np.complex64).reshape(n)
    bursts = []
    span = 240 * spc + 8
    if starts is None:
        if min_gap is not None:
            # non-overlapping: jittered grid
            slots = int((n - 2 * span) // (span + min_gap))
            pick = np.sort(rng.choice(slots, size=min(n_bursts, slots), replace=False))
            starts = span / 2 + pick * (span + min_gap) + rng.uniform(0, min_gap, pick.size)
        else:
            starts = np.sort(rng.uniform(span, n - 2 * span, n_bursts))
    for k, s in enumerate(starts):
        df = int(df_choices[int(rng.integers(0, len(df_choices)))])
        garble = int(rng.integers(1, 6)) if rng.random() < garble_frac else 0
        frame = make_frame(df, rng, garble)
        if amplitude is None:
            snr = rng.uniform(*snr_db)
            amp = float(np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (snr / 10))) if noise_sigma > 0 else 0.5
        else:
            amp = float(amplitude)
        b = Burst(float(s), frame, amp, float(rng.uniform(0, 2 * np.pi)))
        n0, w = burst_waveform(b, spc)
        lo, hi = max(n0, 0), min(n0 + w.size, n)
        if hi > lo:
            c[lo:hi] += w[lo - n0:hi - n0]
        bursts.append(b)
    for _ in range(fruit):
        s = rng.uniform(0, n - 64 * spc)
        amp = float(np.sqrt(2.0 * max(noise_sigma, 1e-3) ** 2 * 10 ** (rng.uniform(10, 30) / 10)))
        ph = rng.uniform(0, 2 * np.pi)
        for off in (0.0, rng.integers(1, 14) * 1.45 * 2 * spc):  # two pulses 1.45 us multiples apart
            a0 = int(s + off)
            a1 = min(a0 + max(int(round(0.9 * spc)), 1), n)
            c[a0:a1] += np.complex64(amp * np.exp(1j * ph))
    if quantize_bits is not None:
        q = float(1 << (quantize_bits - 1))
        np.clip(np.rint(iq * q), -q, q - 1, out=iq)
        iq /= np.float32(q)
    return Scene(rate, n, iq.reshape(2 * n), bursts)


# ---------------------------------------------------------------------------------------------------------
# The same scene model, vectorised (numpy for the frames, torch for the waveforms): bench.py needs scenes of
# 2^28 samples with up to ~10^6 bursts (BASELINE configs[4]), which the per-burst Python loop above cannot
# deliver in bench time. Not bit-identical to make_scene (other random streams); parity is always checked
# against the oracle on the very buffer this returns.
# ---------------------------------------------------------------------------------------------------------
_CRC_TABLE = None


def _crc_table():
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = np.zeros(256, np.uint32)
        for n in range(256):
            c = n << 16
            for _ in range(8):
                c = ((c << 1) ^ POLY) & 0xFFFFFF if c & 0x800000 else (c << 1) & 0xFFFFFF
            t[n] = c
        _CRC_TABLE = t
    return _CRC_TABLE


def make_frames(dfs: np.ndarray, rng: np.random.Generator, garble_frac: float = 0.0):
    """Vectorised make_frame: (frames uint8[nb,14], nbytes int[nb]); short frames are zero beyond byte 7."""
    nb = dfs.size
    long_ = np.isin(dfs, (16, 17, 20, 21))
    nbytes = np.where(long_, 14, 7)
    fr = rng.integers(0, 256, (nb, 14), dtype=np.uint8)
    fr[:, 0] = ((dfs.astype(np.uint8) & 0x1F) << 3) | (fr[:, 0] & 0x07)
    T = _crc_table()
    crc_s = np.zeros(nb, np.uint32)
    crc_l = np.zeros(nb, np.uint32)
    for i in range(11):
        crc_l = T[((crc_l >> 16) ^ fr[:, i]) & 0xFF] ^ ((crc_l << 8) & 0xFFFFFF)
        if i == 3:
            crc_s = crc_l.copy()
    crc = np.where(long_, crc_l, crc_s)
    col = np.where(long_, 11, 4)
    rows = np.arange(nb)
    for k in range(3):
        fr[rows, col + k] = (crc >> (16 - 8 * k)) & 0xFF
    fr[~long_, 7:] = 0
    if garble_frac > 0:
        g = np.nonzero(rng.random(nb) < garble_frac)[0]
        nflip = rng.integers(1, 6, g.size)
        for k in range(5):
            sel = g[nflip > k]
            bit = (rng.random(sel.size) * (nbytes[sel] * 8)).astype(np.int64)
            fr[sel, bit // 8] ^= (0x80 >> (bit % 8)).astype(np.uint8)
    return fr, nbytes


def make_scene_device(rate: float, n: int, n_bursts: int, seed: int, device, *, noise_sigma: float = 0.01,
                      snr_db=(6.0, 30.0), df_choices=(11, 17), garble_frac: float = 0.0, fruit: int = 0, out=None):
    """(iq float32 CUDA tensor[2n], list of frame hex strings). Same waveform model as make_scene: box-car integrated
    rectangular chips at fractional start offsets, random carrier phase, uniform starts (overlaps allowed)."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    g = torch.Generator(device=device)
    g.manual_seed(1000 + seed)
    iq = out if out is not None else torch.empty(2 * n, device=device, dtype=torch.float32)
    step = 1 << 26
    for a in range(0, 2 * n, step):
        m = min(step, 2 * n - a)
        torch.randn(m, device=device, generator=g, out=iq[a:a + m])
        iq[a:a + m] *= noise_sigma
    iq2 = iq.view(n, 2)
    span = 240 * spc + 8
    starts = np.sort(rng.uniform(span, n - 2 * span, n_bursts))
    dfs = np.asarray(df_choices)[rng.integers(0, len(df_choices), n_bursts)]
    frames, nbytes = make_frames(dfs, rng, garble_frac)
    snr = rng.uniform(snr_db[0], snr_db[1], n_bursts)
    amp = np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (snr / 10)) if noise_sigma > 0 else np.full(n_bursts, 0.5)
    phase = rng.uniform(0, 2 * np.pi, n_bursts)
    bits = np.unpackbits(frames, axis=1)                                   # [nb, 112]
    valid = np.arange(112)[None, :] < (nbytes * 8)[:, None]
    chips = np.zeros((n_bursts, 240), np.float32)
    chips[:, [0, 2, 7, 9]] = 1.0
    chips[:, 16:240:2] = bits * valid
    chips[:, 17:240:2] = (1 - bits) * valid
    M = int(np.ceil(240 * spc)) + 2
    mgrid = torch.arange(M + 1, device=device, dtype=torch.float64)
    B = max(1, (1 << 24) // (M + 1))
    for a in range(0, n_bursts, B):
        b = min(a + B, n_bursts)
        s = torch.from_numpy(starts[a:b]).to(device)
        n0 = torch.floor(s)
        ch = torch.from_numpy(chips[a:b]).to(device).to(torch.float64)
        cum = torch.cumsum(ch, 1) - ch                                       # exclusive
        t = ((n0 - s)[:, None] + mgrid[None, :]) / spc                       # edges in chips
        t = t.clamp_(0.0, 240.0)
        k = t.floor().clamp_(max=239.0)
        ki = k.to(torch.int64)
        integ = (torch.gather(cum, 1, ki) + torch.gather(ch, 1, ki) * (t - k)) * spc
        cover = integ[:, 1:] - integ[:, :-1]                                 # [b, M]
        w = torch.from_numpy(amp[a:b]).to(device)[:, None] * cover
        ph = torch.from_numpy(phase[a:b]).to(device)[:, None]
        vals = torch.stack((w * torch.cos(ph), w * torch.sin(ph)), 2).to(torch.float32).reshape(-1, 2)
        idx = (n0.to(torch.int64)[:, None] + torch.arange(M, device=device)[None, :]).reshape(-1)
        ok = (idx >= 0) & (idx < n)
        iq2.index_add_(0, idx[ok], vals[ok])
    if fruit:
        s = rng.uniform(0, n - 64 * spc, fruit)
        fa = np.sqrt(2.0 * max(noise_sigma, 1e-3) ** 2 * 10 ** (rng.uniform(10, 30, fruit) / 10))
        ph = rng.uniform(0, 2 * np.pi, fruit)
        off2 = rng.integers(1, 14, fruit) * 1.45 * 2 * spc
        wlen = max(int(round(0.9 * spc)), 1)
        a0 = np.concatenate([s.astype(np.int64), (s + off2).astype(np.int64)])
        idx = torch.from_numpy((a0[:, None] + np.arange(wlen)[None, :]).reshape(-1)).to(device)
        v = np.stack([fa * np.cos(ph), fa * np.sin(ph)], 1).astype(np.float32)
        vals = torch.from_numpy(np.repeat(np.concatenate([v, v]), wlen, axis=0)).to(device)
        ok = (idx >= 0) & (idx < n)
        iq2.index_add_(0, idx[ok], vals[ok])
    hexs = [frames[k, :nbytes[k]].tobytes().hex() for k in range(n_bursts)] if n_bursts <= 4096 else None
    return iq, hexs, (frames, nbytes)


# ---------------------------------------------------------------------------------------------------------
# Fleet scenes: a fixed set of aircraft whose replies carry their addresses the way Mode S does, for the address/parity
# check (rx_path(..., ap_filter=S)). The generators above stay as they are; these are separate functions.
#   DF17      squitter, AA in bytes 1..3, parity = CRC
#   DF11      all-call reply, AA in bytes 1..3, parity = CRC xor II (II = 0, or an interrogator code 1..0x7F)
#   AP        DF0/4/5/16/20/21 reply, parity = CRC xor address (address/parity)
# ---------------------------------------------------------------------------------------------------------
FLEET_AP_DFS = (0, 4, 5, 16, 20, 21)
FLEET_MIX = (0.40, 0.15, 0.10, 0.35)      # DF17, DF11 with II = 0, DF11 with an II code, AP replies


def make_fleet_frames(dfs: np.ndarray, addrs: np.ndarray, codes: np.ndarray, rng: np.random.Generator,
                      garble_frac: float = 0.0):
    """(frames uint8[nb,14], nbytes int[nb]): per burst a frame of format dfs[k] from the aircraft addrs[k]. DF11/DF17
    carry the address in bytes 1..3 and CRC xor codes[k] as parity (codes[k] = 0 for DF17); every other format carries
    random fields and CRC xor address as parity. Short frames are zero beyond byte 7; garble flips 1..5 random bits."""
    nb = dfs.size
    fr, nbytes = make_frames(dfs, rng)                  # random bodies, CRC parity (II = 0)
    sq = (dfs == 11) | (dfs == 17)
    for k in range(3):
        fr[sq, 1 + k] = (addrs[sq] >> (16 - 8 * k)) & 0xFF
    long_ = nbytes == 14
    T = _crc_table()
    crc_s = np.zeros(nb, np.uint32)
    crc_l = np.zeros(nb, np.uint32)
    for i in range(11):                                 # the CRC again over the bodies with their addresses
        crc_l = T[((crc_l >> 16) ^ fr[:, i]) & 0xFF] ^ ((crc_l << 8) & 0xFFFFFF)
        if i == 3:
            crc_s = crc_l.copy()
    par = np.where(long_, crc_l, crc_s) ^ np.where(sq, codes, addrs).astype(np.uint32)
    col = np.where(long_, 11, 4)
    rows = np.arange(nb)
    for k in range(3):
        fr[rows, col + k] = (par >> (16 - 8 * k)) & 0xFF
    if garble_frac > 0:
        g = np.nonzero(rng.random(nb) < garble_frac)[0]
        nflip = rng.integers(1, 6, g.size)
        for k in range(5):
            sel = g[nflip > k]
            bit = (rng.random(sel.size) * (nbytes[sel] * 8)).astype(np.int64)
            fr[sel, bit // 8] ^= (0x80 >> (bit % 8)).astype(np.uint8)
    return fr, nbytes


def fleet_plan(n_aircraft: int, n_bursts: int, rng: np.random.Generator, mix=FLEET_MIX):
    """(dfs, addrs, codes, who) of n_bursts replies from n_aircraft aircraft with distinct random addresses; who[k] is
    the aircraft of burst k (uniform), the formats follow `mix` (see FLEET_MIX)."""
    fleet = rng.choice(np.arange(1, 1 << 24), n_aircraft, replace=False).astype(np.uint32)
    who = rng.integers(0, n_aircraft, n_bursts)
    kind = rng.choice(4, n_bursts, p=np.asarray(mix, np.float64) / np.sum(mix))
    dfs = np.where(kind == 0, 17, np.where(kind == 3, np.asarray(FLEET_AP_DFS)[rng.integers(0, 6, n_bursts)], 11))
    codes = np.where(kind == 2, rng.integers(1, 0x80, n_bursts), 0).astype(np.uint32)
    return dfs, fleet[who], codes, who


def make_fleet_scene(rate: float, n: int, n_aircraft: int, n_bursts: int, seed: int, *, noise_sigma: float = 0.01,
                     snr_db=(8.0, 30.0), mix=FLEET_MIX, garble_frac: float = 0.0, fruit: int = 0,
                     min_gap: float | None = 16.0, quantize_bits: int | None = None) -> Scene:
    """make_scene's waveform model (per burst, on the CPU) for a fleet: n_bursts replies of n_aircraft aircraft
    (fleet_plan, make_fleet_frames), non-overlapping on a jittered grid with min_gap samples between bursts (None:
    uniform starts, overlaps allowed). Each Burst's frame is the frame sent."""
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    iq = (rng.standard_normal((n, 2), dtype=np.float32) * np.float32(noise_sigma))
    c = iq.view(np.complex64).reshape(n)
    span = 240 * spc + 8
    if min_gap is not None:
        slots = int((n - 2 * span) // (span + min_gap))
        pick = np.sort(rng.choice(slots, size=min(n_bursts, slots), replace=False))
        starts = span / 2 + pick * (span + min_gap) + rng.uniform(0, min_gap, pick.size)
    else:
        starts = np.sort(rng.uniform(span, n - 2 * span, n_bursts))
    dfs, addrs, codes, _ = fleet_plan(n_aircraft, starts.size, rng, mix)
    frames, nbytes = make_fleet_frames(dfs, addrs, codes, rng, garble_frac)
    bursts = []
    for k, s in enumerate(starts):
        amp = float(np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (rng.uniform(*snr_db) / 10)))
        b = Burst(float(s), frames[k, :nbytes[k]].tobytes(), amp, float(rng.uniform(0, 2 * np.pi)))
        n0, w = burst_waveform(b, spc)
        lo, hi = max(n0, 0), min(n0 + w.size, n)
        if hi > lo:
            c[lo:hi] += w[lo - n0:hi - n0]
        bursts.append(b)
    for _ in range(fruit):
        s = rng.uniform(0, n - 64 * spc)
        amp = float(np.sqrt(2.0 * max(noise_sigma, 1e-3) ** 2 * 10 ** (rng.uniform(10, 30) / 10)))
        ph = rng.uniform(0, 2 * np.pi)
        for off in (0.0, rng.integers(1, 14) * 1.45 * 2 * spc):
            a0 = int(s + off)
            a1 = min(a0 + max(int(round(0.9 * spc)), 1), n)
            c[a0:a1] += np.complex64(amp * np.exp(1j * ph))
    if quantize_bits is not None:
        q = float(1 << (quantize_bits - 1))
        np.clip(np.rint(iq * q), -q, q - 1, out=iq)
        iq /= np.float32(q)
    return Scene(rate, n, iq.reshape(2 * n), bursts)


def make_fleet_scene_device(rate: float, n: int, n_aircraft: int, n_bursts: int, seed: int, device, *,
                            noise_sigma: float = 0.01, snr_db=(6.0, 30.0), mix=FLEET_MIX, garble_frac: float = 0.0,
                            fruit: int = 0, out=None):
    """The fleet on the device, for long scenes: make_scene_device's renderer (uniform starts, overlaps allowed) over
    the frames of fleet_plan / make_fleet_frames. Returns (iq float32 CUDA tensor[2n], (frames, nbytes, starts, who))."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    g = torch.Generator(device=device)
    g.manual_seed(2000 + seed)
    iq = out if out is not None else torch.empty(2 * n, device=device, dtype=torch.float32)
    step = 1 << 26
    for a in range(0, 2 * n, step):
        m = min(step, 2 * n - a)
        torch.randn(m, device=device, generator=g, out=iq[a:a + m])
        iq[a:a + m] *= noise_sigma
    iq2 = iq.view(n, 2)
    span = 240 * spc + 8
    starts = np.sort(rng.uniform(span, n - 2 * span, n_bursts))
    dfs, addrs, codes, who = fleet_plan(n_aircraft, n_bursts, rng, mix)
    frames, nbytes = make_fleet_frames(dfs, addrs, codes, rng, garble_frac)
    snr = rng.uniform(snr_db[0], snr_db[1], n_bursts)
    amp = np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (snr / 10))
    phase = rng.uniform(0, 2 * np.pi, n_bursts)
    bits = np.unpackbits(frames, axis=1)
    valid = np.arange(112)[None, :] < (nbytes * 8)[:, None]
    chips = np.zeros((n_bursts, 240), np.float32)
    chips[:, [0, 2, 7, 9]] = 1.0
    chips[:, 16:240:2] = bits * valid
    chips[:, 17:240:2] = (1 - bits) * valid
    M = int(np.ceil(240 * spc)) + 2
    mgrid = torch.arange(M + 1, device=device, dtype=torch.float64)
    B = max(1, (1 << 24) // (M + 1))
    for a in range(0, n_bursts, B):
        b = min(a + B, n_bursts)
        s = torch.from_numpy(starts[a:b]).to(device)
        n0 = torch.floor(s)
        ch = torch.from_numpy(chips[a:b]).to(device).to(torch.float64)
        cum = torch.cumsum(ch, 1) - ch
        t = (((n0 - s)[:, None] + mgrid[None, :]) / spc).clamp_(0.0, 240.0)
        k = t.floor().clamp_(max=239.0)
        ki = k.to(torch.int64)
        integ = (torch.gather(cum, 1, ki) + torch.gather(ch, 1, ki) * (t - k)) * spc
        w = torch.from_numpy(amp[a:b]).to(device)[:, None] * (integ[:, 1:] - integ[:, :-1])
        ph = torch.from_numpy(phase[a:b]).to(device)[:, None]
        vals = torch.stack((w * torch.cos(ph), w * torch.sin(ph)), 2).to(torch.float32).reshape(-1, 2)
        idx = (n0.to(torch.int64)[:, None] + torch.arange(M, device=device)[None, :]).reshape(-1)
        ok = (idx >= 0) & (idx < n)
        iq2.index_add_(0, idx[ok], vals[ok])
    if fruit:
        s = rng.uniform(0, n - 64 * spc, fruit)
        fa = np.sqrt(2.0 * max(noise_sigma, 1e-3) ** 2 * 10 ** (rng.uniform(10, 30, fruit) / 10))
        ph = rng.uniform(0, 2 * np.pi, fruit)
        off2 = rng.integers(1, 14, fruit) * 1.45 * 2 * spc
        wlen = max(int(round(0.9 * spc)), 1)
        a0 = np.concatenate([s.astype(np.int64), (s + off2).astype(np.int64)])
        idx = torch.from_numpy((a0[:, None] + np.arange(wlen)[None, :]).reshape(-1)).to(device)
        v = np.stack([fa * np.cos(ph), fa * np.sin(ph)], 1).astype(np.float32)
        vals = torch.from_numpy(np.repeat(np.concatenate([v, v]), wlen, axis=0)).to(device)
        ok = (idx >= 0) & (idx < n)
        iq2.index_add_(0, idx[ok], vals[ok])
    return iq, (frames, nbytes, starts, who)


# ---- several synchronized receivers (multilateration) -------------------------------------------------------------
def ac13(feet: int) -> int:
    """The 13-bit AC field of `feet` (a multiple of 25 from -1000 ft) in the 25-ft Q-bit coding."""
    n = (feet + 1000) // 25
    return ((n >> 5) << 7) | (((n >> 4) & 1) << 5) | 0x10 | (n & 0x0F)


def me_alt12(feet: int) -> int:
    """The 12-bit ME altitude of `feet` (25-ft Q-bit coding)."""
    n = (feet + 1000) // 25
    return ((n >> 4) << 5) | 0x10 | (n & 0x0F)


def mlat_frame(kind: int, addr: int, feet: int, rng: np.random.Generator) -> bytes:
    """DF4 / DF20 altitude reply (AP = CRC ^ address) or DF17 TC 11 airborne position with the ME altitude `feet`."""
    if kind == 17:
        me = (11 << 51) | (me_alt12(feet) << 36) | int(rng.integers(0, 1 << 35))
        body = bytes([(17 << 3) | 5]) + addr.to_bytes(3, "big") + me.to_bytes(7, "big")
        return body + crc24(body).to_bytes(3, "big")
    head = (kind << 27) | (int(rng.integers(0, 2)) << 24) | ac13(feet)       # FS 0/1, DR 0, UM 0
    body = head.to_bytes(4, "big")
    if kind == 20:
        body += bytes(7)                                                     # MB: no register
    return body + (crc24(body) ^ addr).to_bytes(3, "big")


def make_mlat_scenes(rate: float, n: int, stations, aircraft, n_tx: int, seed: int, *, t0=(1_700_000_000, 0.25),
                     noise_sigma: float = 0.01, snr_db: float = 25.0, kinds=(4, 20, 17)):
    """K Scenes of the same n_tx transmissions as K synchronized receivers hear them.

    stations: [(lat, lon, height_m)]; aircraft: [(addr, lat, lon, height_m)] (the altitude code is the height in feet
    rounded to 25 ft). The receivers' sample 0 is at t0 = (secs, frac); transmission j leaves at T_j (spread over the
    recording at least 400 us apart) and starts at (T_j - t0 + |p - s_k| / c) * rate in scene k, each scene with its
    own noise. Returns (scenes, truth): truth[j] = dict(frame, kind, addr, feet, ecef, T) with T in seconds after t0."""
    from .mlat import SPEED_OF_LIGHT, llh2ecef
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    S = [np.array(llh2ecef(*s)) for s in stations]
    span = 240 * spc + 8
    guard = 4e-3 * rate                                                      # the longest baseline delay, with room
    slots = int((n - 2 * guard) // (400e-6 * rate))
    pick = np.sort(rng.choice(slots, size=min(n_tx, slots), replace=False))
    truth = []
    for j in pick:
        addr, lat, lon, h = aircraft[int(rng.integers(0, len(aircraft)))]
        feet = int(round(h / 0.3048 / 25.0)) * 25
        kind = int(kinds[int(rng.integers(0, len(kinds)))])
        p = np.array(llh2ecef(lat, lon, h))
        T = (guard + j * 400e-6 * rate + rng.uniform(0, 100e-6 * rate)) / rate
        truth.append({"frame": mlat_frame(kind, addr, feet, rng), "kind": kind, "addr": addr, "feet": feet, "ecef": p,
                      "T": T})
    scenes = []
    amp = float(np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (snr_db / 10)))
    for k, s in enumerate(S):
        iq = (rng.standard_normal((n, 2), dtype=np.float32) * np.float32(noise_sigma))
        c = iq.view(np.complex64).reshape(n)
        bursts = []
        for tr in truth:
            start = (tr["T"] + float(np.linalg.norm(tr["ecef"] - s)) / SPEED_OF_LIGHT) * rate
            if start + span >= n:
                continue
            b = Burst(float(start), tr["frame"], amp, float(rng.uniform(0, 2 * np.pi)))
            n0, w = burst_waveform(b, spc)
            c[n0:n0 + w.size] += w
            bursts.append(b)
        scenes.append(Scene(rate, n, iq.reshape(2 * n), bursts))
    return scenes, truth


# ---------------------------------------------------------------------------------------------------------
# Mode A/C replies (option "modeac"): F1, the 13 code pulses C1 A1 C2 A2 C4 A4 X B1 D1 B2 D2 B4 D4 at 1.45 us steps,
# F2 at 20.3 us and the optional SPI pulse at 24.65 us, each 0.45 us long. New functions with random streams of their own.
# ---------------------------------------------------------------------------------------------------------
MODEAC_PULSE_US = 0.45


def modeac_waveform(code: int, spi: bool, start: float, amplitude: float, phase: float, spc: float):
    """(first_sample, complex64 samples) of one reply whose F1 leading edge is at fractional sample `start`: box-car
    integrated rectangular pulses, as burst_waveform. `code` is the 13-bit C1..D4 word (bit 12 = C1); X (bit 6) is
    never sent."""
    spu = 2.0 * spc                                   # samples per microsecond
    t = [0.0] + [1.45 * k for k in range(1, 14) if k != 7 and (code >> (13 - k)) & 1] + [20.3]
    if spi:
        t.append(24.65)
    n0 = int(np.floor(start))
    n1 = int(np.ceil(start + (24.65 + MODEAC_PULSE_US) * spu)) + 1
    lo = np.arange(n0, n1, dtype=np.float64) - start
    cover = np.zeros(lo.size)
    for p in t:                                       # overlap of [lo, lo + 1) with [p, p + width) in samples
        a, b = p * spu, (p + MODEAC_PULSE_US) * spu
        cover += np.clip(np.minimum(lo + 1, b) - np.maximum(lo, a), 0.0, None)
    return n0, (amplitude * cover * np.exp(1j * phase)).astype(np.complex64)


@dataclasses.dataclass
class ModeacReply:
    start: float          # fractional sample index of the F1 leading edge
    code: int
    spi: bool
    amplitude: float
    phase: float


def make_modeac_scene(rate: float, n: int, n_replies: int, seed: int, *, noise_sigma: float = 0.01,
                      snr_db=(15.0, 30.0), n_bursts: int = 0, codes=None, spis=None, gap_us: float = 30.0):
    """Complex Gaussian noise + `n_replies` Mode A/C replies + `n_bursts` Mode S bursts, none overlapping another: each
    goes into its own slot of a jittered grid (a reply's slot is 26 us + gap, a burst's 120 us + gap, in random order).
    codes / spis: the replies' codes and SPI flags (default random, X = 0). Returns (Scene, [ModeacReply]) with the
    replies in start order; Scene.bursts holds the Mode S bursts."""
    rng = np.random.Generator(np.random.PCG64(seed))
    spc = rate / 2e6
    spu = 2.0 * spc
    iq = (rng.standard_normal((n, 2), dtype=np.float32) * np.float32(noise_sigma))
    c = iq.view(np.complex64).reshape(n)
    kinds = np.array([0] * n_replies + [1] * n_bursts)
    rng.shuffle(kinds)
    lens = np.where(kinds == 0, 26.0, 120.0) * spu + gap_us * spu
    if lens.sum() > n - 64 * spu:
        raise ValueError("make_modeac_scene: %d replies and %d bursts do not fit in %d samples" % (n_replies, n_bursts, n))
    slack = (n - 64 * spu - lens.sum()) / max(kinds.size, 1)
    if codes is None:
        codes = rng.integers(0, 1 << 13, n_replies) & ~0x40
    if spis is None:
        spis = rng.random(n_replies) < 0.5
    pos = 32 * spu
    replies, bursts, r = [], [], 0
    for k, kind in enumerate(kinds):
        s = pos + rng.uniform(0, slack)
        amp = float(np.sqrt(2.0 * noise_sigma ** 2 * 10 ** (rng.uniform(*snr_db) / 10)))
        ph = float(rng.uniform(0, 2 * np.pi))
        if kind == 0:
            rep = ModeacReply(float(s), int(codes[r]) & ~0x40, bool(spis[r]), amp, ph)
            n0, w = modeac_waveform(rep.code, rep.spi, rep.start, amp, ph, spc)
            replies.append(rep)
            r += 1
        else:
            b = Burst(float(s), make_frame(int(rng.choice((11, 17))), rng), amp, ph)
            n0, w = burst_waveform(b, spc)
            bursts.append(b)
        c[n0:n0 + w.size] += w[:max(0, min(w.size, n - n0))]
        pos += lens[k] + slack
    return Scene(rate, n, iq.reshape(2 * n), bursts), replies
