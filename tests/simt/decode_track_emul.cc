// TEST HARNESS (not a product path): the decoder's kernel source under the SIMT emulator, as tests/simt/decode_emul.cc
// runs it, plus entry points that also run the per-aircraft table (option "track", amb_decode_track.cuh) and read it
// out, through the stage's own launchers. tests/test_track_simt.py builds this file with plain g++.
#include "decode_emul.cc"

#include <sys/mman.h>

#include <algorithm>

// The pairing table and the local stage's table are indexed by ICAO below 2^log2_slots (the test keeps the addresses
// small); the aircraft rows span all 2^24 addresses like the decoder's, in a reserve-only mapping (only the pages of
// rows that are written get memory).
struct EmulTrack {
    Emul* base;
    std::vector<AmbRefPos> ltable;
    amb_aircraft* rows;
    std::vector<unsigned> occ;
    AmbTrackClock clk;
    std::vector<uint32_t> snap;
};

static const size_t kRowBytes = (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft);

extern "C" void emul_track_reset(void* h)
{
    EmulTrack* e = static_cast<EmulTrack*>(h);
    std::fill(e->occ.begin(), e->occ.end(), 0u);
    e->clk.last_t = NAN; e->clk.last_k = 0; e->clk.pad_ = 0;
}

extern "C" void* emul_track_new(int log2_slots)
{
    EmulTrack* e = new EmulTrack();
    e->base = static_cast<Emul*>(emul_new(log2_slots));
    e->ltable.resize((size_t)1 << log2_slots);
    memset(e->ltable.data(), 0xFF, e->ltable.size() * sizeof(AmbRefPos));
    void* p = mmap(nullptr, kRowBytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) { emul_free(e->base); delete e; return nullptr; }
    memset(p, 0xA5, 4096 * 4);                          // rows are never cleared: the first ones start as garbage
    e->rows = static_cast<amb_aircraft*>(p);
    e->occ.assign(AMB_TRACK_WORDS, 0u);
    e->snap.assign(2 * AMB_TRACK_WORDS / AMB_SNAP_WORDS + 1, 0u);
    emul_track_reset(e);
    return e;
}

extern "C" void emul_track_free(void* h)
{
    EmulTrack* e = static_cast<EmulTrack*>(h);
    munmap(e->rows, kRowBytes);
    emul_free(e->base);
    delete e;
}

// One decode as amb_decode_frames runs it: fields, pairing, resolve, the local stage (local_S > 0), the track stage
// (track_S > 0).
extern "C" int emul_decode_track(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int local_S,
                                 int track_S, amb_fields* out)
{
    EmulTrack* e = static_cast<EmulTrack*>(h);
    Emul* b = e->base;
    if (n <= 0) return 0;
    std::vector<AmbPosRec> pos(n), keys(n);
    std::vector<AmbPair> pair(n);
    const int nb = (n + 127) / 128;
    simt_launch(nb, 128, [&] { amb_fields_kernel(frames, n, out, pos.data(), pair.data()); });
    for (int k = 0; k < n; k++)
        if (pos[k].key != AMB_NO_KEY && (((size_t)pos[k].key << 1) | 1u) >= b->table.size()) return -1;   // test table too small
    cudaError_t err = cudaSuccess;
    if (amb_v3_launch(&b->v3, pos.data(), n, b->table.data(), pair.data(), nullptr, &err) < 0) return -2;
    simt_launch(nb, 128, [&] { amb_resolve_kernel(out, pos.data(), pair.data(), n, have_loc, lat, lon, b->T); });
    if (local_S > 0 && amb_local_launch(&b->v3, pos.data(), keys.data(), n, out, e->ltable.data(), local_S, have_loc, lat, lon,
                                        b->T, nullptr, &err) < 0) return -3;
    if (track_S > 0 && amb_track_launch(&b->v3, frames, out, pos.data(), keys.data(), n, e->rows, e->occ.data(), &e->clk,
                                        track_S, nullptr, &err) < 0) return -4;
    return 0;
}

// amb_decoder_aircraft over the first `words` bitmap words (a multiple of AMB_SNAP_WORDS): out == NULL returns the count.
extern "C" int emul_track_snapshot(void* h, double now, int S, unsigned words, amb_aircraft* out, int max)
{
    EmulTrack* e = static_cast<EmulTrack*>(h);
    const unsigned nb = words / AMB_SNAP_WORDS;
    uint32_t* off = e->snap.data() + nb;
    cudaError_t err = cudaSuccess;
    if (amb_snap_count_launch(e->occ.data(), e->rows, &e->clk, now, S, words, e->snap.data(), off, nullptr, &err) < 0) return -1;
    const int total = (int)off[nb];
    if (!out) return total;
    if (total > max) return -5;
    if (total && amb_snap_gather_launch(e->occ.data(), e->rows, &e->clk, now, S, words, off, out, nullptr, &err) < 0) return -1;
    return total;
}
