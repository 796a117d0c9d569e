// TEST HARNESS (not a product path): runs the decoder's kernel source - gr_air_modes_b200/csrc/amb_decode_kernels.cuh
// and the stage headers it includes - on the host under tests/simt/simt_emul.h, through the decoder's own launch
// sequence amb_decode_launch: fields, pairing, resolve, and the local CPR, Comm-B and track stages whose S is > 0.
// tests/test_decode_simt.py, test_local_cpr_simt.py, test_commb_simt.py and test_track_simt.py build it with plain g++
// (tests/emul_build.py).
#include "simt_emul.h"

#include "../../gr_air_modes_b200/csrc/amb_decode_kernels.cuh"

#include <sys/mman.h>

#include <algorithm>
#include <vector>

// The pairing table and the local stage's table are indexed by ICAO below 2^log2_slots (the tests keep the position
// squitters' addresses small). The velocity table and the aircraft rows span all 2^24 addresses like the decoder's,
// since a DF20/21 record's address is its AP syndrome; they are allocated at the first decode with their stage on, the
// rows in a reserve-only mapping (only the pages of rows that are written get memory).
struct Emul {
    AmbDecodeState st;                                  // kept across calls, like the decoder's
    std::vector<AmbCprSlot> table;
    double T[AMB_NL_MAX];
    std::vector<AmbRefPos> ltable;
    std::vector<AmbCommbRef> ctable;
    std::vector<unsigned> occ;
    AmbTrackClock clk;
    std::vector<uint32_t> snap;
    std::vector<AmbPosRec> pos, keys;
    std::vector<AmbPair> pair;
};

static const size_t kRowBytes = (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft);

// amb_decoder_reset: every table empty again, the aircraft rows stay (a row whose bit is clear is never read)
extern "C" void emul_reset(void* h)
{
    Emul* e = static_cast<Emul*>(h);
    memset(e->table.data(), 0xFF, e->table.size() * sizeof(AmbCprSlot));
    memset(e->ltable.data(), 0xFF, e->ltable.size() * sizeof(AmbRefPos));
    if (!e->ctable.empty()) memset(e->ctable.data(), 0xFF, e->ctable.size() * sizeof(AmbCommbRef));
    std::fill(e->occ.begin(), e->occ.end(), 0u);
    e->clk.last_t = NAN; e->clk.last_k = 0; e->clk.pad_ = 0;
}

extern "C" void* emul_new(int log2_slots)
{
    Emul* e = new Emul();
    e->table.resize((size_t)1 << log2_slots);
    e->ltable.resize((size_t)1 << log2_slots);
    amb_build_nl_table(e->T);
    e->st.table = e->table.data();
    e->st.nl_T = e->T;
    e->st.ltable = e->ltable.data();
    e->st.tclk = &e->clk;
    emul_reset(e);
    return e;
}

extern "C" void emul_free(void* h)
{
    Emul* e = static_cast<Emul*>(h);
    if (e->st.trows) munmap(e->st.trows, kRowBytes);
    amb_v3_free(&e->st.v3);
    delete e;
}

// amb_decode_frames: returns 0, or -1 when a position squitter's address does not fit the test's tables
extern "C" int emul_decode(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int local_S,
                           int commb_S, int track_S, amb_fields* out)
{
    Emul* e = static_cast<Emul*>(h);
    if (n <= 0) return 0;
    for (int k = 0; k < n; k++) {
        amb_fields r; AmbPosRec p;
        amb_decode_fields(frames[k], &r, &p);
        if (p.key != AMB_NO_KEY && (((size_t)p.key << 1) | 1u) >= e->table.size()) return -1;   // test table too small
    }
    if (commb_S > 0 && e->ctable.empty()) {
        e->ctable.resize((size_t)AMB_COMMB_SLOTS);
        memset(e->ctable.data(), 0xFF, e->ctable.size() * sizeof(AmbCommbRef));
        e->st.ctable = e->ctable.data();
    }
    if (track_S > 0 && !e->st.trows) {
        void* p = mmap(nullptr, kRowBytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (p == MAP_FAILED) return -3;
        memset(p, 0xA5, 4096 * 4);                      // rows are never cleared: the first ones start as garbage
        e->st.trows = static_cast<amb_aircraft*>(p);
        e->occ.assign(AMB_TRACK_WORDS, 0u);
        e->st.tocc = e->occ.data();
        e->snap.assign(2 * AMB_TRACK_WORDS / AMB_SNAP_WORDS + 1, 0u);
    }
    e->pos.resize(n); e->pair.resize(n); e->keys.resize(n);
    e->st.pos = e->pos.data(); e->st.pair = e->pair.data(); e->st.keys = e->keys.data();
    e->st.have_loc = have_loc; e->st.lat = lat; e->st.lon = lon;
    e->st.local_cpr = local_S; e->st.commb = commb_S; e->st.track = track_S;
    cudaError_t err = cudaSuccess;
    return amb_decode_launch(&e->st, frames, n, out, nullptr, &err) < 0 ? -2 : 0;
}

// amb_decoder_aircraft over the first `words` bitmap words (a multiple of AMB_SNAP_WORDS): out == NULL returns the count.
extern "C" int emul_snapshot(void* h, double now, int S, unsigned words, amb_aircraft* out, int max)
{
    Emul* e = static_cast<Emul*>(h);
    if (!e->st.trows) return 0;                         // nothing decoded with the track stage on yet
    const unsigned nb = words / AMB_SNAP_WORDS;
    uint32_t* off = e->snap.data() + nb;
    cudaError_t err = cudaSuccess;
    if (amb_snap_count_launch(e->st.tocc, e->st.trows, &e->clk, now, S, words, e->snap.data(), off, nullptr, &err) < 0)
        return -1;
    const int total = (int)off[nb];
    if (!out) return total;
    if (total > max) return -5;
    if (total && amb_snap_gather_launch(e->st.tocc, e->st.trows, &e->clk, now, S, words, off, out, nullptr, &err) < 0)
        return -1;
    return total;
}
