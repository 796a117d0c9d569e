// TEST HARNESS (not a product path): the op-status harness tests/simt/decode_opstatus_emul.cc (and through it the shared
// decoder harness tests/simt/decode_emul.cc), unchanged, plus the option "track_ext". emul_decode_ext sets the
// extension's S2, rows and bitmap on the state and decodes through emul_decode_all - the decoder's own
// amb_decode_launch, with every stage whose S is > 0. emul_snapshot_ext runs amb_decoder_aircraft_ext's kernels. The
// rows span all 2^24 addresses like the decoder's, in a reserve-only mapping allocated at the first decode with the
// option on (only the pages of rows that are written get memory). tests/test_track_ext_simt.py builds it with plain g++
// (tests/emul_build.py).
#include "decode_opstatus_emul.cc"

static const size_t kExtBytes = (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft_ext);

struct EmulExt {
    std::vector<unsigned> occ;
    amb_aircraft_ext* rows = nullptr;
};
static std::map<void*, EmulExt> g_ext;   // the extension of each handle

// amb_decode_frames with every option; returns what emul_decode returns
extern "C" int emul_decode_ext(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int local_S,
                               int commb_S, int opstatus_S, int track_S, int ext_S, amb_fields* out)
{
    Emul* e = static_cast<Emul*>(h);
    if (track_S > 0 && ext_S > 0 && !e->st.xrows) {
        EmulExt& x = g_ext[h];
        void* p = mmap(nullptr, kExtBytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (p == MAP_FAILED) return -3;
        memset(p, 0xA5, 4096 * 4);                      // rows are never cleared: the first ones start as garbage
        x.rows = static_cast<amb_aircraft_ext*>(p);
        x.occ.assign(AMB_TRACK_WORDS, 0u);
        e->st.xrows = x.rows;
        e->st.xocc = x.occ.data();
    }
    e->st.track_ext = ext_S;
    return emul_decode_all(h, frames, n, have_loc, lat, lon, local_S, commb_S, opstatus_S, track_S, out);
}

// amb_decoder_reset: the shared harness's reset, and the extension's bitmap cleared (its rows stay)
extern "C" void emul_reset_ext(void* h)
{
    emul_reset(h);
    Emul* e = static_cast<Emul*>(h);
    if (e->st.xocc) std::fill(g_ext[h].occ.begin(), g_ext[h].occ.end(), 0u);
}

// amb_decoder_aircraft_ext over the first `words` bitmap words (a multiple of AMB_SNAP_WORDS): out == NULL returns the
// count, too small a `max` -5.
extern "C" int emul_snapshot_ext(void* h, double now, int S, int S2, unsigned words, amb_aircraft* out,
                                 amb_aircraft_ext* ext, int max)
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
    if (total && amb_snap_gather_ext_launch(e->st.tocc, e->st.trows, &e->clk, now, S, words, off, out, e->st.xocc,
                                            e->st.xrows, S2, ext, nullptr, &err) < 0)
        return -1;
    return total;
}

extern "C" void emul_free_ext(void* h)
{
    auto it = g_ext.find(h);
    if (it != g_ext.end()) {
        if (it->second.rows) munmap(it->second.rows, kExtBytes);
        g_ext.erase(it);
    }
    emul_free_all(h);
}
