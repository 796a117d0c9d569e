// TEST HARNESS (not a product path): the track-extension harness tests/simt/decode_track_ext_emul.cc (and through it
// the op-status and the shared decoder harness), unchanged, plus the option "sbs1". emul_decode_sbs1 sets the SBS-1
// stage's option, time zone, id table, counter and scratch on the state, decodes through emul_decode_ext - the
// decoder's own amb_decode_launch, with every stage whose option is on - and copies the call's packed lines out, as
// amb_decoder_sbs1 does. The id table spans all 2^24 addresses like the decoder's, in a reserve-only zero mapping.
// tests/test_sbs1_simt.py builds it with plain g++ (tests/emul_build.py).
#include "decode_track_ext_emul.cc"

static const size_t kIdBytes = (size_t)AMB_SBS1_SLOTS * sizeof(unsigned long long);

struct EmulSbs1 {
    AmbSbs1Ctr ctr = {0ull, 0ull, 0u, 0u};
    unsigned long long* table = nullptr;
    std::vector<unsigned long long> src, gid, flag, boff;
    std::vector<char> slots, text;
    std::vector<uint32_t> len, bsum;
};
static std::map<void*, EmulSbs1> g_sbs1;   // the SBS-1 stage of each handle

// amb_decode_frames with every option, then amb_decoder_sbs1: returns what emul_decode returns, or -5 when the text
// does not fit `cap` (*n_bytes = its length either way)
extern "C" int emul_decode_sbs1(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon,
                                int local_S, int commb_S, int opstatus_S, int track_S, int ext_S, int sbs1, int tz,
                                amb_fields* out, char* text, size_t cap, size_t* n_bytes)
{
    Emul* e = static_cast<Emul*>(h);
    *n_bytes = 0;
    if (sbs1) {
        EmulSbs1& x = g_sbs1[h];
        if (!x.table) {
            void* p = mmap(nullptr, kIdBytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
            if (p == MAP_FAILED) return -3;
            x.table = static_cast<unsigned long long*>(p);
        }
        const size_t nn = (size_t)(n > 0 ? n : 1), nb = (nn + 127) / 128;
        x.src.assign(nn, 0xDEADBEEFull); x.gid.assign(nn, 0xDEADBEEFull);
        x.flag.assign((nn + AMB_SBS1_CHUNK - 1) / AMB_SBS1_CHUNK, 0xDEADBEEFull);
        x.slots.assign(nn * AMB_SBS1_STRIDE, '?'); x.text.assign(nn * AMB_SBS1_STRIDE, '?');
        x.len.assign(nn, 7u); x.bsum.assign(nb, 7u); x.boff.assign(nb + 1, 7ull);
        AmbSbs1Bufs& b = e->st.sb;
        b.src = x.src.data(); b.gid = x.gid.data(); b.flag = x.flag.data(); b.slots = x.slots.data();
        b.len = x.len.data(); b.bsum = x.bsum.data(); b.boff = x.boff.data(); b.text = x.text.data();
        e->st.stable = x.table;
        e->st.sctr = &x.ctr;
    }
    e->st.sbs1 = sbs1;
    e->st.sbs1_tz = tz;
    const int rc = emul_decode_ext(h, frames, n, have_loc, lat, lon, local_S, commb_S, opstatus_S, track_S, ext_S, out);
    if (rc != 0 || !sbs1 || n <= 0) return rc;
    const EmulSbs1& x = g_sbs1[h];
    const size_t total = (size_t)x.boff[(n + 127) / 128];
    *n_bytes = total;
    if (total > cap) return -5;
    memcpy(text, x.text.data(), total);
    return 0;
}

// the ids of the last call's published records, in stream order (count returned)
extern "C" int emul_sbs1_ids(void* h, const amb_fields* recs, int n, unsigned long long* ids)
{
    const EmulSbs1& x = g_sbs1[h];
    int m = 0;
    for (int k = 0; k < n; k++)
        if (amb_sbs1_published(&recs[k])) ids[m++] = x.gid[k] - x.ctr.base;
    return m;
}

// amb_decoder_reset: the track-extension harness's reset, and base = G
extern "C" void emul_reset_sbs1(void* h)
{
    emul_reset_ext(h);
    auto it = g_sbs1.find(h);
    if (it != g_sbs1.end()) it->second.ctr.base = it->second.ctr.G;
}

extern "C" void emul_free_sbs1(void* h)
{
    auto it = g_sbs1.find(h);
    if (it != g_sbs1.end()) {
        if (it->second.table) munmap(it->second.table, kIdBytes);
        g_sbs1.erase(it);
    }
    emul_free_ext(h);
}
