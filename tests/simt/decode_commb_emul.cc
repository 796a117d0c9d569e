// TEST HARNESS (not a product path): the decoder's kernel source under the SIMT emulator, as tests/simt/decode_emul.cc
// runs it, plus an entry point that also runs the Comm-B stage (option "commb", amb_decode_commb.cuh) through its own
// launcher, after the local CPR stage when that is on. tests/test_commb_simt.py builds this file with plain g++.
#include "decode_emul.cc"

#include <algorithm>

// The pairing table and the local stage's table are indexed by ICAO below 2^log2_slots (the test keeps the position
// squitters' addresses small); the velocity table spans all 2^24 addresses like the decoder's, since a DF20/21 record's
// address is its AP syndrome.
struct EmulCommb {
    Emul* base;
    std::vector<AmbRefPos> ltable;
    std::vector<AmbCommbRef> ctable;
};

extern "C" void emul_commb_reset(void* h)
{
    EmulCommb* e = static_cast<EmulCommb*>(h);
    memset(e->ctable.data(), 0xFF, e->ctable.size() * sizeof(AmbCommbRef));
}

extern "C" void* emul_commb_new(int log2_slots)
{
    EmulCommb* e = new EmulCommb();
    e->base = static_cast<Emul*>(emul_new(log2_slots));
    e->ltable.resize((size_t)1 << log2_slots);
    memset(e->ltable.data(), 0xFF, e->ltable.size() * sizeof(AmbRefPos));
    e->ctable.resize((size_t)AMB_COMMB_SLOTS);
    emul_commb_reset(e);
    return e;
}

extern "C" void emul_commb_free(void* h)
{
    EmulCommb* e = static_cast<EmulCommb*>(h);
    emul_free(e->base);
    delete e;
}

// One decode as amb_decode_frames runs it: fields, pairing, resolve, the local stage (local_S > 0), the Comm-B stage
// (commb_S > 0).
extern "C" int emul_decode_commb(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int local_S,
                                 int commb_S, amb_fields* out)
{
    EmulCommb* e = static_cast<EmulCommb*>(h);
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
    if (commb_S > 0 && amb_commb_launch(&b->v3, frames, out, pos.data(), keys.data(), n, e->ctable.data(), commb_S, nullptr,
                                        &err) < 0) return -4;
    return 0;
}
