// TEST HARNESS (not a product path): the decoder's kernel source under the SIMT emulator, as tests/simt/decode_emul.cc
// runs it, plus an entry point that also runs the local CPR stage (option "local_cpr"). tests/test_local_cpr_simt.py
// builds this file with plain g++.
#include "decode_emul.cc"

// Option "local_cpr": the same decode followed by the local CPR stage through its own launcher amb_local_launch
// (amb_decode_local.cuh), as amb_decode_frames runs it with the option on. The table of reference positions is indexed
// by ICAO; the test keeps the addresses below 2^log2_slots. S = 0 runs the plain decode (the stage is off).
struct EmulLocal {
    Emul* base;
    std::vector<AmbRefPos> ltable;
};

extern "C" void* emul_local_new(int log2_slots)
{
    EmulLocal* e = new EmulLocal();
    e->base = static_cast<Emul*>(emul_new(log2_slots));
    e->ltable.resize((size_t)1 << log2_slots);
    memset(e->ltable.data(), 0xFF, e->ltable.size() * sizeof(AmbRefPos));
    return e;
}
extern "C" void emul_local_free(void* h)
{
    EmulLocal* e = static_cast<EmulLocal*>(h);
    emul_free(e->base);
    delete e;
}

extern "C" int emul_decode_local(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int S, amb_fields* out)
{
    EmulLocal* e = static_cast<EmulLocal*>(h);
    Emul* b = e->base;
    if (n <= 0) return 0;
    std::vector<AmbPosRec> pos(n), lpos(n);
    std::vector<AmbPair> pair(n);
    const int nb = (n + 127) / 128;
    simt_launch(nb, 128, [&] { amb_fields_kernel(frames, n, out, pos.data(), pair.data()); });
    for (int k = 0; k < n; k++)
        if (pos[k].key != AMB_NO_KEY && (((size_t)pos[k].key << 1) | 1u) >= b->table.size()) return -1;   // test table too small
    cudaError_t err = cudaSuccess;
    if (amb_v3_launch(&b->v3, pos.data(), n, b->table.data(), pair.data(), nullptr, &err) < 0) return -2;
    simt_launch(nb, 128, [&] { amb_resolve_kernel(out, pos.data(), pair.data(), n, have_loc, lat, lon, b->T); });
    if (S > 0 && amb_local_launch(&b->v3, pos.data(), lpos.data(), n, out, e->ltable.data(), S, have_loc, lat, lon, b->T,
                                  nullptr, &err) < 0) return -3;
    return 0;
}
