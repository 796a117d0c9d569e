// TEST HARNESS (not a product path): runs the decoder's kernel source - gr_air_modes_b200/csrc/amb_decode_kernels.cuh
// and amb_decode_v3.cuh - on the host under tests/simt/simt_emul.h, in the launch sequence of amb_decode_frames
// (amb_decode.cu): the fields kernel, the pairing stage through its own launcher amb_v3_launch, the resolve kernel.
// tests/test_decode_simt.py compares the result with the sequential host shim and the oracle. Built by the test with
// plain g++.
#include "simt_emul.h"

#include "../../gr_air_modes_b200/csrc/amb_decode_kernels.cuh"

#include <vector>

struct Emul {
    std::vector<AmbCprSlot> table;
    double T[AMB_NL_MAX];
    AmbV3Bufs v3;                                       // kept across calls, like the decoder's
};

extern "C" void* emul_new(int log2_slots)
{
    Emul* e = new Emul();
    e->table.resize((size_t)1 << log2_slots);
    memset(e->table.data(), 0xFF, e->table.size() * sizeof(AmbCprSlot));
    amb_build_nl_table(e->T);
    return e;
}
extern "C" void emul_free(void* h)
{
    Emul* e = static_cast<Emul*>(h);
    amb_v3_free(&e->v3);
    delete e;
}

extern "C" int emul_decode(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, amb_fields* out)
{
    Emul* e = static_cast<Emul*>(h);
    if (n <= 0) return 0;
    std::vector<AmbPosRec> pos(n);
    std::vector<AmbPair> pair(n);
    const int nb = (n + 127) / 128;
    simt_launch(nb, 128, [&] { amb_fields_kernel(frames, n, out, pos.data(), pair.data()); });
    for (int k = 0; k < n; k++)
        if (pos[k].key != AMB_NO_KEY && (((size_t)pos[k].key << 1) | 1u) >= e->table.size()) return -1;   // test table too small
    cudaError_t err = cudaSuccess;
    if (amb_v3_launch(&e->v3, pos.data(), n, e->table.data(), pair.data(), nullptr, &err) < 0) return -2;
    simt_launch(nb, 128, [&] { amb_resolve_kernel(out, pos.data(), pair.data(), n, have_loc, lat, lon, e->T); });
    return 0;
}
