// TEST HARNESS, not a product path: compiles the product's per-message decode functions
// (gr_air_modes_b200/csrc/amb_decode_core.h - the __host__ __device__ code the CUDA kernels call) for the host, so
// that tests/test_decode_cpu.py can check that arithmetic against the reference's golden without a GPU. The
// kernels of amb_decode.cu are replayed one message at a time; the report table is a std::unordered_map here
// (direct-mapped HBM table + warp bookkeeping on the device - that part is only exercised by the GPU tests).
// Built by the test into a temporary directory with plain g++; never shipped, never loaded by the package.
#include <unordered_map>
#include <vector>

#include "../gr_air_modes_b200/csrc/amb_decode_core.h"

struct Slot { uint32_t lat, lon; double t; };

extern "C" int shim_decode(const amb_frame* frames, int n, int have_loc, double lat, double lon, amb_fields* out)
{
    double T[AMB_NL_MAX];
    amb_build_nl_table(T);
    std::unordered_map<uint64_t, Slot> table;
    for (int k = 0; k < n; k++) {
        AmbPosRec me;
        amb_decode_fields(frames[k], &out[k], &me);                 // amb_fields_kernel
        if (me.key == AMB_NO_KEY) continue;
        const uint64_t slot_other = ((uint64_t)me.key << 1) | (me.fmt ? 0u : 1u);
        const uint64_t slot_mine = ((uint64_t)me.key << 1) | (me.fmt ? 1u : 0u);
        auto it = table.find(slot_other);                           // amb_v3_pair, one lane at a time
        const bool have = it != table.end();
        const AmbPair pr = amb_make_pair(me, have, have ? it->second.lat : 0, have ? it->second.lon : 0, have ? it->second.t : 0.0);
        table[slot_mine] = Slot{me.lat, me.lon, me.t};
        amb_resolve_position(&out[k], pr, have_loc, lat, lon, T);  // amb_resolve_kernel
    }
    return 0;
}

extern "C" int shim_nl(double lat)
{
    double T[AMB_NL_MAX];
    amb_build_nl_table(T);
    return amb_nl(lat, T);
}

extern "C" int shim_sizeof_fields(void) { return (int)sizeof(amb_fields); }

// Stateful variant (one decoder instance whose report table lives across calls), for the cpr_decoder drop-in test.
struct ShimState { std::unordered_map<uint64_t, Slot> table; double T[AMB_NL_MAX]; };
extern "C" void* shim_new(void) { ShimState* s = new ShimState(); amb_build_nl_table(s->T); return s; }
extern "C" int shim_step(void* p, const amb_frame* frames, int n, int have_loc, double lat, double lon, amb_fields* out)
{
    ShimState* s = static_cast<ShimState*>(p);
    for (int k = 0; k < n; k++) {
        AmbPosRec me;
        amb_decode_fields(frames[k], &out[k], &me);
        if (me.key == AMB_NO_KEY) continue;
        const uint64_t slot_other = ((uint64_t)me.key << 1) | (me.fmt ? 0u : 1u);
        const uint64_t slot_mine = ((uint64_t)me.key << 1) | (me.fmt ? 1u : 0u);
        auto it = s->table.find(slot_other);
        const bool have = it != s->table.end();
        const AmbPair pr = amb_make_pair(me, have, have ? it->second.lat : 0, have ? it->second.lon : 0, have ? it->second.t : 0.0);
        s->table[slot_mine] = Slot{me.lat, me.lon, me.t};
        amb_resolve_position(&out[k], pr, have_loc, lat, lon, s->T);
    }
    return 0;
}
