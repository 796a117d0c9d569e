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

extern "C" void shim_nl_table(double* T) { amb_build_nl_table(T); }

// Every latitude of one CPR lattice at which the decoder evaluates nl(): d * (j + y / 2^17) for j = j_lo..j_hi and
// y = 0..2^17-1 with d = span / div, the expression of amb_cpr_global (:301-302, j there is pymod(j, 60 or 59)) and of
// amb_cpr_local (:377), then `post`: 0 none, 1 the global decode's "> 270 -> -360" (:303-304), 2 the surface decode's
// -90 for a receiver south of the equator (:307). amb_nl() through the table against cpr.py:48-51 evaluated directly
// (1 at |lat| >= 87, else amb_nl_formula). The first max_bad disagreeing latitudes go to bad[], their count to *n_bad;
// near[2k] / near[2k+1] receive the lattice latitude nearest below / at or above T[k] (k = 3..T[0]), in |lat|.
// Returns the number of latitudes checked.
extern "C" long long shim_nl_lattice(double span, int div, long long j_lo, long long j_hi, int post, double* bad,
                                     int max_bad, long long* n_bad, double* near)
{
    double T[AMB_NL_MAX];
    amb_build_nl_table(T);
    const int kmax = (int)T[0];
    for (int k = 0; k < 2 * AMB_NL_MAX; k++) near[k] = NAN;
    const double d = span / div;
    long long n = 0;
    *n_bad = 0;
    for (long long j = j_lo; j <= j_hi; j++)
        for (uint32_t y = 0; y < 131072; y++) {
            double lat = d * ((double)j + (double)y / 131072);
            if (post == 1) { if (lat > 270.0) lat -= 360.0; }
            else if (post == 2) lat -= 90;
            const double a = fabs(lat);
            const int want = a >= 87.0 ? 1 : (int)amb_nl_formula(lat);
            const int got = amb_nl(lat, T);
            if (got != want) {
                if (*n_bad < max_bad) bad[*n_bad] = lat;
                ++*n_bad;
            }
            // T[got] is the nearest transition above |lat|, T[got + 1] the nearest at or below it
            for (int k = got; k <= got + 1; k++) {
                if (k < 3 || k > kmax || a >= 87.0) continue;
                double* s = &near[2 * k + (a < T[k] ? 0 : 1)];
                if (*s != *s || fabs(a - T[k]) < fabs(fabs(*s) - T[k])) *s = lat;
            }
            n++;
        }
    return n;
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
