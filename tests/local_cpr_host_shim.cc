// TEST HARNESS, not a product path: the host shim of tests/decode_host_shim.cc (the product's per-message decode
// functions compiled for the host) plus the entry points of the decoder option "local_cpr", for
// tests/test_local_cpr_cpu.py and tests/test_local_cpr_simt.py. Built by those tests with plain g++.
#include "decode_host_shim.cc"

// Option "local_cpr": cpr_resolve_local (amb_cpr_local) for one case, and the stateful decode followed by the local
// stage one message at a time (amb_local_step against a map of reference positions per ICAO).
extern "C" void shim_cpr_local(double ref_lat, double ref_lon, uint32_t enclat, uint32_t enclon, int ctype, int surface, double* out2)
{
    double T[AMB_NL_MAX];
    amb_build_nl_table(T);
    amb_cpr_local(ref_lat, ref_lon, enclat, enclon, ctype, surface, T, &out2[0], &out2[1]);
}

struct ShimLocal { ShimState* base; std::unordered_map<uint32_t, AmbRefPos> refs; };
extern "C" void* shim_local_new(void) { ShimLocal* s = new ShimLocal(); s->base = static_cast<ShimState*>(shim_new()); return s; }
extern "C" int shim_local_step(void* p, const amb_frame* frames, int n, int have_loc, double lat, double lon, int S, amb_fields* out)
{
    ShimLocal* s = static_cast<ShimLocal*>(p);
    shim_step(s->base, frames, n, have_loc, lat, lon, out);
    if (S <= 0) return 0;
    for (int k = 0; k < n; k++) {
        AmbPosRec me;
        amb_fields scratch;
        amb_decode_fields(frames[k], &scratch, &me);
        if (me.key == AMB_NO_KEY) continue;
        auto it = s->refs.find(me.key >> 1);
        AmbRefPos ref;
        if (it != s->refs.end()) ref = it->second;
        else ref.lat = ref.lon = ref.t = NAN;
        amb_local_step(&out[k], me.t, &ref, S, have_loc, lat, lon, s->base->T);
        s->refs[me.key >> 1] = ref;
    }
    return 0;
}
