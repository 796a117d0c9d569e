// TEST HARNESS (not a product path): the decoder harness tests/simt/decode_emul.cc plus what tests/test_coverage_simt.py
// needs of the coverage stage (amb_decode_coverage.cuh). The option lives in the decoder's own AmbDecodeState; the
// harness's emul_decode sets every other option from its EmulOpts and leaves this one as emul_set_coverage put it, so
// amb_decode_prepare, amb_decode_launch, amb_decode_reset and amb_decode_free treat the grid as the library does.
#include "decode_emul.cc"

// amb_decoder_set_option(d, "coverage", on): applies from the next emul_decode
extern "C" void emul_set_coverage(void* h, int on)
{
    static_cast<Emul*>(h)->st.coverage = on;
}

// amb_decoder_coverage: the grid into out (AMB_COVERAGE_CELLS doubles), all zeros before the first decode with the
// option on; returns whether the grid is allocated
extern "C" int emul_coverage(void* h, double* out)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    if (st.cgrid) memcpy(out, st.cgrid, AMB_COVERAGE_CELLS * sizeof(double));
    else memset(out, 0, AMB_COVERAGE_CELLS * sizeof(double));
    return st.cgrid != nullptr;
}

// the coverage stage alone (amb_coverage_launch) over n given records, into the decoder's grid (allocated by
// amb_decode_prepare with the option on): for records whose range and bearing a test chooses; returns 0, or -2 / -3
extern "C" int emul_coverage_records(void* h, const amb_fields* recs, int n)
{
    AmbDecodeState& st = static_cast<Emul*>(h)->st;
    st.coverage = 1;
    cudaError_t err = cudaSuccess;
    if (amb_decode_prepare(&st, 0, nullptr, &err) < 0) return -3;
    return amb_coverage_launch(recs, n, st.cgrid, nullptr, &err) < 0 ? -2 : 0;
}
