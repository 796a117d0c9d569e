// TEST HARNESS, not a product path: compiles the SBS-1 formatting of the decoder (gr_air_modes_b200/csrc/
// amb_sbs1_format.h - the __host__ __device__ code amb_sbs1_format calls on the device) for the host, so that
// tests/test_sbs1_cpu.py can check it against Python's % and datetime over whole input domains without a GPU.
// Built by the test into a temporary directory with plain g++.
#include "../gr_air_modes_b200/csrc/amb_sbs1_format.h"

// '%.<prec>f' % x[i] into out + i * 32 (NUL-terminated); "" where the formatter declines
extern "C" void shim_fixed(const double* x, long n, int prec, char* out)
{
    for (long i = 0; i < n; i++) {
        char* e = amb_sbs1_fixed(out + i * 32, x[i], prec);
        *(e ? e : out + i * 32) = 0;
    }
}

// '%i' % x[i] into out + i * 32
extern "C" void shim_trunc(const double* x, long n, char* out)
{
    for (long i = 0; i < n; i++) {
        char* e = amb_sbs1_trunc(out + i * 32, x[i]);
        *(e ? e : out + i * 32) = 0;
    }
}

// "date time" (23 bytes) into out + i * 32, or "" when the fields are empty
extern "C" void shim_stamp(const uint64_t* secs, const double* frac, long n, int tz, char* out)
{
    for (long i = 0; i < n; i++) {
        char* o = out + i * 32;
        if (amb_sbs1_stamp(secs[i], frac[i], tz, o, o + 11)) { o[10] = ' '; o[23] = 0; }
        else o[0] = 0;
    }
}

// the line of record r (NUL-terminated, "" for none)
extern "C" int shim_line(const amb_fields* r, uint64_t id, uint64_t secs, double frac, int tz, char* out)
{
    const int n = amb_sbs1_published(r) ? amb_sbs1_line(r, id, secs, frac, tz, out) : 0;
    out[n] = 0;
    return n;
}
