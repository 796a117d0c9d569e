// TEST HARNESS, not a product path: compiles the text-report formatting of the decoder (gr_air_modes_b200/csrc/
// amb_report_format.h - the __host__ __device__ code amb_decode_reports.cuh calls on the device) for the host, so that
// tests/test_reports_cpu.py can check it against Python's %, float() and report.format_report without a GPU.
// Built by the test into a temporary directory with plain g++.
#include "../gr_air_modes_b200/csrc/amb_report_format.h"

// float("%.<N>g" % x[i]) for N = 6 or 10, and whether that decimal is a power of ten (pow10[i], else INT_MIN)
extern "C" void shim_roundtrip(const double* x, long n, int N, double* out, int* pow10)
{
    for (long i = 0; i < n; i++) out[i] = amb_rep_roundtrip(x[i], N, &pow10[i]);
}

// the rssi of report.prefix for float32 levels (first: precision 6); INT_MIN where no line is written
extern "C" void shim_rssi(const float* lev, long n, int first, int* out)
{
    for (long i = 0; i < n; i++)
        if (!amb_rep_rssi(lev[i], first, &out[i])) out[i] = -2147483647 - 1;
}

// the prefix "(%i %.8f) " into out + i * 64 (NUL-terminated, "" where no line is written)
extern "C" void shim_prefix(const float* lev, const uint64_t* secs, const double* frac, long n, int first, char* out)
{
    for (long i = 0; i < n; i++) {
        char* o = out + i * 64;
        char* e = amb_rep_prefix(o, lev[i], secs[i], frac[i], first);
        *(e ? e : o) = 0;
    }
}

// '%.<prec>f' % x[i] (|x| < 2^lim) into out + i * 48; "" where the formatter declines
extern "C" void shim_fixed(const double* x, long n, int prec, int lim, char* out)
{
    for (long i = 0; i < n; i++) {
        char* e = amb_fmt_fixed(out + i * 48, x[i], prec, lim);
        *(e ? e : out + i * 48) = 0;
    }
}

// the report line of frame f and record r (NUL-terminated, "" for none); returns its length
extern "C" int shim_line(const amb_frame* f, const amb_fields* r, int first, char* out)
{
    const int n = amb_report_line(f, r, first, out);
    out[n] = 0;
    return n;
}

extern "C" int shim_max_line() { return AMB_REP_MAX_LINE; }
