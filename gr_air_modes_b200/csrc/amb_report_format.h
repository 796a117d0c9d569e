// Text reports of the decoder option "reports" (DESIGN.md §8 "Text reports"): the line the reference's stdout printer
// (air_modes.output_print, python/msprint.py) writes for one decoded message, byte for byte what
// gr_air_modes_b200/report.py's format_report returns for the slicer's text of the frame and its record, plus "\n".
// __host__ __device__: amb_decode_reports.cuh calls it on the device, tests/reports_host_shim.cc on the host.
//
// The printer sees only the slicer's message text ("<hex> <crc> <level> <secs> <frac>", slicer_impl.cc:186-192), so the
// level and the fraction of the stamp are what Python's float() reads back from "%.*g" (precision 6 for the stream's
// first message, then 10) and "%.10g" of the frame's values. amb_rep_digits / amb_rep_from_decimal do that round trip
// exactly in integer arithmetic: the decimal is the exact binary value rounded half to even to N significant digits,
// and the double read back is the one nearest to that decimal (ties to even), as glibc's printf and CPython's float()
// do. Numbers in the body are amb_fmt_fixed (%.Nf, exact, half to even), amb_sbs1_trunc (%i of a float) and the
// integer writers of amb_sbs1_format.h.
#pragma once
#include "amb_sbs1_format.h"

// Widths of the variable fields: the rssi (-80 .. 385), the stamp (|secs + frac| < 2^66: sign, 20 digits, point, 8
// decimals), %x of 32 bits, %i of 32 bits (signed or not), %i of a byte, %i of a float below 2^63, %.Nf of |x| < 2^63.
#define AMB_REP_W_PREFIX (1 + 4 + 1 + (1 + 20 + 1 + 8) + 2)
#define AMB_REP_W_X32 9
#define AMB_REP_W_I32 11
#define AMB_REP_W_U8 3
#define AMB_REP_W_I63 20
#define AMB_REP_W_F(n) (1 + 19 + 1 + (n))
// the longest body of each kind (report.py's formats; the TCAS resolutions all set: 224 and 59 bytes of text)
#define AMB_REP_W_TCAS (5 + AMB_REP_W_U8 + 18 + AMB_REP_W_X32 + 2 + 7 + AMB_REP_W_U8 + 10 + AMB_REP_W_I32 + 6 + \
                        AMB_REP_W_I32 + 10 + 224 + 13 + 59 + 19 + 11 + 5 + AMB_REP_W_I32 + 2)
#define AMB_REP_W_COMMB (5 + AMB_REP_W_U8 + 1 + 34 + 6 + AMB_REP_W_X32 + 2 + 5 * (1 + 14 + AMB_REP_W_F(3) + 6))
#define AMB_REP_W_OPS (41 + AMB_REP_W_X32 + 9 + AMB_REP_W_U8 + 9 + 12 + 4 + 6 + 4 + 6 * (10 + AMB_REP_W_U8))
#define AMB_REP_W_TS (38 + AMB_REP_W_X32 + 14 + AMB_REP_W_I32 + 11 + 6 + AMB_REP_W_F(1) + 2 + 9 + AMB_REP_W_F(1) + \
                      29 + 3 * (10 + AMB_REP_W_U8))
#define AMB_REP_W_POS (38 + AMB_REP_W_X32 + 5 + 2 * AMB_REP_W_F(6) + 3 + 2 + AMB_REP_W_F(2) + 3 + AMB_REP_W_F(0) + 1 + \
                       4 + AMB_REP_W_I32 + 2 + 14 + AMB_REP_W_I63)
#define AMB_REP_W_BDS09 (16 + AMB_REP_W_U8 + 25 + AMB_REP_W_X32 + 9 + 4 * AMB_REP_W_F(0) + 48)
#define AMB_REP_W_LINK (5 + AMB_REP_W_U8 + 29 + AMB_REP_W_X32 + 9 + 3 * (AMB_REP_W_X32 + 9) + 11 + AMB_REP_W_I32 + 5 + \
                        AMB_REP_W_I32 + 2)
#define AMB_REP_MAX_LINE (AMB_REP_W_PREFIX + AMB_REP_W_TCAS + 1)    // bytes, with the "\n"
static_assert(AMB_REP_W_COMMB <= AMB_REP_W_TCAS && AMB_REP_W_OPS <= AMB_REP_W_TCAS && AMB_REP_W_TS <= AMB_REP_W_TCAS &&
              AMB_REP_W_POS <= AMB_REP_W_TCAS && AMB_REP_W_BDS09 <= AMB_REP_W_TCAS && AMB_REP_W_LINK <= AMB_REP_W_TCAS,
              "the TCAS report is the longest line");
static_assert(AMB_REP_MAX_LINE == 478, "the longest report line, as DESIGN.md states it");

typedef unsigned __int128 amb_u128;

AMB_HD int amb_rep_bitlen(amb_u128 v)                   // bits of v (0 for 0)
{
    const uint64_t hi = (uint64_t)(v >> 64), lo = (uint64_t)v;
#ifdef __CUDA_ARCH__
    return hi ? 128 - __clzll((long long)hi) : lo ? 64 - __clzll((long long)lo) : 0;
#else
    return hi ? 128 - __builtin_clzll(hi) : lo ? 64 - __builtin_clzll(lo) : 0;
#endif
}

AMB_HD amb_u128 amb_rep_pow5(int k) { amb_u128 v = 1; for (int i = 0; i < k; i++) v *= 5; return v; }

// num / den for a quotient below 2^bits with den << (bits - 1) < 2^128, by shift and subtract (no 128-bit division
// call on the device); *rem = the remainder
AMB_HD uint64_t amb_rep_div(amb_u128 num, amb_u128 den, int bits, amb_u128* rem)
{
    uint64_t q = 0;
    for (int i = bits - 1; i >= 0; i--) {
        const amb_u128 d = den << i;
        if (d <= num) { num -= d; q |= 1ull << i; }
    }
    *rem = num;
    return q;
}

// (v + s) * 2^e2 rounded to the nearest double, ties to even, where 0 <= s < 1 is nonzero iff `sticky`; v > 0 and the
// result a normal double.
AMB_HD double amb_rep_round(amb_u128 v, bool sticky, int e2)
{
    const int L = amb_rep_bitlen(v);
    v <<= 128 - L; e2 -= 128 - L;                       // bit 127 set; s stays below the last bit
    uint64_t m = (uint64_t)(v >> 75);                   // 53 bits
    const amb_u128 rest = v & (((amb_u128)1 << 75) - 1), half = (amb_u128)1 << 74;
    if (rest > half || (rest == half && (sticky || (m & 1)))) m++;
    e2 += 75;
    if (m >> 53) { m >>= 1; e2++; }
    const uint64_t bits = ((uint64_t)(e2 + 52 + 1023) << 52) | (m & ((1ull << 52) - 1));
    double x;
    memcpy(&x, &bits, 8);
    return x;
}

// The N significant digits (N = 6 or 10) of x = m * 2^e2 > 0 as "%.<N>g" writes them: q * 10^(E - N + 1), the exact
// value rounded half to even, 10^(N-1) <= q < 10^N. Exact for m < 2^53 and 2^-61 <= x < 2^128 (every quantity below
// stays under 2^127 there).
AMB_HD void amb_rep_digits(uint64_t m, int e2, int N, uint64_t* q_out, int* E_out)
{
    while (!(m & 1)) { m >>= 1; e2++; }
    uint64_t lo = 1;
    for (int i = 1; i < N; i++) lo *= 10;
    const uint64_t hi = lo * 10;
    int E = (int)floor((double)(amb_rep_bitlen(m) - 1 + e2) * 0.30102999566398120);   // within one of log10(x)
    for (;;) {
        const int p = E - N + 1;                        // q = x / 10^p
        amb_u128 num = m, den = 1;
        if (p >= 0) den = amb_rep_pow5(p); else num *= amb_rep_pow5(-p);
        if (e2 - p >= 0) num <<= (e2 - p); else den <<= (p - e2);
        amb_u128 r;
        uint64_t q = amb_rep_div(num, den, 40, &r);     // q < 10^11: E is within one of floor(log10(x))
        if (q >= hi) { E++; continue; }
        if (q < lo) { E--; continue; }
        const amb_u128 r2 = r * 2;
        if (r2 > den || (r2 == den && (q & 1))) q++;
        if (q == hi) { q = lo; E++; }
        *q_out = q; *E_out = E;
        return;
    }
}

// The double nearest to q * 10^p (0 < q < 2^34, -30 <= p <= 35), ties to even: float() of the decimal.
AMB_HD double amb_rep_from_decimal(uint64_t q, int p)
{
    if (p >= 0) return amb_rep_round((amb_u128)q * amb_rep_pow5(p), false, p);
    const amb_u128 den = amb_rep_pow5(-p);              // < 2^70
    const int s = 58 + amb_rep_bitlen(den) - amb_rep_bitlen(q);
    const amb_u128 num = (amb_u128)q << s;              // < 2^128; the quotient lies in (2^57, 2^59)
    amb_u128 r;
    const uint64_t Q = amb_rep_div(num, den, 59, &r);
    return amb_rep_round(Q, r != 0, -s + p);
}

// float("%.<N>g" % x) for finite x with 2^-61 <= |x| < 2^128, and whether the decimal is a power of ten (*pow10 = its
// exponent, else INT_MIN).
AMB_HD double amb_rep_roundtrip(double x, int N, int* pow10)
{
    const uint64_t b = amb_sbs1_bits(x);
    const int ex = (int)((b >> 52) & 0x7FF);
    const uint64_t m = (b & ((1ull << 52) - 1)) | (1ull << 52);
    uint64_t q; int E;
    amb_rep_digits(m, ex - 1075, N, &q, &E);
    uint64_t lo = 1;
    for (int i = 1; i < N; i++) lo *= 10;
    *pow10 = q == lo ? E : -2147483647 - 1;
    const double v = amb_rep_from_decimal(q, E - N + 1);
    return (b >> 63) ? -v : v;
}

// The "%i" of report.prefix: int(10 * log10(max(1e-8, level'))), level' = float("%.<N>g" % level), N = 6 for the first
// message and 10 after. Returns false where Python raises (+inf). Levels at or below 2^-27 give a level' below 1e-8
// (-80, as do NaN, zero and negative levels); where level' is a power of ten, 10^E, log10 is exactly E (true of
// CPython's libm for every such double, and checked by tests/test_reports_cpu.py), so the rssi is 10 E without a log;
// everywhere else 10 * log10(level') lies far enough from an integer (tests/test_reports_cpu.py bounds the distance over
// all float32 levels) that a log10 within a few ulps of the true value truncates to the same integer.
AMB_HD bool amb_rep_rssi(float level, int first, int* rssi)
{
    if (!(level > 7.450580596923828125e-9f)) { *rssi = -80; return true; }    // 2^-27; NaN too
    if (level > 3.4028234663852886e38f) return false;                         // +inf: int(inf) raises OverflowError
    int e10;
    const double L = amb_rep_roundtrip((double)level, first ? 6 : 10, &e10);
    if (e10 != -2147483647 - 1) { *rssi = e10 < -8 ? -80 : 10 * e10; return true; }
    if (!(L > 1e-8)) { *rssi = -80; return true; }
    *rssi = (int)(10.0 * log10(L));
    return true;
}

// "(%i %.8f) " of report.prefix for the frame's level and stamp, or nullptr where no line is written: +inf level, frac
// not finite or |frac| >= 2^64 (Python prints such stamps; the receiver never writes them). frac' = float("%.10g" %
// frac); secs' = secs + int(frac'), frac' -= int(frac'), and "%.8f" % (float(secs') + frac') with Python's int-to-float
// rounding. For |frac| < 2^-61 the round trip is skipped: it changes such a frac by less than 2^-90, which never moves
// "%.8f" of the sum.
AMB_HD char* amb_rep_prefix(char* p, float level, uint64_t secs, double frac, int first)
{
    int rssi;
    if (!amb_rep_rssi(level, first, &rssi)) return nullptr;
    if (!(fabs(frac) < 18446744073709551616.0)) return nullptr;
    int e10;
    const double f = fabs(frac) < 4.336808689942017736e-19 ? frac : amb_rep_roundtrip(frac, 10, &e10);
    const double fi = trunc(f);                         // |fi| < 2^64: "%.10g" never rounds up to 2^64
    const uint64_t mag = (uint64_t)fabs(fi);
    const __int128 s = (__int128)secs + (fi < 0 ? -(__int128)mag : (__int128)mag);
    const amb_u128 sm = s < 0 ? (amb_u128)(-s) : (amb_u128)s;
    double fs = sm ? amb_rep_round(sm, false, 0) : 0.0;   // float(secs'), exact to nearest even
    if (s < 0) fs = -fs;
    const double v = fs + (f - (fi == 0.0 ? 0.0 : fi));   // int(frac') is an int: 0 subtracts as +0.0
    *p++ = '(';
    p = amb_sbs1_i64(p, rssi);
    *p++ = ' ';
    p = amb_fmt_fixed(p, v, 8, 66);
    *p++ = ')'; *p++ = ' ';
    return p;
}

AMB_HD char* amb_rep_hex(char* p, int64_t v, int w)     // "%0<w>x" % v (w = 0: "%x"), lower case, '-' for a negative
{
    uint64_t u = (uint64_t)v;
    if (v < 0) { *p++ = '-'; u = 0ull - u; }
    char t[16]; int n = 0;
    do { const unsigned x = (unsigned)(u & 15u); t[n++] = (char)(x < 10 ? '0' + x : 'a' + x - 10); u >>= 4; } while (u);
    for (int i = n; i < w; i++) *p++ = '0';
    while (n) *p++ = t[--n];
    return p;
}

AMB_HD char* amb_rep_ident(char* p, const char* id)     // the record's ident with its trailing NULs stripped
{
    int n = 8;
    while (n && !id[n - 1]) n--;
    for (int i = 0; i < n; i++) *p++ = id[i];
    return p;
}

AMB_HD const char* amb_rep_fs(unsigned fs)              // msprint.py:86-98; nullptr where fs_text raises
{
    switch (fs) {
    case 1: return " (aircraft is on the ground)";
    case 2: return " (AIRBORNE ALERT)";
    case 3: return " (GROUND ALERT)";
    case 4: return " (SPI ALERT)";
    case 5: return " (SPI)";
    default: return nullptr;
    }
}

// Comm-B inference (option "commb"): "Type %i %s from %x: " and the fields present, as report._commb_text of
// decode.commb_values: raw 16-bit field i of aux, times its LSB (+ 800 for baro) in fp64.
AMB_HD char* amb_rep_commb(char* p, const amb_fields* r)
{
    const unsigned reg = (unsigned)((r->pad_ >> 16) & 0xFF), mask = (unsigned)((r->pad_ >> 24) & 0xFF);
    if (reg != 0x40 && reg != 0x50 && reg != 0x60) return nullptr;
    p = amb_sbs1_str(p, "Type "); p = amb_sbs1_u64(p, r->df);
    p = amb_sbs1_str(p, reg == 0x40 ? " BDS4,0 selected vertical intention" : reg == 0x50 ? " BDS5,0 track and turn report"
                                                                                       : " BDS6,0 heading and speed report");
    p = amb_sbs1_str(p, " from "); p = amb_rep_hex(p, r->ecc, 0); p = amb_sbs1_str(p, ": ");
    bool any = false;
    for (int i = 0; i < 5; i++) {
        if (!(mask & (1u << i))) continue;
        const int raw = (int)(int16_t)(uint16_t)((r->aux[i / 2] >> (16 * (i % 2))) & 0xFFFF);
        if (any) *p++ = ' ';
        any = true;
        const int k = (int)(reg >> 4) - 4;              // 0, 1, 2
        static const char* const name[3][5] = {{"MCP alt ", "FMS alt ", "baro ", "modes ", "alt source "},
                                               {"roll ", "track ", "GS ", "track rate ", "TAS "},
                                               {"heading ", "IAS ", "Mach ", "baro rate ", "inertial rate "}};
        static const char* const unit[3][5] = {{"ft", "ft", "mb", "", ""}, {"", "", "kt", "", "kt"},
                                               {"", "kt", "", "ft/min", "ft/min"}};
        p = amb_sbs1_str(p, name[k][i]);
        char* e = p;
        if (k == 0) {
            if (i < 2) e = amb_sbs1_trunc(p, raw * 16.0 + 0.0);
            else if (i == 2) e = amb_fmt_fixed(p, raw * 0.1 + 800.0, 1, 63);
            else e = amb_sbs1_i64(p, raw);
        } else if (k == 1) {
            if (i == 0) e = amb_fmt_fixed(p, raw * (45.0 / 256) + 0.0, 1, 63);
            else if (i == 1) e = amb_fmt_fixed(p, raw * (90.0 / 512) + 0.0, 1, 63);
            else if (i == 3) e = amb_fmt_fixed(p, raw * (8.0 / 256) + 0.0, 2, 63);
            else e = amb_sbs1_trunc(p, raw * 2.0 + 0.0);
        } else {
            if (i == 0) e = amb_fmt_fixed(p, raw * (90.0 / 512) + 0.0, 1, 63);
            else if (i == 1) e = amb_sbs1_i64(p, raw);
            else if (i == 2) e = amb_fmt_fixed(p, raw * (2.048 / 512) + 0.0, 3, 63);
            else e = amb_sbs1_trunc(p, raw * 32.0 + 0.0);
        }
        if (!e) return nullptr;
        p = amb_sbs1_str(e, unit[k][i]);
    }
    return p;
}

// Op status (option "opstatus"): report._opstatus_text of decode.opstatus_values for a TC 31 or TC 29 record.
AMB_HD char* amb_rep_opstatus(char* p, const amb_fields* r)
{
    const unsigned es = (unsigned)((r->pad_ >> 40) & 0xFF), ver = (unsigned)((r->pad_ >> 48) & 0xFF);
    const uint8_t* b = (const uint8_t*)r->aux;
    const unsigned w0 = b[0] | (unsigned)b[1] << 8, w1 = b[2] | (unsigned)b[3] << 8, w2 = b[4] | (unsigned)b[5] << 8;
    if (es == AMB_ES_OPSTATUS) {
        p = amb_sbs1_str(p, "Type 17 BDS6,5 (operational status) from "); p = amb_rep_hex(p, r->icao, 0);
        p = amb_sbs1_str(p, " version "); p = amb_sbs1_u64(p, ver);
        p = amb_sbs1_str(p, b[4] ? " surface capability " : " airborne capability "); p = amb_rep_hex(p, w0, 4);
        p = amb_sbs1_str(p, " mode "); p = amb_rep_hex(p, w1, 4);
        if (ver) {
            p = amb_sbs1_str(p, " NIC-A "); p = amb_sbs1_u64(p, b[5]);
            p = amb_sbs1_str(p, " NACp "); p = amb_sbs1_u64(p, b[6]);
            p = amb_sbs1_str(p, " SIL "); p = amb_sbs1_u64(p, b[8]);
            if (b[4]) {
                p = amb_sbs1_str(p, " NIC-C "); p = amb_sbs1_u64(p, b[12]);
                p = amb_sbs1_str(p, " TRK/HDG "); p = amb_sbs1_u64(p, b[9]);
                p = amb_sbs1_str(p, " L/W "); p = amb_sbs1_u64(p, b[13]);
            } else {
                p = amb_sbs1_str(p, " GVA "); p = amb_sbs1_u64(p, b[7]);
                p = amb_sbs1_str(p, " NICbaro "); p = amb_sbs1_u64(p, b[9]);
            }
            p = amb_sbs1_str(p, " HRD "); p = amb_sbs1_u64(p, b[10]);
            p = amb_sbs1_str(p, " SIL supp "); p = amb_sbs1_u64(p, b[11]);
        }
        return p;
    }
    if (es != AMB_ES_TARGET_STATE) return nullptr;
    p = amb_sbs1_str(p, "Type 17 BDS6,2 (target state) from "); p = amb_rep_hex(p, r->icao, 0);
    if (w0) {
        p = amb_sbs1_str(p, " selected alt "); p = amb_sbs1_i64(p, ((int64_t)w0 - 1) * 32);
        p = amb_sbs1_str(p, b[7] ? "ft (FMS)" : "ft (MCP/FCU)");
    }
    if (w1) { p = amb_sbs1_str(p, " baro "); p = amb_fmt_fixed(p, 800.0 + ((int)w1 - 1) * 0.8, 1, 63); p = amb_sbs1_str(p, "mb"); }
    if (b[8]) { p = amb_sbs1_str(p, " heading "); p = amb_fmt_fixed(p, w2 * 180.0 / 256, 1, 63); }
    const unsigned modes = b[12];
    static const char* const mname[6] = {"AP", "VNAV", "ALT", "APP", "LNAV", "TCAS"};
    static const unsigned mbit[6] = {0x40, 0x20, 0x10, 0x04, 0x01, 0x02};
    bool any = false;
    for (int i = 0; i < 6; i++) {
        if (!(modes & mbit[i]) || (i < 5 && !(modes & 0x80))) continue;
        p = amb_sbs1_str(p, any ? " " : " modes ");
        p = amb_sbs1_str(p, mname[i]);
        any = true;
    }
    p = amb_sbs1_str(p, " NACp "); p = amb_sbs1_u64(p, b[9]);
    p = amb_sbs1_str(p, " NICbaro "); p = amb_sbs1_u64(p, b[10]);
    p = amb_sbs1_str(p, " SIL "); p = amb_sbs1_u64(p, b[11]);
    return p;
}

// " " + text of every resolution bit set (parse.py:380-397)
AMB_HD char* amb_rep_resolutions(char* p, uint32_t bits, int n, int top, const char* const* text)
{
    for (int k = 0; k < n; k++)
        if (bits & (1u << (top - k))) { *p++ = ' '; p = amb_sbs1_str(p, text[k]); }
    return p;
}

// The body of format_report after the prefix (report.py:113-212) for a queued record that the parser handled.
AMB_HD char* amb_rep_body(char* p, const amb_fields* r)
{
    const unsigned df = r->df, st = r->status;
    const uint32_t ecc = r->ecc;
    if (!(df == 0 || df == 4 || df == 5 || df == 11 || df == 16 || df == 17 || df == 20 || df == 21)) {
        p = amb_sbs1_str(p, "No handler for message type "); p = amb_sbs1_u64(p, df);
        p = amb_sbs1_str(p, " from "); return amb_rep_hex(p, ecc, 6);
    }
    const bool metric = st & AMB_FS_METRIC_ALT;
    if (df == 0) {
        if (metric) return nullptr;
        p = amb_sbs1_str(p, "Type 0 (short A-A surveillance) from "); p = amb_rep_hex(p, ecc, 0);
        p = amb_sbs1_str(p, " at "); p = amb_sbs1_i64(p, r->altitude); p = amb_sbs1_str(p, "ft");
        const unsigned ri = r->ri;
        if (ri == 0) p = amb_sbs1_str(p, " (No TCAS)");
        else if (ri == 2) p = amb_sbs1_str(p, " (TCAS resolution inhibited)");
        else if (ri == 3) p = amb_sbs1_str(p, " (Vertical TCAS resolution only)");
        else if (ri == 4) p = amb_sbs1_str(p, " (Full TCAS resolution)");
        else if (ri == 9) p = amb_sbs1_str(p, " (speed <75kt)");
        else if (ri > 9) {
            p = amb_sbs1_str(p, " (speed "); p = amb_sbs1_u64(p, 75ull << (ri - 10)); *p++ = '-';
            p = amb_sbs1_u64(p, 75ull << (ri - 9)); p = amb_sbs1_str(p, "kt)");
        } else return nullptr;
        if (r->vs == 1) p = amb_sbs1_str(p, " (aircraft is on the ground)");
        return p;
    }
    if (df == 4 || df == 5) {
        const char* fs = amb_rep_fs(r->fs);
        if ((df == 4 && metric) || !fs) return nullptr;
        if (df == 4) {
            p = amb_sbs1_str(p, "Type 4 (short surveillance altitude reply) from "); p = amb_rep_hex(p, ecc, 0);
            p = amb_sbs1_str(p, " at "); p = amb_sbs1_i64(p, r->altitude); p = amb_sbs1_str(p, "ft");
        } else {
            p = amb_sbs1_str(p, "Type 5 (short surveillance ident reply) from "); p = amb_rep_hex(p, ecc, 0);
            p = amb_sbs1_str(p, " with ident "); p = amb_sbs1_i64(p, r->squawk);
        }
        return amb_sbs1_str(p, fs);
    }
    if (df == 11) {
        p = amb_sbs1_str(p, "Type 11 (all call reply) from "); p = amb_rep_hex(p, r->icao, 0);
        p = amb_sbs1_str(p, " in reply to interrogator "); p = amb_sbs1_u64(p, ecc & 0xF);
        p = amb_sbs1_str(p, " with capability level "); return amb_sbs1_u64(p, r->ca + 1u);
    }
    if (df == 17) {
        const unsigned bds = r->bds;
        if (bds == 0x08) {
            static const char* const cats[4][8] = {
                {"NO INFO", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED", "RESERVED"},
                {"NO INFO", "SURFACE EMERGENCY VEHICLE", "SURFACE SERVICE VEHICLE", "FIXED OBSTRUCTION",
                 "CLUSTER OBSTRUCTION", "LINE OBSTRUCTION", "RESERVED", nullptr},
                {"NO INFO", "GLIDER", "BALLOON/BLIMP", "PARACHUTE", "ULTRALIGHT", "RESERVED", "UAV", "SPACECRAFT"},
                {"NO INFO", "LIGHT", "SMALL", "LARGE", "LARGE HIGH VORTEX", "HEAVY", "HIGH PERFORMANCE", "ROTORCRAFT"}};
            const int row = r->ftc == 0 ? 3 : (int)r->ftc - 1;          // Python's categories[-1] for ftc 0
            if (row > 3 || r->cat >= 8 || !cats[row][r->cat]) return nullptr;   // IndexError (parse.py:268)
            p = amb_sbs1_str(p, "Type 17 BDS0,8 (ident) from "); p = amb_rep_hex(p, r->icao, 0);
            p = amb_sbs1_str(p, " type "); p = amb_sbs1_str(p, cats[row][r->cat]);
            p = amb_sbs1_str(p, " ident "); return amb_rep_ident(p, r->ident);
        }
        if (bds == 0x05 || bds == 0x06) {
            if (!(st & AMB_FS_HAS_POS)) return nullptr;
            p = amb_sbs1_str(p, bds == 0x06 ? "Type 17 BDS0,6 (surface report) from " : "Type 17 BDS0,5 (position report) from ");
            p = amb_rep_hex(p, r->icao, 0);
            p = amb_sbs1_str(p, " at (");
            if (!(p = amb_fmt_fixed(p, r->lat, 6, 63))) return nullptr;
            p = amb_sbs1_str(p, ", ");
            if (!(p = amb_fmt_fixed(p, r->lon, 6, 63))) return nullptr;
            *p++ = ')';
            if (bds == 0x06) {
                p = amb_sbs1_str(p, " ground track ");
                if (!(p = amb_sbs1_trunc(p, r->val[0]))) return nullptr;
            }
            if (st & AMB_FS_HAS_RANGE) {
                p = amb_sbs1_str(p, " (");
                if (!(p = amb_fmt_fixed(p, r->range, 2, 63))) return nullptr;
                p = amb_sbs1_str(p, " @ ");
                if (!(p = amb_fmt_fixed(p, r->bearing, 0, 63))) return nullptr;
                *p++ = ')';
            }
            if (bds == 0x06) return p;
            p = amb_sbs1_str(p, " at "); p = amb_sbs1_i64(p, r->altitude); return amb_sbs1_str(p, "ft");
        }
        if (bds == 0x09) {
            const unsigned sub = r->subtype;
            p = amb_sbs1_str(p, "Type 17 BDS0,9-"); p = amb_sbs1_u64(p, sub);
            p = amb_sbs1_str(p, sub <= 1 ? " (track report) from " : " (air course report) from ");
            p = amb_rep_hex(p, r->icao, 0);
            const double* v = r->val;
            static const char* const tr[4] = {" with velocity ", "kt heading ", " VS ", " turn rate "};
            static const char* const ac[4] = {"kt magnetic heading ", " VS ", " geo. diff. from baro. alt. ", "ft"};
            if (sub <= 1) {
                for (int i = 0; i < (sub == 0 ? 4 : 3); i++) {
                    p = amb_sbs1_str(p, tr[i]);
                    if (!(p = amb_fmt_fixed(p, v[i], 0, 63))) return nullptr;
                }
                return p;
            }
            p = amb_sbs1_str(p, r->ast == 1 ? " with TAS " : " with IAS ");
            const int order[4] = {1, 0, 2, 3};
            for (int i = 0; i < 4; i++) {
                if (!(p = amb_fmt_fixed(p, v[order[i]], 0, 63))) return nullptr;
                p = amb_sbs1_str(p, ac[i]);
            }
            return p;
        }
        p = amb_sbs1_str(p, "Type 17 with FTC="); p = amb_sbs1_u64(p, r->ftc);
        p = amb_sbs1_str(p, " from "); p = amb_rep_hex(p, r->icao, 0); return amb_sbs1_str(p, " not implemented");
    }
    if (df == 16) return nullptr;                       // printTCAS reads a field DF16 does not have (report.py:179-180)
    const unsigned bds1 = r->bds;
    const uint32_t* a = r->aux;
    if (bds1 == 0) {
        p = amb_sbs1_str(p, "No handler in type "); p = amb_sbs1_u64(p, df);
        p = amb_sbs1_str(p, " for BDS1 == 0 from "); p = amb_rep_hex(p, ecc, 0);
    } else if (bds1 == 1) {
        p = amb_sbs1_str(p, "Type "); p = amb_sbs1_u64(p, df);
        p = amb_sbs1_str(p, " link capability report from "); p = amb_rep_hex(p, ecc, 0);
        p = amb_sbs1_str(p, ": ACS: 0x"); p = amb_rep_hex(p, a[0], 0);
        p = amb_sbs1_str(p, ", BCS: 0x"); p = amb_rep_hex(p, a[1], 0);
        p = amb_sbs1_str(p, ", ECS: 0x"); p = amb_rep_hex(p, a[2], 0);
        p = amb_sbs1_str(p, ", continues "); p = amb_sbs1_u64(p, a[3]);
    } else if (bds1 == 2) {
        p = amb_sbs1_str(p, "Type "); p = amb_sbs1_u64(p, df);
        p = amb_sbs1_str(p, " identification from "); p = amb_rep_hex(p, ecc, 0);
        p = amb_sbs1_str(p, " with text "); p = amb_rep_ident(p, r->ident);
    } else {
        static const char* const ara[14] = {"CLIMB", "DON'T DESCEND", "DON'T DESCEND >500FPM", "DON'T DESCEND >1000FPM",
                                            "DON'T DESCEND >2000FPM", "DESCEND", "DON'T CLIMB", "DON'T CLIMB >500FPM",
                                            "DON'T CLIMB >1000FPM", "DON'T CLIMB >2000FPM", "TURN LEFT", "TURN RIGHT",
                                            "DON'T TURN LEFT", "DON'T TURN RIGHT"};
        static const char* const rac[4] = {"DON'T DESCEND", "DON'T CLIMB", "DON'T TURN LEFT", "DON'T TURN RIGHT"};
        p = amb_sbs1_str(p, "Type "); p = amb_sbs1_u64(p, df);
        p = amb_sbs1_str(p, " TCAS report from "); p = amb_rep_hex(p, ecc, 0); p = amb_sbs1_str(p, ": ");
        const unsigned tti = r->tti;
        unsigned rat = a[2] & 1, mte = (a[2] >> 1) & 1;
        if (tti == 1 || tti == 2) {
            if (tti == 1) { p = amb_sbs1_str(p, "threat ID: "); p = amb_rep_hex(p, a[3], 0); }
            else {
                if (r->threat_alt == AMB_NO_ALTITUDE) return nullptr;  // MetricAltError (parse.py:407)
                p = amb_sbs1_str(p, "range: "); p = amb_sbs1_u64(p, a[3] & 0x7F);
                p = amb_sbs1_str(p, " bearing: "); p = amb_sbs1_u64(p, a[3] >> 8);
                p = amb_sbs1_str(p, " alt: "); p = amb_sbs1_i64(p, r->threat_alt);
            }
            p = amb_sbs1_str(p, " advised: "); p = amb_rep_resolutions(p, a[0], 14, 13, ara);
            p = amb_sbs1_str(p, " complement: "); p = amb_rep_resolutions(p, a[1], 4, 3, rac);
        } else {
            rat = mte = 0;
            p = amb_sbs1_str(p, " (no handler for TTI="); p = amb_sbs1_u64(p, tti); *p++ = ')';
        }
        if (mte) p = amb_sbs1_str(p, " (multiple threats)");
        if (rat) p = amb_sbs1_str(p, " (resolved)");
    }
    if (df == 20) {
        if (r->altitude == AMB_NO_ALTITUDE) return nullptr;         // MetricAltError (msprint.py:251)
        p = amb_sbs1_str(p, " at "); p = amb_sbs1_i64(p, r->altitude); return amb_sbs1_str(p, "ft");
    }
    p = amb_sbs1_str(p, " ident "); return amb_rep_hex(p, r->squawk, 0);
}

// The whole line of the frame f and its record r, "\n" included, into out (at least AMB_REP_MAX_LINE bytes, no
// terminator); first: the frame is the stream's first queued message (precision 6). Returns its length, 0 for none.
AMB_HD int amb_report_line(const amb_frame* f, const amb_fields* r, int first, char* out)
{
    const unsigned st = r->status, df = r->df;
    char* p = nullptr;
    if (st == AMB_FS_NO_HANDLER && (df == 20 || df == 21)) {
        const unsigned oc = (unsigned)((r->pad_ >> 8) & 0xFF);
        if (oc == AMB_COMMB_DECODED || oc == AMB_COMMB_RESOLVED) {
            if (!(p = amb_rep_prefix(out, f->ref_level, f->secs, f->frac, first))) return 0;
            p = amb_rep_commb(p, r);
        }
    } else if (st == AMB_FS_NO_HANDLER && df == 17) {
        const unsigned es = (unsigned)((r->pad_ >> 40) & 0xFF);
        if (es == AMB_ES_OPSTATUS || es == AMB_ES_TARGET_STATE) {
            if (!(p = amb_rep_prefix(out, f->ref_level, f->secs, f->frac, first))) return 0;
            p = amb_rep_opstatus(p, r);
        }
    } else if (!(st & (AMB_FS_NO_HANDLER | AMB_FS_NOT_QUEUED))) {
        if (!(p = amb_rep_prefix(out, f->ref_level, f->secs, f->frac, first))) return 0;
        p = amb_rep_body(p, r);
    }
    if (!p) return 0;
    *p++ = '\n';
    return (int)(p - out);
}
