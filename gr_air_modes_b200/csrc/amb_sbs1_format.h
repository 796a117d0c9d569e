// SBS-1 (BaseStation) lines of the decoder option "sbs1" (DESIGN.md §8 "SBS-1 feed"): which records are published,
// and the text of one line, byte for byte what the reference's python/sbs1.py (pp0 .. pp17, :153-222) writes for the
// same message, with the date and time taken from the frame's stamp. __host__ __device__: amb_decode_sbs1.cuh calls it
// on the device, tests/sbs1_host_shim.cc on the host. Numbers are formatted from the exact binary value with integer
// arithmetic, as Python's % does: %.Nf rounds half to even, %i of a float truncates toward zero.
#pragma once
#include <string.h>

#include "amb_decode_core.h"

#define AMB_SBS1_WINDOW 10000ull                 // ids kept live, as sbs1.py:83-88 prunes its map (Python 2)
#define AMB_SBS1_LAST_SEC 253402300799ll         // 9999-12-31 23:59:59 UTC: the last second %Y can write in 4 digits
#define AMB_SBS1_STRIDE 192                      // bytes of one line's slot on the device

// Widths of the variable fields: ids (uint64), the 24-bit address, the stamp, a signed 32-bit altitude, an 8-character
// ident, %.5f and %.1f of |x| < 2^63 (sign, 19 digits, point, decimals), %i of such a float (sign and 19 digits).
#define AMB_SBS1_W_ID 20
#define AMB_SBS1_W_HEAD (8 + AMB_SBS1_W_ID + 1 + 6 + 1 + AMB_SBS1_W_ID + 1 + 10 + 1 + 12 + 1 + 10 + 1 + 12)   // MSG,n,0, .. time
#define AMB_SBS1_W_INT32 11
#define AMB_SBS1_W_F5 (1 + 19 + 1 + 5)
#define AMB_SBS1_W_F1 (1 + 19 + 1 + 1)
#define AMB_SBS1_W_I64 20
// the longest tail of each line after the head (the formats of sbs1.py:156-220)
#define AMB_SBS1_W_MSG7 (2 + AMB_SBS1_W_INT32 + 10 + 3)
#define AMB_SBS1_W_MSG5 (2 + AMB_SBS1_W_INT32 + 7 + 7 + 2)
#define AMB_SBS1_W_MSG6 (8 + AMB_SBS1_W_INT32 + 1 + 7 + 2)
#define AMB_SBS1_W_MSG8 14
#define AMB_SBS1_W_MSG1 (1 + 8 + 13)
#define AMB_SBS1_W_MSG23 (2 + AMB_SBS1_W_INT32 + 3 + AMB_SBS1_W_F5 + 1 + AMB_SBS1_W_F5 + 11)
#define AMB_SBS1_W_MSG4 (3 + AMB_SBS1_W_F1 + 1 + AMB_SBS1_W_F1 + 3 + AMB_SBS1_W_I64 + 7)
#define AMB_SBS1_MAX2(a, b) ((a) > (b) ? (a) : (b))
#define AMB_SBS1_MAX_LINE (AMB_SBS1_W_HEAD + AMB_SBS1_MAX2(AMB_SBS1_MAX2(AMB_SBS1_MAX2(AMB_SBS1_W_MSG7, AMB_SBS1_W_MSG5), \
    AMB_SBS1_MAX2(AMB_SBS1_W_MSG6, AMB_SBS1_W_MSG8)), AMB_SBS1_MAX2(AMB_SBS1_MAX2(AMB_SBS1_W_MSG1, AMB_SBS1_W_MSG23), \
    AMB_SBS1_W_MSG4)))
static_assert(AMB_SBS1_MAX_LINE <= AMB_SBS1_STRIDE, "an SBS-1 line must fit its slot");

// Rule 1: the records output_sbs1.output sees (sbs1.py:64-65 subscribes to DF0/4/5/11/17; make_parser publishes
// nothing for a message whose parse raised NoHandlerError, parse.py:422-436).
AMB_HD bool amb_sbs1_published(const amb_fields* r)
{
    const unsigned df = r->df;
    return !(r->status & (AMB_FS_NOT_QUEUED | AMB_FS_NO_HANDLER)) && r->icao < (1u << 24) &&
           (df == 0 || df == 4 || df == 5 || df == 11 || df == 17);
}

AMB_HD char* amb_sbs1_str(char* p, const char* s) { while (*s) *p++ = *s++; return p; }

AMB_HD char* amb_sbs1_u64(char* p, uint64_t v)          // %i of a non-negative int
{
    char t[20]; int n = 0;
    do { t[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) *p++ = t[--n];
    return p;
}

AMB_HD char* amb_sbs1_i64(char* p, int64_t v)           // %i of an int
{
    if (v < 0) { *p++ = '-'; return amb_sbs1_u64(p, 0ull - (uint64_t)v); }
    return amb_sbs1_u64(p, (uint64_t)v);
}

AMB_HD char* amb_sbs1_dec(char* p, unsigned v, int w)   // v zero-padded to w digits (v < 10^w)
{
    for (int i = w - 1; i >= 0; i--) { p[i] = (char)('0' + v % 10); v /= 10; }
    return p + w;
}

AMB_HD char* amb_sbs1_hex6(char* p, uint32_t v)         // %06X of a 24-bit value
{
    for (int i = 5; i >= 0; i--) { const unsigned x = v & 15u; p[i] = (char)(x < 10 ? '0' + x : 'A' + x - 10); v >>= 4; }
    return p + 6;
}

AMB_HD uint64_t amb_sbs1_bits(double x) { uint64_t b; memcpy(&b, &x, 8); return b; }

AMB_HD char* amb_fmt_u128(char* p, unsigned __int128 v)  // %i of a non-negative int below 2^128
{
    if (!(v >> 64)) return amb_sbs1_u64(p, (uint64_t)v);
    uint32_t w[4] = {(uint32_t)(v >> 96), (uint32_t)(v >> 64), (uint32_t)(v >> 32), (uint32_t)v};
    char t[39]; int n = 0;
    for (bool more = true; more;) {                     // divide the 32-bit limbs by 10, most significant first
        uint64_t r = 0;
        more = false;
        for (int i = 0; i < 4; i++) {
            const uint64_t x = (r << 32) | w[i];
            w[i] = (uint32_t)(x / 10); r = x % 10;
            more = more || w[i];
        }
        t[n++] = (char)('0' + r);
    }
    while (n) *p++ = t[--n];
    return p;
}

// '%.<prec>f' % x (prec 0..8) as Python writes it: the exact binary value rounded half to even (for prec 0 the last
// digit is the integer part's, and no point is written), the sign of -0.0 and of a value that rounds to zero kept,
// nan / inf / -inf. Returns nullptr for |x| >= 2^lim (lim 53..66), which the caller never formats.
AMB_HD char* amb_fmt_fixed(char* p, double x, int prec, int lim)
{
    const uint64_t b = amb_sbs1_bits(x);
    const int ex = (int)((b >> 52) & 0x7FF);
    uint64_t m = b & ((1ull << 52) - 1);
    if (ex == 0x7FF) {
        if (m) return amb_sbs1_str(p, "nan");
        return amb_sbs1_str(p, (b >> 63) ? "-inf" : "inf");
    }
    if (b >> 63) *p++ = '-';
    int sh;                                             // |x| = m * 2^-sh
    if (ex) { m |= 1ull << 52; sh = 1075 - ex; } else sh = 1074;
    uint64_t P = 1;
    for (int i = 0; i < prec; i++) P *= 10;
    unsigned __int128 ip;                               // integer part
    uint64_t fd;                                        // decimals
    if (sh <= 0) {
        if (-sh > lim - 53) return nullptr;             // m << -sh would reach 2^lim
        ip = (unsigned __int128)m << -sh; fd = 0;
    } else {
        ip = sh < 64 ? m >> sh : 0;
        const uint64_t f = sh < 64 ? m & ((1ull << sh) - 1) : m;    // the fraction is f / 2^sh
        if (sh >= 128) fd = 0;                          // f * P < 2^80 < 2^(sh - 1): below half a unit of the last digit
        else {
            const unsigned __int128 num = (unsigned __int128)f * P;
            uint64_t q = (uint64_t)(num >> sh);
            const unsigned __int128 rem = num - ((unsigned __int128)q << sh), half = (unsigned __int128)1 << (sh - 1);
            if (!prec) { if (rem > half || (rem == half && (ip & 1))) ip++; }   // the last digit is the integer part's
            else if (rem > half || (rem == half && (q & 1))) q++;
            if (q == P) { q = 0; ip++; }
            fd = q;
        }
    }
    p = amb_fmt_u128(p, ip);
    if (!prec) return p;
    *p++ = '.';
    return amb_sbs1_dec(p, (unsigned)fd, prec);
}

// '%.<prec>f' % x (prec 1..5) of a line's field; nullptr for |x| >= 2^63 (never a field of a line).
AMB_HD char* amb_sbs1_fixed(char* p, double x, int prec) { return amb_fmt_fixed(p, x, prec, 63); }

// '%i' % x of a float: int(x), truncated toward zero (-0.0 and -0.5 print 0). nullptr where Python raises (nan, inf)
// or |x| >= 2^63.
AMB_HD char* amb_sbs1_trunc(char* p, double x)
{
    if (!(fabs(x) < 9223372036854775808.0)) return nullptr;
    return amb_sbs1_i64(p, (int64_t)x);
}

// Rule 5: "%Y/%m/%d" and "%H:%M:%S.mmm" of the frame's stamp. The stamp is first normalised as modes_types.stamp does
// (secs += int(frac); frac -= int(frac), exactly, for any finite frac); milliseconds are max(0, min(999,
// floor(frac * 1000))) of the normalised frac in fp64 (a frame's frac is never negative; a negative one counts as 0);
// the date is proleptic Gregorian of secs + 60 * tz_min. Returns false, with nothing written, when that lies outside
// 1970-01-01 00:00:00 .. 9999-12-31 23:59:59, or when frac is not finite (int(frac) raises in Python).
AMB_HD bool amb_sbs1_stamp(uint64_t secs, double frac, int tz_min, char* date, char* tod)
{
    const double fi = trunc(frac);
    if (!(fabs(fi) < 18446744073709551616.0)) return false;   // |int(frac)| >= 2^64, nan, inf: outside the range
    const uint64_t mag = (uint64_t)fabs(fi);            // exact: an integral double below 2^64
    const __int128 s128 = (__int128)secs + (fi < 0 ? -(__int128)mag : (__int128)mag) + 60 * (__int128)tz_min;
    if (s128 < 0 || s128 > AMB_SBS1_LAST_SEC) return false;
    const int64_t s = (int64_t)s128;
    const double f = frac - fi;
    double msf = floor(f * 1000.0);
    msf = msf < 0.0 ? 0.0 : msf > 999.0 ? 999.0 : msf;
    const int64_t days = s / 86400, sod = s % 86400;
    // civil date of a day count (days since 1970-01-01), in 400-year eras of 146097 days starting on a March 1st
    const int64_t z = days + 719468, era = z / 146097, doe = z - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100), mp = (5 * doy + 2) / 153;
    const unsigned d = (unsigned)(doy - (153 * mp + 2) / 5 + 1), mo = (unsigned)(mp < 10 ? mp + 3 : mp - 9);
    const unsigned y = (unsigned)(yoe + era * 400 + (mo <= 2));
    char* p = amb_sbs1_dec(date, y, 4); *p++ = '/'; p = amb_sbs1_dec(p, mo, 2); *p++ = '/'; amb_sbs1_dec(p, d, 2);
    p = amb_sbs1_dec(tod, (unsigned)(sod / 3600), 2); *p++ = ':';
    p = amb_sbs1_dec(p, (unsigned)(sod / 60 % 60), 2); *p++ = ':';
    p = amb_sbs1_dec(p, (unsigned)(sod % 60), 2); *p++ = '.';
    amb_sbs1_dec(p, (unsigned)msf, 3);
    return true;
}

AMB_HD const char* amb_sbs1_fs(unsigned fs)             // output_sbs1.decode_fs (sbs1.py:117-131)
{
    switch (fs) {
    case 0: return "0,0,0,0";
    case 1: return "0,0,0,1";
    case 2: return "1,0,0,0";
    case 3: return "1,0,0,1";
    case 4: return "1,0,1,";
    case 5: return "0,0,1,";
    default: return ",,,";
    }
}

// Rules 3 and 4: the line of published record r whose aircraft id is `id`, stamped secs + frac, into out (at least
// AMB_SBS1_MAX_LINE bytes, no terminator). Returns its length, or 0 for a record that writes no line.
AMB_HD int amb_sbs1_line(const amb_fields* r, uint64_t id, uint64_t secs, double frac, int tz_min, char* out)
{
    const unsigned df = r->df, st = r->status;
    const char* kind;
    if (df == 0) kind = "MSG,7,0,";
    else if (df == 4) kind = "MSG,5,0,";
    else if (df == 5) kind = "MSG,6,0,";
    else if (df == 11) kind = "MSG,8,0,";
    else if (r->bds == 0x08) kind = "MSG,1,0,";
    else if (r->bds == 0x06) kind = "MSG,2,0,";
    else if (r->bds == 0x05) kind = "MSG,3,0,";
    else if (r->bds == 0x09 && r->subtype == 1) kind = "MSG,4,0,";
    else return 0;                                      // BDS0,9 subtypes 0 (ValueError) and 3, BDS6,1: no line
    if ((df == 0 || df == 4) && (st & AMB_FS_METRIC_ALT)) return 0;              // MetricAltError
    if (df == 17 && (r->bds == 0x05 || r->bds == 0x06) && !(st & AMB_FS_HAS_POS)) return 0;
    if (df == 17 && r->bds == 0x08) {                   // categories[ftc - 1][cat] (parse.py:275): IndexError
        const unsigned n = r->ftc == 2 ? 7u : 8u;
        if (r->ftc < 1 || r->ftc > 4 || r->cat >= n) return 0;
    }
    char date[10], tod[12];
    const bool stamped = amb_sbs1_stamp(secs, frac, tz_min, date, tod);
    char* p = amb_sbs1_str(out, kind);
    p = amb_sbs1_u64(p, id); *p++ = ',';
    p = amb_sbs1_hex6(p, r->icao); *p++ = ',';
    p = amb_sbs1_u64(p, id + 100);
    for (int i = 0; i < 2; i++) {
        *p++ = ',';
        if (stamped) { memcpy(p, date, 10); p += 10; }
        *p++ = ',';
        if (stamped) { memcpy(p, tod, 12); p += 12; }
    }
    if (df == 0) {
        p = amb_sbs1_str(p, ",,"); p = amb_sbs1_i64(p, r->altitude);
        p = amb_sbs1_str(p, r->vs ? ",,,,,,,,,,1\r\n" : ",,,,,,,,,,0\r\n");
    } else if (df == 4) {
        p = amb_sbs1_str(p, ",,"); p = amb_sbs1_i64(p, r->altitude);
        p = amb_sbs1_str(p, ",,,,,,,"); p = amb_sbs1_str(p, amb_sbs1_fs(r->fs)); p = amb_sbs1_str(p, "\r\n");
    } else if (df == 5) {
        p = amb_sbs1_str(p, ",,,,,,,,");
        if (r->squawk < 0) { *p++ = '-'; p = amb_sbs1_dec(p, (unsigned)-r->squawk, 3); }   // '%04i' of a negative
        else if (r->squawk < 10000) p = amb_sbs1_dec(p, (unsigned)r->squawk, 4);
        else p = amb_sbs1_i64(p, r->squawk);
        *p++ = ','; p = amb_sbs1_str(p, amb_sbs1_fs(r->fs)); p = amb_sbs1_str(p, "\r\n");
    } else if (df == 11) {
        p = amb_sbs1_str(p, ",,,,,,,,,,,,\r\n");
    } else if (r->bds == 0x08) {
        *p++ = ',';
        for (int i = 0; i < 8; i++) *p++ = r->ident[i];
        p = amb_sbs1_str(p, ",,,,,,,,,,,\r\n");
    } else if (r->bds == 0x06 || r->bds == 0x05) {
        p = amb_sbs1_str(p, ",,");
        p = amb_sbs1_i64(p, r->bds == 0x06 ? 0 : r->altitude);
        p = amb_sbs1_str(p, ",,,");
        if (!(p = amb_sbs1_fixed(p, r->lat, 5))) return 0;
        *p++ = ',';
        if (!(p = amb_sbs1_fixed(p, r->lon, 5))) return 0;
        p = amb_sbs1_str(p, ",,,,0,0,0\r\n");
    } else {
        p = amb_sbs1_str(p, ",,,");
        if (!(p = amb_sbs1_fixed(p, r->val[0], 1))) return 0;
        *p++ = ',';
        if (!(p = amb_sbs1_fixed(p, r->val[1], 1))) return 0;
        p = amb_sbs1_str(p, ",,,");
        if (!(p = amb_sbs1_trunc(p, r->val[2]))) return 0;
        p = amb_sbs1_str(p, ",,,,,\r\n");
    }
    return (int)(p - out);
}
