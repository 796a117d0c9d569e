// Per-message decode arithmetic of SURVEY.md 8 row f4: what the reference's python/parse.py, python/altitude.py and
// python/cpr.py compute for one queued message, as __host__ __device__ functions. The CUDA kernels in amb_decode.cu
// are the only product code that calls them; tests/decode_host_shim.cc compiles the same functions for the host so
// that the arithmetic is checked against the reference's golden where no GPU is present (a test harness, not a
// product path). Citations are file:line under gr-air-modes/python.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/airmodes_b200.h"

#if defined(__CUDACC__)
#define AMB_HD __host__ __device__ __forceinline__
#else
#define AMB_HD static inline
#endif

#define AMB_NO_KEY 0xFFFFFFFFu
#define AMB_NL_MAX 64            // nl_T[k]: smallest |lat| at which cpr.py:48-51 evaluates below k (k = 3..nl_T[0])

// A CPR report as the pairing stage sees it (cpr.py:214-221: [encoded_lat, encoded_lon, time] per icao, per
// even/odd, per airborne/surface list).
struct AmbPosRec {
    uint32_t key;        // (icao24 << 1) | surface; AMB_NO_KEY = not a position message
    uint32_t lat, lon;   // 17-bit encoded values
    uint32_t fmt;        // 0 even, 1 odd ("cpr" field, parse.py:126-127)
    double t;            // secs + frac of the message
};

// What the pairing stage found for a position message: the latest even and odd report of its aircraft that are
// still alive (cpr.py:196-204), and which is newer (cpr.py:229).
struct AmbPair {
    uint32_t elat, elon, olat, olon;
    int have, mostrecent;
};

// ---- bit fields: data_field.get_bits (parse.py:71-87), fields 1-based from the MSB ---------------------------------
struct AmbMsg { uint64_t w0, w1; int numbits; };   // message bits 1..64 in w0 (MSB first), 65..112 in the top of w1

AMB_HD uint64_t amb_bits(const AmbMsg& m, int s, int n)
{
    if (s + n - 1 > m.numbits) return 0;            // negative shift -> ValueError -> field reads 0 (parse.py:83-86)
    const int a = s - 1;
    uint64_t x;
    if (a == 0) x = m.w0;
    else if (a < 64) x = (m.w0 << a) | (m.w1 >> (64 - a));
    else x = m.w1 << (a - 64);
    return x >> (64 - n);
}

AMB_HD AmbMsg amb_msg_from_frame(const amb_frame& f)
{
    AmbMsg m;
    uint64_t hi = 0, lo = 0;
    for (int k = 0; k < 7; k++) hi = (hi << 8) | f.data[k];
    if (f.nbits == 112) {
        for (int k = 7; k < 14; k++) lo = (lo << 8) | f.data[k];
        // modes_reply.is_long: int(data, 16) > (1 << 56) (parse.py:222-223)
        if (hi > 1 || (hi == 1 && lo > 0)) {
            m.w0 = (hi << 8) | (lo >> 48); m.w1 = lo << 16; m.numbits = 112;
        } else {                                    // a 28-digit string with a small value parses as a short reply
            m.w0 = lo << 8; m.w1 = 0; m.numbits = 56;
        }
    } else {
        m.w0 = hi << 8; m.w1 = 0; m.numbits = 56;
    }
    return m;
}

// ---- altitude.py --------------------------------------------------------------------------------------------------
AMB_HD int amb_gray2bin(int g)                      // altitude.py:110-117
{
    for (int i = g >> 1; i != 0; i >>= 1) g ^= i;
    return g;
}

// decode_alt(alt, bit13) (altitude.py:28-108). Returns 0 and *feet, or 1 for MetricAltError (:32-43).
AMB_HD int amb_decode_alt(int alt, int bit13, int32_t* feet)
{
    if ((alt & 0x40) && bit13) return 1;
    if (alt & 0x10) {                               // Mode S style, 25 ft (:45-56)
        const int t = bit13 ? (((alt & 0x3F80) >> 2) | ((alt & 0x20) >> 1)) : ((alt & 0x1FE0) >> 1);
        *feet = ((alt & 0x0F) | t) * 25 - 1000;
        return 0;
    }
    if (!bit13) alt = (alt & 0x3F) | (alt & (0x0FC0 << 1));      // :67 exactly as written (operator precedence)
    const int big = ((alt & 0x0002) >> 1) + ((alt & 0x0008) >> 2) + ((alt & 0x0020) >> 3) + ((alt & 0x0080) >> 4) +
                    ((alt & 0x0200) >> 5) + ((alt & 0x0800) >> 6) + ((alt & 0x0001) << 6) + ((alt & 0x0004) << 5);   // :82-89
    int d = amb_gray2bin(big);
    int c = amb_gray2bin(((alt & 0x0100) >> 8) + ((alt & 0x0400) >> 9) + ((alt & 0x1000) >> 10));               // :95-96
    if (c == 7) c = 5;
    if (d % 2) c = 6 - c;
    *feet = d * 500 + c * 100 - 1300;               // :104-106
    return 0;
}

AMB_HD int amb_decode_id(int v)                     // parse.py:233-254
{
    const int a = ((v & 0x0800) >> 11) + ((v & 0x0200) >> 8) + ((v & 0x0080) >> 5);
    const int b = ((v & 0x0020) >> 5) + ((v & 0x0008) >> 2) + ((v & 0x0002) << 1);
    const int c = ((v & 0x1000) >> 12) + ((v & 0x0400) >> 9) + ((v & 0x0100) >> 6);
    const int d = ((v & 0x0010) >> 2) + ((v & 0x0004) >> 1) + ((v & 0x0001) << 2);
    return a * 1000 + b * 100 + c * 10 + d;
}

AMB_HD void amb_ident48(uint64_t v, char* out)      // charmap + parseBDS08 / parseMB_id (parse.py:257-279, 374-378)
{
    for (int i = 0; i < 8; i++) {
        const int d = (int)((v >> (42 - 6 * i)) & 0x3F);
        char ch = ' ';
        if (d > 0 && d < 27) ch = (char)('A' + d - 1);
        else if (d > 47 && d < 58) ch = (char)('0' + d - 48);
        out[i] = ch;
    }
}

// ---- one message -> fields (everything but the CPR resolution) ------------------------------------------------------
AMB_HD void amb_fields_blank(amb_fields* r, int df, uint32_t ecc)
{
    r->icao = ecc; r->ecc = ecc;
    r->df = (uint8_t)df; r->status = 0; r->bds = 0; r->subtype = 0xFF;
    r->ca = r->fs = r->vs = r->ri = 0; r->sl = r->cc = r->dr = r->um = 0;
    r->ftc = r->cat = r->cpr_format = r->surface = 0; r->eps = r->ast = r->bds2 = r->tti = 0;
    r->altitude = AMB_NO_ALTITUDE; r->squawk = -1; r->threat_alt = AMB_NO_ALTITUDE;
    r->cpr_lat = r->cpr_lon = 0;
    for (int k = 0; k < 4; k++) { r->aux[k] = 0; r->val[k] = NAN; }
    for (int k = 0; k < 8; k++) r->ident[k] = 0;
    r->lat = r->lon = r->range = r->bearing = NAN;
    r->pad_ = 0;
}

AMB_HD void amb_alt_into(amb_fields* r, int code, int bit13, int32_t* dst, int flag = AMB_FS_METRIC_ALT)
{
    int32_t feet;
    if (amb_decode_alt(code, bit13, &feet)) r->status |= (uint8_t)flag;
    else *dst = feet;
}

// The reference's parser raises NoHandlerError while building the field dict, so nothing of the message survives
// (parse.py:52-68, make_parser :431-434): keep only what identifies it.
AMB_HD void amb_no_handler(amb_fields* r, int keep_icao)
{
    const uint32_t icao = r->icao, ecc = r->ecc; const int df = r->df;
    amb_fields_blank(r, df, ecc);
    if (keep_icao) r->icao = icao;
    r->status = AMB_FS_NO_HANDLER;
}

// modes_reply / me_reply / bds09_reply / mb_reply / tcas_reply field tables (parse.py:89-220) and the parseBDS*
// functions (parse.py:276-372). pos->key stays AMB_NO_KEY unless the message is a BDS0,5 / BDS0,6 position.
AMB_HD void amb_decode_fields(const amb_frame& f, amb_fields* r, AmbPosRec* pos)
{
    pos->key = AMB_NO_KEY; pos->lat = pos->lon = 0; pos->fmt = 0;
    pos->t = (double)f.secs + f.frac;
    const AmbMsg g = amb_msg_from_frame(f);
    const int df = (int)amb_bits(g, 1, 5);
    amb_fields_blank(r, df, f.crc);
    if (!f.passed) { r->status = AMB_FS_NOT_QUEUED; return; }
    if (!(df == 0 || df == 4 || df == 5 || df == 11 || df == 16 || df == 17 || df == 20 || df == 21 || df == 24)) {
        r->status = AMB_FS_NO_HANDLER;              // parse.py:210-220 has no table for this DF
        return;
    }
    if (df == 0 || df == 16) {
        r->vs = (uint8_t)amb_bits(g, 6, 1); r->sl = (uint8_t)amb_bits(g, 9, 3); r->ri = (uint8_t)amb_bits(g, 14, 4);
        if (df == 0) r->cc = (uint8_t)amb_bits(g, 7, 1);
        amb_alt_into(r, (int)amb_bits(g, 20, 13), 1, &r->altitude);          // msprint.py:64,251
    } else if (df == 4 || df == 5 || df == 20 || df == 21) {
        r->fs = (uint8_t)amb_bits(g, 6, 3); r->dr = (uint8_t)amb_bits(g, 9, 5); r->um = (uint8_t)amb_bits(g, 14, 6);
        if (df >= 20) {
            // "mb": (33,56, mb_reply) (parse.py:218-219): the sub-fields are read from that 56-bit word, which is 0 when
            // the reply is short (negative shift, parse.py:83-86). b(s, n) = mb_reply/tcas_reply field at message bit s.
            AmbMsg mb; mb.w0 = amb_bits(g, 33, 56) << 8; mb.w1 = 0; mb.numbits = 56;
#define AMB_MB(s, n) amb_bits(mb, (s) - 32, (n))
            const int bds1 = (int)AMB_MB(33, 4), bds2 = (int)AMB_MB(37, 4);
            r->bds = (uint8_t)bds1; r->bds2 = (uint8_t)bds2;
            if (bds1 > 3 || bds2 != 0) { amb_no_handler(r, 0); return; }     // parse.py:185-190
            if (bds1 == 1) {
                r->aux[0] = (uint32_t)AMB_MB(45, 20); r->aux[1] = (uint32_t)AMB_MB(65, 16);
                r->aux[2] = (uint32_t)AMB_MB(81, 8);  r->aux[3] = (uint32_t)AMB_MB(41, 4);   // acs, bcs, ecs, cfs
            } else if (bds1 == 2) {
                amb_ident48(AMB_MB(41, 48), r->ident);                      // parse.py:374-378
            } else if (bds1 == 3) {
                const int tti = (int)AMB_MB(61, 2);
                r->tti = (uint8_t)tti;
                if (tti == 3) { amb_no_handler(r, 0); return; }              // tcas_reply has types 0-2 (parse.py:157-165)
                r->aux[0] = (uint32_t)AMB_MB(41, 14); r->aux[1] = (uint32_t)AMB_MB(55, 4);
                r->aux[2] = (uint32_t)(AMB_MB(59, 1) | (AMB_MB(60, 1) << 1));   // rat | mte << 1
                if (tti == 1) r->aux[3] = (uint32_t)AMB_MB(63, 26);          // tid
                else if (tti == 2) {
                    r->aux[3] = (uint32_t)(AMB_MB(76, 7) | (AMB_MB(83, 6) << 8));   // tidr | tidb << 8
                    amb_alt_into(r, (int)AMB_MB(63, 13), 1, &r->threat_alt, AMB_FS_METRIC_THREAT);   // parse.py:407
                }
            }
#undef AMB_MB
        }
        if (df == 4 || df == 20) amb_alt_into(r, (int)amb_bits(g, 20, 13), 1, &r->altitude);
        else r->squawk = amb_decode_id((int)amb_bits(g, 20, 13));
    } else if (df == 11) {
        r->ca = (uint8_t)amb_bits(g, 6, 3); r->icao = (uint32_t)amb_bits(g, 9, 24);
    } else if (df == 17) {
        r->ca = (uint8_t)amb_bits(g, 6, 3); r->icao = (uint32_t)amb_bits(g, 9, 24);
        AmbMsg m; m.w0 = amb_bits(g, 33, 56) << 8; m.w1 = 0; m.numbits = 56;       // "me" (parse.py:217)
        const int ftc = (int)amb_bits(m, 1, 5);
        r->ftc = (uint8_t)ftc;
        if (ftc >= 1 && ftc <= 4) {                                         // parse.py:140-152 maps ftc to the BDS register
            r->bds = 0x08;
            r->cat = (uint8_t)amb_bits(m, 6, 3);
            amb_ident48(amb_bits(m, 9, 48), r->ident);
        } else if (ftc >= 5 && ftc <= 8) {
            r->bds = 0x06; r->surface = 1;
            r->cpr_format = (uint8_t)amb_bits(m, 22, 1);
            r->cpr_lat = (uint32_t)amb_bits(m, 23, 17); r->cpr_lon = (uint32_t)amb_bits(m, 40, 17);
            r->val[0] = (double)(int)amb_bits(m, 14, 7) * 360. / 128;        // parse.py:283
            pos->key = (r->icao << 1) | 1u;
        } else if (ftc >= 9 && ftc <= 18 && ftc != 15) {
            r->bds = 0x05;
            r->cpr_format = (uint8_t)amb_bits(m, 22, 1);
            r->cpr_lat = (uint32_t)amb_bits(m, 23, 17); r->cpr_lon = (uint32_t)amb_bits(m, 40, 17);
            amb_alt_into(r, (int)amb_bits(m, 9, 12), 0, &r->altitude);       // parse.py:277
            pos->key = (r->icao << 1);
        } else if (ftc == 19) {
            r->bds = 0x09;
            const int sub = (int)amb_bits(m, 6, 3);
            if (sub == 0) {                                                 // parseBDS09_0 (parse.py:288-313)
                r->subtype = 0;
                int vs = (int)amb_bits(m, 42, 9) * 32;
                if (amb_bits(m, 41, 1)) vs = 0 - vs;
                double tr = (double)((int)amb_bits(m, 35, 6) * 15) / 62;
                if (amb_bits(m, 34, 1)) tr = 0 - tr;
                int ns = (int)amb_bits(m, 23, 11) - 1, ew = (int)amb_bits(m, 11, 11) - 1;
                // hypot of integers: the root of the exact integer sum is correctly rounded (device hypot is not: one
                // ulp off in about a quarter of the words, perfect squares included) - DESIGN.md §8
                const double vel = sqrt((double)(ns * ns + ew * ew));
                if (amb_bits(m, 10, 1)) ew = 0 - ew;
                if (amb_bits(m, 22, 1)) ns = 0 - ns;
                double hdg = atan2((double)ew, (double)ns) * (180.0 / M_PI);
                if (hdg < 0) hdg += 360;
                r->val[0] = vel; r->val[1] = hdg; r->val[2] = (double)vs; r->val[3] = tr;
            } else if (sub == 1 || sub == 2) {                              // parseBDS09_1 (parse.py:315-348)
                r->subtype = 1;
                int geo = (int)amb_bits(m, 50, 6) * 25;
                if (amb_bits(m, 49, 1)) geo = 0 - geo;
                double vs = (double)((int)amb_bits(m, 38, 9) - 1) * 64;
                if (amb_bits(m, 37, 1)) vs = 0 - vs;
                double ns = (double)(int)amb_bits(m, 26, 10), ew = (double)(int)amb_bits(m, 15, 10);
                if (sub == 2) { ns *= 4; ew *= 4; }
                const double vel = sqrt(ns * ns + ew * ew);                 // exact sum (< 2^25), as above
                if (amb_bits(m, 14, 1)) ew = 0 - ew;
                double hdg = (ns == 0) ? 0.0 : atan(ew / ns) * (180.0 / M_PI);
                if (amb_bits(m, 25, 1)) hdg = 180 - hdg;
                if (hdg < 0) hdg += 360;
                r->val[0] = vel; r->val[1] = hdg; r->val[2] = vs; r->val[3] = (double)geo;
            } else if (sub == 3 || sub == 4) {                              // parseBDS09_3 (parse.py:350-364)
                r->subtype = 3;
                r->ast = (uint8_t)amb_bits(m, 25, 1);
                int vel = (int)amb_bits(m, 26, 10);
                if (sub == 4) vel *= 4;
                double vs = (double)((int)amb_bits(m, 38, 9) - 1) * 64;
                if (amb_bits(m, 37, 1) == 1) vs = 0 - vs;
                r->val[0] = (double)(int)amb_bits(m, 14, 1) * 360. / 1024;   // :353 reads "mhs", the 1-bit status field
                r->val[1] = (double)vel; r->val[2] = vs;
                r->val[3] = (double)((int)amb_bits(m, 50, 6) - 1) * 25;
            } else {                                                        // bds09_reply.get_type() -> None (parse.py:110-117)
                amb_no_handler(r, 1); return;
            }
        } else if (ftc == 28) {
            r->bds = 0x61;
            r->eps = (uint8_t)amb_bits(m, 9, 3);
        } else {
            amb_no_handler(r, 1); return;
        }
        if (pos->key != AMB_NO_KEY) { pos->lat = r->cpr_lat; pos->lon = r->cpr_lon; pos->fmt = r->cpr_format; }
    }
    /* df == 24: "ke"/"nd"/"md" have no consumer in the reference */
}

// ---- cpr.py ---------------------------------------------------------------------------------------------------------
// nl(declat_in) (cpr.py:46-51) through the transition table built by amb_build_nl_table() from the same libm
// expression: the value is floor(f(|lat|)) with f decreasing, so NL = the largest k with |lat| < T[k].
AMB_HD int amb_nl(double lat, const double* T)
{
    const double a = fabs(lat);
    if (a >= 87.0) return 1;
    for (int k = (int)T[0]; k >= 3; k--)
        if (a < T[k]) return k;
    return 2;
}

AMB_HD long long amb_pymod(long long a, long long b)     // Python's % for b > 0
{
    const long long r = a % b;
    return r < 0 ? r + b : r;
}

// cpr_resolve_global (cpr.py:89-153). 0 = ok, AMB_FS_CPR_NO_POS, or AMB_FS_CPR_NO_POS | AMB_FS_CPR_STRADDLE.
AMB_HD int amb_cpr_global(const AmbPair& pr, int surface, int have_loc, double mylat, double mylon, const double* T,
                          double* out_lat, double* out_lon)
{
    if (surface && !have_loc) return AMB_FS_CPR_NO_POS;                     // :97-99
    const double span = surface ? 90.0 : 360.0;                             // dlat/dlon (:37-45, :53-59)
    const double dle = span / 60, dlo = span / 59;
    const double elat = (double)pr.elat, elon = (double)pr.elon, olat = (double)pr.olat, olon = (double)pr.olon;
    const long long j = (long long)floor(((59 * elat - 60 * olat) / 131072) + 0.5);                 // :107
    double rle = dle * ((double)amb_pymod(j, 60) + elat / 131072);          // :109
    double rlo = dlo * ((double)amb_pymod(j, 59) + olat / 131072);          // :110
    if (rle > 270.0) rle -= 360.0;
    if (rlo > 270.0) rlo -= 360.0;
    if (amb_nl(rle, T) != amb_nl(rlo, T)) return AMB_FS_CPR_NO_POS | AMB_FS_CPR_STRADDLE;           // :120-121
    double rlat = pr.mostrecent ? rlo : rle;
    if (surface && mylat < 0) rlat -= 90;                                   // :129-131
    const int n = amb_nl(rlat, T);
    const int nn = (n - pr.mostrecent) > 1 ? (n - pr.mostrecent) : 1;
    const double dl = span / nn;                                            // dlon(rlat, mostrecent, surface) :133
    const long long m = (long long)floor(((elon * (n - 1) - olon * n) / 131072) + 0.5);             // :136
    const double enclon = pr.mostrecent ? olon : elon;
    double rlon = dl * ((double)amb_pymod(m, nn) + enclon / 131072.);       // :147
    if (surface) {                                                          // :152-158, `zone` with Python-3 true division
        double wat = mylon;
        if (wat < 0) wat += 360;
        const double za = 90 * ((double)(long long)wat / 90), zb = 90 * ((double)(long long)rlon / 90);
        rlon += (za - zb);
    }
    if (rlon > 180) rlon -= 360.0;                                          // :160-162
    *out_lat = rlat; *out_lon = rlon;
    return 0;
}

AMB_HD void amb_range_bearing(double a_lat, double a_lon, double b_lat, double b_lon, double* rnge, double* bearing)
{                                                                           // cpr.py:158-181
    const double esquared = (1 / 298.257223563) * (2 - (1 / 298.257223563));
    const double earth_radius_mi = 3963.19059 * (M_PI / 180);
    const double delta_lat = b_lat - a_lat, delta_lon = b_lon - a_lon;
    const double avg_lat = ((a_lat + b_lat) / 2.0) * M_PI / 180;
    const double s2 = pow(sin(avg_lat), 2.0);
    const double R1 = earth_radius_mi * (1.0 - esquared) / pow((1.0 - esquared * s2), 1.5);
    const double R2 = earth_radius_mi / sqrt(1.0 - esquared * s2);
    const double north = R1 * delta_lat;
    const double east = R2 * cos(avg_lat) * delta_lon;
    double b = atan2(east, north) * (180.0 / M_PI);
    if (b < 0.0) b += 360.0;
    *rnge = hypot(east, north);
    *bearing = b;
}

// parseBDS05 / parseBDS06 tail (parse.py:276-286) + cpr_decoder.decode after the pair lookup (cpr.py:226-240).
AMB_HD void amb_resolve_position(amb_fields* r, const AmbPair& pr, int have_loc, double mylat, double mylon, const double* T)
{
    if (!pr.have) { r->status |= AMB_FS_CPR_NO_POS; return; }               // cpr.py:231
    double lat, lon;
    const int e = amb_cpr_global(pr, r->surface, have_loc, mylat, mylon, T, &lat, &lon);
    if (e) { r->status |= (uint8_t)e; return; }
    r->lat = lat; r->lon = lon; r->status |= AMB_FS_HAS_POS;
    if (have_loc) {
        amb_range_bearing(mylat, mylon, lat, lon, &r->range, &r->bearing);
        r->status |= AMB_FS_HAS_RANGE;
    }
}

// ---- locally referenced CPR decode (decoder option "local_cpr"; DESIGN.md §8) --------------------------------------
// The last position of an aircraft (global or local fix) and the timestamp of its message; t is NaN when there is none.
struct AmbRefPos { double lat, lon, t; };

AMB_HD double amb_pyfmod(double a, double b)                // Python's float % for b > 0 (float_rem: fmod + sign fix-up)
{
    double m = fmod(a, b);
    if (m != 0.0) { if (m < 0.0) m += b; }
    else m = 0.0;                                           // copysign(0, b)
    return m;
}

// cpr_resolve_local (cpr.py:75-82 with decode_lat :61-66, decode_lon :68-73, dlat :36-46, dlon :53-59), expression by
// expression; nl() from the transition table.
AMB_HD void amb_cpr_local(double my_lat, double my_lon, uint32_t enclat, uint32_t enclon, int ctype, int surface,
                          const double* T, double* out_lat, double* out_lon)
{
    const double span = surface ? 90.0 : 360.0;
    const double dla = span / (60 - ctype);
    const double la2 = (double)enclat / 131072;
    const double j = floor(my_lat / dla) + floor(0.5 + (amb_pyfmod(my_lat, dla) / dla) - la2);
    const double lat = dla * (j + la2);
    const int nn = (amb_nl(lat, T) - ctype) > 1 ? (amb_nl(lat, T) - ctype) : 1;
    const double dlo = span / nn;
    const double lo2 = (double)enclon / 131072;
    const double m = floor(my_lon / dlo) + floor(0.5 + (amb_pyfmod(my_lon, dlo) / dlo) - lo2);
    *out_lat = lat;
    *out_lon = dlo * (m + lo2);
}

// One position message after the global resolve, given its aircraft's reference position `ref` as of this message
// (updated in place). Returns the AMB_LOCAL_* outcome, which is also stored in the record.
AMB_HD int amb_local_step(amb_fields* r, double t, AmbRefPos* ref, int max_age, int have_loc, double mylat, double mylon,
                          const double* T)
{
    int v;
    if (r->status & AMB_FS_HAS_POS) {                       // the global fix stands and becomes the reference
        ref->lat = r->lat; ref->lon = r->lon; ref->t = t;
        v = AMB_LOCAL_NOT_TRIED;
    } else if (ref->t != ref->t) {
        v = AMB_LOCAL_NO_REF;
    } else if (!(t - ref->t >= 0.0) || t - ref->t > (double)max_age) {   // the expiry rule of amb_report_alive
        v = AMB_LOCAL_STALE;
    } else {
        double lat, lon;
        amb_cpr_local(ref->lat, ref->lon, r->cpr_lat, r->cpr_lon, r->cpr_format, r->surface, T, &lat, &lon);
        if (lon > 180.0) lon -= 360.0;
        else if (lon <= -180.0) lon += 360.0;
        const double dla = (r->surface ? 90.0 : 360.0) / (60 - r->cpr_format);
        if (fabs(lat) > 90.0 || fabs(lat - ref->lat) > dla / 2) {
            v = AMB_LOCAL_REJECTED;
        } else {
            r->lat = lat; r->lon = lon; r->status |= AMB_FS_HAS_POS;
            if (have_loc) {
                amb_range_bearing(mylat, mylon, lat, lon, &r->range, &r->bearing);
                r->status |= AMB_FS_HAS_RANGE;
            }
            ref->lat = lat; ref->lon = lon; ref->t = t;
            v = AMB_LOCAL_DECODED;
        }
    }
    AMB_FIELDS_LOCAL(r) = (uint8_t)v;
    return v;
}

// ---- Comm-B register inference (decoder option "commb"; DESIGN.md §8 "Comm-B inference") --------------------------
// The ADS-B velocity of an address as of a message: t, speed (val[0]) and track (val[1]) of its latest DF17 BDS0,9
// subtype 0/1 record; t is NaN when there is none.
struct AmbCommbRef { double t, speed, track; };

#define AMB_COMMB_R40 0x1u
#define AMB_COMMB_R50 0x2u
#define AMB_COMMB_R60 0x4u

// The MB word of a record the stage tries: MB bit k (1..56) is bit 56 - k of the result.
AMB_HD uint64_t amb_commb_mb(const amb_frame& f) { return amb_bits(amb_msg_from_frame(f), 33, 56); }

AMB_HD int amb_commb_count(unsigned c) { return (int)(c & 1u) + (int)((c >> 1) & 1u) + (int)((c >> 2) & 1u); }

AMB_HD unsigned amb_commb_bits(uint64_t mb, int s, int n) { return (unsigned)((mb >> (57 - s - n)) & ((1ull << n) - 1)); }

// Field i of register g (0 = 4,0, 1 = 5,0, 2 = 6,0): status bit, first value bit (the sign bit of a signed field) and
// width (sign included), packed as status | first << 8 | width << 16 | signed << 24 (the table in include/airmodes_b200.h).
AMB_HD unsigned amb_commb_spec(int g, int i)
{
#define AMB_CS(st, first, w, sg) ((st) | ((first) << 8) | ((w) << 16) | ((sg) << 24))
    switch (g * 5 + i) {
    case 0: return AMB_CS(1, 2, 12, 0);   case 1: return AMB_CS(14, 15, 12, 0);  case 2: return AMB_CS(27, 28, 12, 0);
    case 3: return AMB_CS(48, 49, 3, 0);  case 4: return AMB_CS(54, 55, 2, 0);
    case 5: return AMB_CS(1, 2, 10, 1);   case 6: return AMB_CS(12, 13, 11, 1);  case 7: return AMB_CS(24, 25, 10, 0);
    case 8: return AMB_CS(35, 36, 10, 1); case 9: return AMB_CS(46, 47, 10, 0);
    case 10: return AMB_CS(1, 2, 11, 1);  case 11: return AMB_CS(13, 14, 10, 0); case 12: return AMB_CS(24, 25, 10, 0);
    case 13: return AMB_CS(35, 36, 10, 1); default: return AMB_CS(46, 47, 10, 1);
    }
#undef AMB_CS
}

// Read register g out of mb: raw values of fields 0..4 (0 when absent) and their status bits; returns 1 when the register
// is a candidate (status/value consistency, at least one field, reserved bits 0, plausible values).
AMB_HD int amb_commb_read(uint64_t mb, int g, int raw[5], unsigned* mask)
{
    unsigned m = 0;
    int ok = 1;
    for (int i = 0; i < 5; i++) {
        const unsigned sp = amb_commb_spec(g, i);
        const int first = (int)((sp >> 8) & 0xFF), w = (int)((sp >> 16) & 0xFF);
        const unsigned v = amb_commb_bits(mb, first, w);
        raw[i] = 0;
        if (amb_commb_bits(mb, (int)(sp & 0xFF), 1)) {
            m |= 1u << i;
            raw[i] = (sp >> 24) && (v >> (w - 1)) ? (int)v - (1 << w) : (int)v;
        } else if (v) {
            ok = 0;                                         // data behind a status bit of 0
        }
    }
    if (!m) ok = 0;
    const int abs0 = raw[0] < 0 ? -raw[0] : raw[0], abs3 = raw[3] < 0 ? -raw[3] : raw[3];
    const int abs4 = raw[4] < 0 ? -raw[4] : raw[4];
    if (g == 0) {
        if (amb_commb_bits(mb, 40, 8) || amb_commb_bits(mb, 52, 2)) ok = 0;
        if (raw[0] > 3125 || raw[1] > 3125 || ((m & 4u) && (raw[2] < 700 || raw[2] > 3000))) ok = 0;
    } else if (g == 1) {
        const int d = raw[2] - raw[4];
        if (abs0 > 284 || raw[2] > 400 || raw[4] > 300 || ((m & 4u) && (m & 16u) && (d > 125 || d < -125))) ok = 0;
    } else {
        if (raw[1] > 500 || raw[2] > 250 || abs3 > 187 || abs4 > 187) ok = 0;
    }
    *mask = m;
    return ok;
}

AMB_HD unsigned amb_commb_candidates(uint64_t mb)
{
    unsigned c = 0;
    for (int g = 0; g < 3; g++) {
        int raw[5]; unsigned m;
        if (amb_commb_read(mb, g, raw, &m)) c |= 1u << g;
    }
    return c;
}

// The record the stage tries: queued, DF20/21, 112 bits, status exactly AMB_FS_NO_HANDLER, and an MB first byte that
// is not one of the parser's registers (those stay the parser's, as in the reference).
AMB_HD int amb_commb_eligible(const amb_frame& f, const amb_fields* r)
{
    if (!f.passed || f.nbits != 112 || r->status != AMB_FS_NO_HANDLER || (r->df != 20 && r->df != 21)) return 0;
    const unsigned b1 = amb_commb_bits(amb_commb_mb(f), 1, 8);
    return !((b1 & 0x0F) == 0 && (b1 >> 4) <= 3);
}

// A record that carries its address's ADS-B velocity: queued DF17 BDS0,9 subtype 0/1 with speed and track.
AMB_HD int amb_commb_is_ref(const amb_fields* r)
{
    return !(r->status & AMB_FS_NOT_QUEUED) && r->df == 17 && r->bds == 0x09 && (r->subtype == 0 || r->subtype == 1) &&
           r->val[0] == r->val[0] && r->val[1] == r->val[1];
}

// Does a 5,0 reading agree with the ADS-B speed and track? (fp64, no contraction: the decoder is built -fmad=false)
AMB_HD int amb_commb_agree(int gs_raw, int trk_raw, double speed, double track)
{
    const double trk = (double)trk_raw * 90.0 / 512.0;
    double d = fmod(fabs(trk - track), 360.0);
    d = d < 360.0 - d ? d : 360.0 - d;
    return fabs(2.0 * (double)gs_raw - speed) <= 20.0 && d <= 10.0;
}

// Does the reference rule apply to this word? (5,0 among several candidates, with GS and track present)
AMB_HD int amb_commb_needs_ref(uint64_t mb, unsigned cand)
{
    if (!(cand & AMB_COMMB_R50) || amb_commb_count(cand) < 2) return 0;
    int raw[5]; unsigned m;
    amb_commb_read(mb, 1, raw, &m);
    return (m & 0x6u) == 0x6u;
}

// Write the outcome into the record: aux = raw values of register g (g < 0: none), pad_ bytes 1..4.
AMB_HD void amb_commb_write(amb_fields* r, uint64_t mb, unsigned cand, int outcome, int g)
{
    int raw[5] = {0, 0, 0, 0, 0};
    unsigned m = 0;
    if (g >= 0) amb_commb_read(mb, g, raw, &m);
    r->aux[0] = (uint32_t)(uint16_t)raw[0] | ((uint32_t)(uint16_t)raw[1] << 16);   // int16_t[8], little endian
    r->aux[1] = (uint32_t)(uint16_t)raw[2] | ((uint32_t)(uint16_t)raw[3] << 16);
    r->aux[2] = (uint32_t)(uint16_t)raw[4];
    r->aux[3] = 0;
    const uint64_t keep = r->pad_ & ~0xFFFFFFFF00ull;
    r->pad_ = keep | ((uint64_t)outcome << 8) | ((uint64_t)(g >= 0 ? 0x40 + 0x10 * g : 0) << 16) | ((uint64_t)m << 24) |
              ((uint64_t)cand << 32);
}

// One eligible record, given its address's velocity reference as of it (ref->t NaN: none). Returns the outcome.
AMB_HD int amb_commb_step(amb_fields* r, uint64_t mb, double t, const AmbCommbRef* ref, int max_age)
{
    unsigned c = amb_commb_candidates(mb);
    const unsigned cand = c;
    int v;
    if (!c) v = AMB_COMMB_NONE;
    else if (amb_commb_count(c) == 1) v = AMB_COMMB_DECODED;
    else {
        v = AMB_COMMB_AMBIGUOUS;
        if (amb_commb_needs_ref(mb, c) && ref->t == ref->t && t - ref->t >= 0.0 && t - ref->t <= (double)max_age) {
            int raw[5]; unsigned m;
            amb_commb_read(mb, 1, raw, &m);
            c = amb_commb_agree(raw[2], raw[1], ref->speed, ref->track) ? AMB_COMMB_R50 : (c & ~AMB_COMMB_R50);
            if (amb_commb_count(c) == 1) v = AMB_COMMB_RESOLVED;
        }
    }
    const int g = (v == AMB_COMMB_DECODED || v == AMB_COMMB_RESOLVED) ? (c == AMB_COMMB_R40 ? 0 : c == AMB_COMMB_R50 ? 1 : 2) : -1;
    amb_commb_write(r, mb, cand, v, g);
    return v;
}

// Latest-report bookkeeping of cpr_decoder.decode for ONE message given the table state before it (cpr.py:214-229):
// used by the pairing kernel lane by lane and, sequentially, by the host shim.
// A stored report stamped LATER than the current message can only stem from an earlier stream (frame timestamps restart
// after amb_reset / a new recording, while a decoder keeps its table): the reference's wall clock would have expired it
// long ago, so it counts as expired here too instead of being paired with (ADVICE round 1).
AMB_HD int amb_report_alive(double now, double t, int surface) { const double age = now - t; return age >= 0.0 && !(age > (surface ? 25.0 : 10.0)); }

// `me` has just been stored as the latest report of its format; (o_*) is the latest stored report of the other
// format, if any. -> what cpr_decoder.decode hands to cpr_resolve_global (cpr.py:226-229), or have = 0 (:231).
AMB_HD AmbPair amb_make_pair(const AmbPosRec& me, int o_have, uint32_t o_lat, uint32_t o_lon, double o_t)
{
    AmbPair pr; pr.have = 0; pr.mostrecent = 0; pr.elat = pr.elon = pr.olat = pr.olon = 0;
    if (o_have && amb_report_alive(me.t, o_t, (int)(me.key & 1u))) {       // weed_poslists (cpr.py:196-204)
        pr.have = 1;
        if (me.fmt) { pr.olat = me.lat; pr.olon = me.lon; pr.elat = o_lat; pr.elon = o_lon; pr.mostrecent = (me.t - o_t) > 0 ? 1 : 0; }
        else        { pr.elat = me.lat; pr.elon = me.lon; pr.olat = o_lat; pr.olon = o_lon; pr.mostrecent = (o_t - me.t) > 0 ? 1 : 0; }
    }
    return pr;
}

// Transition latitudes of nl() from the host libm, evaluated exactly as cpr.py:48-51 writes it (float ** 2 and
// float ** -1 are C pow() in CPython). T[0] = nl(0) = the largest NL; T[k], k = 3..T[0]. Host only: called once by
// amb_decoder_create, the table then lives in device memory.
static inline double amb_nl_formula(double x)
{
    const double c = cos(M_PI / (2.0 * 15));
    const double a = acos(1.0 - (1.0 - c) / pow(cos((M_PI / 180.0) * fabs(x)), 2.0));
    return floor((2.0 * M_PI) * pow(a, -1.0));
}
static inline void amb_build_nl_table(double* T)
{
    for (int k = 0; k < AMB_NL_MAX; k++) T[k] = 0.0;
    const int kmax = (int)amb_nl_formula(0.0);
    T[0] = (double)(kmax < AMB_NL_MAX ? kmax : AMB_NL_MAX - 1);
    for (int k = 3; k <= (int)T[0]; k++) {
        double lo = 0.0, hi = 86.99;                 // f(lo) >= k, f(hi) = 2 < k
        for (;;) {
            const double mid = lo + (hi - lo) / 2;
            if (!(mid > lo && mid < hi)) break;
            if (amb_nl_formula(mid) >= (double)k) lo = mid; else hi = mid;
        }
        T[k] = hi;
    }
}
