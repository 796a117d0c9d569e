// FlightGear multiplayer position packets of the decoder option "flightgear" (DESIGN.md §8 "FlightGear multiplayer
// feed"): which records the feed reads, the model of a BDS0,8 category, and the 232 bytes of one packet, byte for byte
// what the reference's fg_posmsg.pack (python/flightgear.py:134-206, with its Python 3 repair) writes for the same
// inputs. __host__ __device__: amb_decode_flightgear.cuh calls it on the device, tests/flightgear_host_shim.cc on the
// host. Every expression keeps the reference's operations and their order (Quaternion.py, mlat.py); the file is
// compiled without contraction (-fmad=false on the device, -ffp-contract=off on the host).
#pragma once
#include <string.h>

#include "amb_decode_core.h"

#define AMB_FG_PACKET 232        // '!4sLLLLL8s0L' (32 bytes) + '!96sdd3d3f3f3f3f3fI' (200 bytes)
#define AMB_FG_MODELS 16         // the 15 paths of modelmap (flightgear.py:116-132), then santa
#define AMB_FG_SANTA 15          // a category modelmap does not list
#define AMB_FG_KTS_MS 0.514444444                // flightgear.py:185

// What one published record does (include/airmodes_b200.h rules 1-4).
enum { AMB_FG_NONE = 0, AMB_FG_CALLSIGN = 1, AMB_FG_VELOCITY = 2, AMB_FG_POSITION = 3 };

// The model of BDS0,8 type code ftc (1..4) and category cat: categories[ftc - 1][cat] (parse.py:270-275) looked up in
// modelmap, santa where it has no entry; -1 where the row has no index cat (the reference raises IndexError). One
// nibble per category, cat 0 lowest.
AMB_HD int amb_fg_model(int ftc, int cat)
{
    const uint32_t rows[4] = {0xFFFFFFF0u, 0xFFFFFED0u, 0xCBFAF980u, 0x76543210u};
    if (ftc < 1 || ftc > 4 || cat < 0 || cat > 7 || (ftc == 2 && cat == 7)) return -1;   // the ftc 2 row has 7 entries
    return (int)((rows[ftc - 1] >> (4 * cat)) & 15u);
}

AMB_HD const char* amb_fg_model_path(int m)
{
    switch (m) {
    case 0: return "Aircraft/777-200/Models/777-200ER.xml";           // None, NO INFO
    case 1: return "Aircraft/c172p/Models/c172p.xml";                 // LIGHT
    case 2: return "Aircraft/CitationX/Models/Citation-X.xml";        // SMALL
    case 3: return "Aircraft/CRJ700-family/Models/CRJ700.xml";        // LARGE
    case 4: return "Aircraft/757-200/Models/757-200.xml";             // LARGE HIGH VORTEX
    case 5: return "Aircraft/IDG-A32X/Models/A320neo-CFM.xml";        // HEAVY
    case 6: return "Aircraft/SR71-BlackBird/Models/Blackbird-SR71B.xml";   // HIGH PERFORMANCE
    case 7: return "Aircraft/ec130/Models/ec130b4.xml";               // ROTORCRAFT
    case 8: return "Aircraft/ASK21-MI/Models/ask21mi.xml";            // GLIDER
    case 9: return "Aircraft/ZLT-NT/Models/ZLT-NT.xml";               // BALLOON/BLIMP
    case 10: return "Aircraft/cri-cri/Models/MC-15.xml";              // ULTRALIGHT
    case 11: return "Aircraft/YardStik/Models/yardstik.xml";          // UAV
    case 12: return "Aircraft/SpaceShip-One/Models/spaceshipone.xml"; // SPACECRAFT
    case 13: return "Aircraft/followme/Models/follow_me.xml";         // SURFACE EMERGENCY VEHICLE
    case 14: return "Aircraft/pushback/Models/Pushback.xml";          // SURFACE SERVICE VEHICLE
    default: return "Aircraft/santa/Models/santa.xml";
    }
}

// Rules 1-4: what record r does to its address's state (AMB_FG_*). A callsign needs a category in its row, a velocity
// subtype 0 or 1, a position AMB_FS_HAS_POS (a local fix counts).
AMB_HD int amb_fg_kind(const amb_fields* r)
{
    if ((r->status & (AMB_FS_NOT_QUEUED | AMB_FS_NO_HANDLER)) || r->df != 17) return AMB_FG_NONE;
    switch (r->bds) {
    case 0x08: return amb_fg_model(r->ftc, r->cat) >= 0 ? AMB_FG_CALLSIGN : AMB_FG_NONE;
    case 0x09: return r->subtype == 0 || r->subtype == 1 ? AMB_FG_VELOCITY : AMB_FG_NONE;
    case 0x05: case 0x06: return (r->status & AMB_FS_HAS_POS) ? AMB_FG_POSITION : AMB_FG_NONE;
    default: return AMB_FG_NONE;
    }
}

// Orientation of an aircraft at lat, lon (degrees) heading hdg (degrees): angle * axis of
// Quat([lat, lon]) * Quat([hdg, 0, 0]) (flightgear.py:174-181), as float32. Returns 0 where the reference raises
// TypeError (sin of the half angle, or the norm, below 1e-12): then no packet is written.
AMB_HD int amb_fg_orientation(double lat, double lon, double hdg, float* o)
{
    const double pi = M_PI;
    // _latlontoquat (Quaternion.py:356-372); _set_latlon keeps it as it is
    const double lon_r = lon * (pi / 180.), lat_r = lat * (pi / 180.);
    const double zd2 = 0.5 * lon_r, yd2 = -0.25 * pi - 0.5 * lat_r;
    const double Szd2 = sin(zd2), Syd2 = sin(yd2), Czd2 = cos(zd2), Cyd2 = cos(yd2);
    const double a[4] = {-Szd2 * Syd2, Czd2 * Syd2, Szd2 * Cyd2, Czd2 * Cyd2};
    // _equatorial2transform (:274-297) with ra = radians(hdg), dec = roll = radians(0); T = its transpose's transpose
    const double ra = hdg * (pi / 180.0), dec = 0.0 * (pi / 180.0), roll = 0.0 * (pi / 180.0);
    const double ca = cos(ra), sa = sin(ra), cd = cos(dec), sd = sin(dec), cr = cos(roll), sr = sin(roll);
    const double T00 = ca * cd, T01 = sa * cd, T02 = sd;
    const double T10 = -ca * sd * sr - sa * cr, T11 = -sa * sd * sr + ca * cr, T12 = cd * sr;
    const double T20 = -ca * sd * cr + sa * sr, T21 = -sa * sd * cr - ca * sr, T22 = cd * cr;
    // _transform2quat (:299-335): the first index of the largest den
    const double den[4] = {1.0 + T00 - T11 - T22, 1.0 - T00 + T11 - T22, 1.0 - T00 - T11 + T22, 1.0 + T00 + T11 + T22};
    int m = 0;
    for (int i = 1; i < 4; i++)
        if (den[i] > den[m]) m = i;
    double b[4] = {0.0, 0.0, 0.0, 0.0};
    b[m] = 0.5 * sqrt(den[m]);
    const double denom = 4.0 * b[m];
    if (m == 0) { b[1] = (T10 + T01) / denom; b[2] = (T20 + T02) / denom; b[3] = -(T21 - T12) / denom; }
    if (m == 1) { b[0] = (T10 + T01) / denom; b[2] = (T21 + T12) / denom; b[3] = -(T02 - T20) / denom; }
    if (m == 2) { b[0] = (T20 + T02) / denom; b[1] = (T21 + T12) / denom; b[3] = -(T10 - T01) / denom; }
    if (m == 3) { b[0] = -(T21 - T12) / denom; b[1] = -(T02 - T20) / denom; b[2] = -(T10 - T01) / denom; }
    // the product (:393-415), then _set_q's sign rule: q if q[3] > 0 else -q
    double q[4] = {a[3] * b[0] - a[2] * b[1] + a[1] * b[2] + a[0] * b[3],
                   a[2] * b[0] + a[3] * b[1] - a[0] * b[2] + a[1] * b[3],
                   -a[1] * b[0] + a[0] * b[1] + a[3] * b[2] + a[2] * b[3],
                   -a[0] * b[0] - a[1] * b[1] - a[2] * b[2] + a[3] * b[3]};
    if (!(q[3] > 0))
        for (int i = 0; i < 4; i++) q[i] = -q[i];
    // _get_angle_axis (:337-354), the norm summed in index order
    const double norm = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    if (norm < 1e-12) return 0;
    const double rnorm = 1.0 / norm;
    const double c = rnorm * q[3];
    double angle = acos(c > 1 ? 1.0 : c < -1 ? -1.0 : c);
    const double sangle = sin(angle);
    if (sangle < 1e-12) return 0;
    angle *= 2;
    for (int i = 0; i < 3; i++) o[i] = (float)(angle * ((rnorm / sangle) * q[i]));
    return 1;
}

AMB_HD void amb_fg_be32(char* p, uint32_t v)
{
    for (int i = 0; i < 4; i++) p[i] = (char)(v >> (24 - 8 * i));
}

AMB_HD void amb_fg_be64(char* p, uint64_t v)
{
    for (int i = 0; i < 8; i++) p[i] = (char)(v >> (56 - 8 * i));
}

AMB_HD void amb_fg_f32(char* p, float v) { uint32_t u; memcpy(&u, &v, 4); amb_fg_be32(p, u); }
AMB_HD void amb_fg_f64(char* p, double v) { uint64_t u; memcpy(&u, &v, 8); amb_fg_be64(p, u); }

// Rule 5: the packet of a position at lat, lon, alt (feet) and time t for an aircraft with callsign ident (8
// characters) and model m, heading hdg, vel_ms = (float)(velocity * 0.514444444) and turn = (float)(turn rate *
// (pi / 180.)), into out (AMB_FG_PACKET bytes), or nothing when the orientation does not exist. Returns the bytes written.
AMB_HD unsigned amb_fg_packet(const char* ident, int m, double lat, double lon, double alt, double t, double hdg,
                              float vel_ms, float turn, char* out)
{
    float o[3];
    if (!amb_fg_orientation(lat, lon, hdg, o)) return 0u;
    double s[3];
    amb_llh2ecef(lat, lon, alt * 0.3048, s, nullptr);
    memset(out, 0, AMB_FG_PACKET);
    out[0] = 'F'; out[1] = 'G'; out[2] = 'F'; out[3] = 'S';
    amb_fg_be32(out + 4, 0x00010001u);                  // proto
    amb_fg_be32(out + 8, 7u);                           // msgid: a position
    amb_fg_be32(out + 12, AMB_FG_PACKET);               // msglen; reply address and port stay 0
    for (int i = 0; i < 8; i++) out[24 + i] = ident[i];
    const char* path = amb_fg_model_path(m);
    for (int i = 0; path[i]; i++) out[32 + i] = path[i];   // NUL-padded to 96 bytes
    amb_fg_f64(out + 128, t);                           // time; lag stays 0.0
    for (int i = 0; i < 3; i++) amb_fg_f64(out + 144 + 8 * i, s[i]);
    for (int i = 0; i < 3; i++) amb_fg_f32(out + 168 + 4 * i, o[i]);
    amb_fg_f32(out + 180, vel_ms);                      // linear velocity (vel_ms, 0, 0)
    amb_fg_f32(out + 200, turn);                        // angular velocity (0, 0, turn); the rest stays 0
    return AMB_FG_PACKET;
}
