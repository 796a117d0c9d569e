// Multilateration (SURVEY.md 8 row f12, include/airmodes_b200.h amb_mlat, DESIGN.md 8 "Multilateration"): the frames of
// K synchronized receivers grouped by transmission, and each group of three or more solved for the aircraft position.
// Launch-free like the decoder's stage headers, so that tests/simt runs the same kernels and sequence under the host
// emulator; compiled into amb_decode.cu with -fmad=false, so that the solve is the CPU checker's IEEE arithmetic.
//
// One call, in stream order (N = carried + new eligible frames, npad = next power of two >= N):
//   amb_mlat_count    per 128 raw frames (each station's frames padded to whole blocks): how many are eligible
//   amb_sbs1_scan     their offsets                                  (then E = the new eligible count goes to the host)
//   amb_mlat_items    every eligible frame as an AmbMlatItem after the carried ones, station by station in stream order
//   amb_mlat_rank     each item's place in time order (t, station, list): a merge rank over the carried list and the K
//                     station lists, each of which is in time order; key = payload hash << 32 | rank
//   amb_order_*       the bitonic network of the device-side drain (amb_order_kernels.cuh) on (key, item)
//   amb_mlat_link     per sorted item: the next item of the same payload in time order, and whether a run starts here
//   amb_mlat_runs     per run start: walk the run, carry it, reject it (counted) or select it as a group
//   amb_mlat_select_count, amb_sbs1_scan x 2   groups and carried items counted in time order
//                     (then the group count, the new carry count and the counters go to the host: overflow check)
//   amb_mlat_select   the groups in the order of their reference time, and the new carry in time order
//   amb_mlat_solve    one thread per group: Gauss-Newton with Householder QR, the fix
#pragma once

#define AMB_MLAT_C (299792458.0 / 1.0003)       // mlat.py:95
#define AMB_MLAT_MAX_STEPS 25
#define AMB_MLAT_STOP 1e-3                       // |dx| in m
#define AMB_MLAT_RCOND 1e-9
#define AMB_MLAT_FT 0.3048
#define AMB_MLAT_BLOCK 128

int amb_launch_bitonic(unsigned long long* key, unsigned* val, unsigned npad, unsigned tile, cudaStream_t s);   // amb_order_kernels.cuh

// counters of one call (device, cleared per call)
enum { AMB_MC_CARRIED, AMB_MC_TOO_FEW, AMB_MC_DUPLICATE, AMB_MC_SPAN, AMB_MC_UNORDERED, AMB_MC_SOLVED, AMB_MC_NO_CONV,
       AMB_MC_DEGENERATE, AMB_MC_N };

struct AmbMlatItem {                 // one eligible frame (48 bytes)
    unsigned long long secs; double frac;   // t: frac less the station's offset
    uint8_t data[14]; uint8_t nbits, station;
    uint32_t addr; int32_t alt;
    uint8_t df, pad_[7];
};

struct AmbMlatStation {              // ECEF, and N, cos / sin of lat and lon (the start point overhead it)
    double s[3]; double n, cl, sl, co, so;
};

struct AmbMlatCall {                 // the new frames of one call, by value
    const amb_frame* f[AMB_MLAT_MAX_STATIONS];
    int count[AMB_MLAT_MAX_STATIONS];
    int base[AMB_MLAT_MAX_STATIONS + 1];    // station k's raw frames start at base[k] (a multiple of 128)
    double off[AMB_MLAT_MAX_STATIONS];
    int K;
};

// d(a, b) of the header: never the difference of two secs + frac sums
AMB_HD double amb_mlat_diff(unsigned long long sa, double fa, unsigned long long sb, double fb)
{
    return (double)(long long)(sa - sb) + (fa - fb);
}

AMB_HD double amb_mlat_dt(const AmbMlatItem& a, const AmbMlatItem& b) { return amb_mlat_diff(a.secs, a.frac, b.secs, b.frac); }

// Eligible: DF 0/4/16/20 with an AC13 altitude in feet (address: the AP overlay), DF17 TC 9..18 with a 12-bit ME
// altitude in feet (address: AA). Code 0 (no altitude) and metric altitudes are not eligible.
AMB_HD int amb_mlat_eligible(const amb_frame& f, uint32_t* addr, int32_t* feet, int* df_out)
{
    if (!f.passed) return 0;
    const AmbMsg g = amb_msg_from_frame(f);
    const int df = (int)amb_bits(g, 1, 5);
    int code, bit13;
    if (df == 0 || df == 4 || df == 16 || df == 20) {
        code = (int)amb_bits(g, 20, 13); bit13 = 1; *addr = f.crc;
    } else if (df == 17) {
        const int tc = (int)amb_bits(g, 33, 5);
        if (tc < 9 || tc > 18) return 0;
        code = (int)amb_bits(g, 41, 12); bit13 = 0; *addr = (uint32_t)amb_bits(g, 9, 24);
    } else {
        return 0;
    }
    if (code == 0 || amb_decode_alt(code, bit13, feet)) return 0;
    *df_out = df;
    return 1;
}

AMB_HD int amb_mlat_same_payload(const AmbMlatItem& a, const AmbMlatItem& b)
{
    if (a.nbits != b.nbits) return 0;
    for (int k = 0; k < 14; k++) if (a.data[k] != b.data[k]) return 0;
    return 1;
}

AMB_HD uint32_t amb_mlat_hash(const AmbMlatItem& a)       // FNV-1a over nbits and the payload
{
    uint32_t h = 2166136261u;
    h = (h ^ a.nbits) * 16777619u;
    for (int k = 0; k < a.nbits / 8; k++) h = (h ^ a.data[k]) * 16777619u;
    return h;
}

AMB_HD double amb_mlat_norm3(double a, double b, double c) { return sqrt(a * a + b * b + c * c); }

// ecef2llh (mlat.py:58-75), Bowring's one-step form; lat, lon in radians
AMB_HD void amb_mlat_ecef2llh(const double* x, double* lat, double* lon, double* h)
{
    const double a = AMB_MLAT_WGS_A, b = AMB_MLAT_WGS_B;
    const double ep = sqrt((a * a - b * b) / (b * b));
    const double p = sqrt(x[0] * x[0] + x[1] * x[1]);
    const double th = atan2(a * x[2], b * p);
    *lon = atan2(x[1], x[0]);
    const double st = sin(th), ct = cos(th);
    *lat = atan2(x[2] + ep * ep * b * (st * st * st), p - AMB_MLAT_WGS_E2 * a * (ct * ct * ct));
    const double sl = sin(*lat);
    const double n = a / sqrt(1 - AMB_MLAT_WGS_E2 * (sl * sl));
    *h = p / cos(*lat) - n;
}

// The n x 3 rows at x: f (residuals) and J; the TDOA rows in ascending station order, the altitude row last
AMB_HD int amb_mlat_rows(const double* x, const AmbMlatStation* sta, uint32_t mask, int r, const double* dt, double h,
                         double (*J)[3], double* f)
{
    int n = 0;
    const double* sr = sta[r].s;
    const double er0 = x[0] - sr[0], er1 = x[1] - sr[1], er2 = x[2] - sr[2];
    const double dr = amb_mlat_norm3(er0, er1, er2);
    for (int k = 0; k < AMB_MLAT_MAX_STATIONS; k++) {
        if (!((mask >> k) & 1u) || k == r) continue;
        const double* si = sta[k].s;
        const double e0 = x[0] - si[0], e1 = x[1] - si[1], e2 = x[2] - si[2];
        const double di = amb_mlat_norm3(e0, e1, e2);
        f[n] = (di - dr) - AMB_MLAT_C * dt[k];
        J[n][0] = e0 / di - er0 / dr; J[n][1] = e1 / di - er1 / dr; J[n][2] = e2 / di - er2 / dr;
        n++;
    }
    double lat, lon, hh;
    amb_mlat_ecef2llh(x, &lat, &lon, &hh);
    const double sl = sin(lat), cl = cos(lat);
    const double nn = AMB_MLAT_WGS_A / sqrt(1 - AMB_MLAT_WGS_E2 * (sl * sl));
    const double q = (nn + h) * cl, z = (nn * (1 - AMB_MLAT_WGS_E2) + h) * sl;
    const double rho = sqrt(q * q + z * z);                  // |llh2ecef(lat, lon, h)|, which lon does not change
    const double nx = amb_mlat_norm3(x[0], x[1], x[2]);
    f[n] = nx - rho;
    J[n][0] = x[0] / nx; J[n][1] = x[1] / nx; J[n][2] = x[2] / nx;
    return n + 1;
}

// Householder QR of A (n x 3) applied to b, in place: R in the upper triangle of A (diagonal = alpha), Q^T b in b.
// Returns 1 when R is degenerate (some |R_jj| < 1e-9 max |R_jj|, or no positive maximum).
AMB_HD int amb_mlat_qr(double (*A)[3], double* b, int n)
{
    for (int j = 0; j < 3; j++) {
        double s = 0.0;
        for (int i = j; i < n; i++) s += A[i][j] * A[i][j];
        const double nrm = sqrt(s);
        const double alpha = A[j][j] > 0.0 ? -nrm : nrm;
        const double vj = A[j][j] - alpha;
        double vtv = vj * vj;
        for (int i = j + 1; i < n; i++) vtv += A[i][j] * A[i][j];
        if (vtv > 0.0) {
            for (int k = j + 1; k < 4; k++) {                // columns j+1..2, then b (k = 3)
                double dot = vj * (k < 3 ? A[j][k] : b[j]);
                for (int i = j + 1; i < n; i++) dot += A[i][j] * (k < 3 ? A[i][k] : b[i]);
                const double tau = (dot + dot) / vtv;
                if (k < 3) {
                    A[j][k] -= tau * vj;
                    for (int i = j + 1; i < n; i++) A[i][k] -= tau * A[i][j];
                } else {
                    b[j] -= tau * vj;
                    for (int i = j + 1; i < n; i++) b[i] -= tau * A[i][j];
                }
            }
        }
        A[j][j] = alpha;
    }
    const double r0 = fabs(A[0][0]), r1 = fabs(A[1][1]), r2 = fabs(A[2][2]);
    double mx = r0 > r1 ? r0 : r1;
    mx = mx > r2 ? mx : r2;
    if (!(mx > 0.0)) return 1;
    const double lim = AMB_MLAT_RCOND * mx;
    return !(r0 >= lim) || !(r1 >= lim) || !(r2 >= lim);
}

// One group: mask of stations, r the reference station, dt[k] = d(t_k, t_r), h the altitude in m. Writes x, the
// status, the steps, rms and dop.
AMB_HD int amb_mlat_solve_group(const AmbMlatStation* sta, uint32_t mask, int r, const double* dt, double h, double* x,
                                int* steps, double* rms, double* dop)
{
    double J[AMB_MLAT_MAX_STATIONS][3], f[AMB_MLAT_MAX_STATIONS];
    const AmbMlatStation& o = sta[r];
    x[0] = (o.n + h) * o.cl * o.co; x[1] = (o.n + h) * o.cl * o.so; x[2] = (o.n * (1 - AMB_MLAT_WGS_E2) + h) * o.sl;
    int status = AMB_MLAT_NO_CONVERGENCE;
    *steps = AMB_MLAT_MAX_STEPS;
    for (int it = 1; it <= AMB_MLAT_MAX_STEPS; it++) {
        const int n = amb_mlat_rows(x, sta, mask, r, dt, h, J, f);
        for (int i = 0; i < n; i++) f[i] = -f[i];
        if (amb_mlat_qr(J, f, n)) { status = AMB_MLAT_DEGENERATE; *steps = it - 1; break; }
        const double d2 = f[2] / J[2][2];
        const double d1 = (f[1] - J[1][2] * d2) / J[1][1];
        const double d0 = (f[0] - J[0][1] * d1 - J[0][2] * d2) / J[0][0];
        x[0] += d0; x[1] += d1; x[2] += d2;
        if (amb_mlat_norm3(d0, d1, d2) <= AMB_MLAT_STOP) { status = AMB_MLAT_SOLVED; *steps = it; break; }
    }
    // rms and dop at the last x
    const int n = amb_mlat_rows(x, sta, mask, r, dt, h, J, f);
    double ss = 0.0;
    for (int i = 0; i < n; i++) ss += f[i] * f[i];
    *rms = sqrt(ss / n);
    if (amb_mlat_qr(J, f, n)) {
        *dop = NAN;
    } else {                                                 // trace((J^T J)^-1) = |R^-1|_F^2
        const double u00 = 1.0 / J[0][0], u11 = 1.0 / J[1][1], u22 = 1.0 / J[2][2];
        const double u01 = -(J[0][1] * u11) / J[0][0];
        const double u12 = -(J[1][2] * u22) / J[1][1];
        const double u02 = -(J[0][1] * u12 + J[0][2] * u22) / J[0][0];
        *dop = sqrt(u00 * u00 + u01 * u01 + u02 * u02 + u11 * u11 + u12 * u12 + u22 * u22);
    }
    return status;
}

// ---- kernels -------------------------------------------------------------------------------------------------------
// the station of raw slot g (base[] ascending, each station's slots a whole number of blocks)
__device__ __forceinline__ int amb_mlat_station_of(const AmbMlatCall& c, int g)
{
    int k = 0;
    while (k + 1 < c.K && c.base[k + 1] <= g) k++;
    return k;
}

// exclusive rank of this thread's pred among the block's set preds, and their total (blockDim.x = 128)
__device__ __forceinline__ unsigned amb_mlat_block_rank(int pred, unsigned* s_w, unsigned* total)
{
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) s_w[warp] = __popc(bal);
    __syncthreads();
    unsigned before = 0, all = 0;
    for (unsigned w = 0; w < AMB_MLAT_BLOCK / 32; w++) { if (w < warp) before += s_w[w]; all += s_w[w]; }
    *total = all;
    return before + __popc(bal & ((1u << lane) - 1u));
}

__device__ __forceinline__ int amb_mlat_raw(const AmbMlatCall& c, int g, AmbMlatItem* it)
{
    const int k = amb_mlat_station_of(c, g), i = g - c.base[k];
    if (i >= c.count[k]) return 0;
    const amb_frame& f = c.f[k][i];
    uint32_t addr = 0; int32_t feet = 0; int df = 0;
    if (!amb_mlat_eligible(f, &addr, &feet, &df)) return 0;
    if (it) {
        it->secs = f.secs; it->frac = f.frac - c.off[k];
        const int nb = f.nbits / 8;
        for (int b = 0; b < 14; b++) it->data[b] = b < nb ? f.data[b] : 0;
        it->nbits = f.nbits; it->station = (uint8_t)k; it->addr = addr; it->alt = feet; it->df = (uint8_t)df;
        for (int b = 0; b < 7; b++) it->pad_[b] = 0;
    }
    return 1;
}

__global__ void __launch_bounds__(AMB_MLAT_BLOCK) amb_mlat_count(AmbMlatCall c, uint32_t* __restrict__ bsum)
{
    __shared__ unsigned s_w[AMB_MLAT_BLOCK / 32];
    const int g = blockIdx.x * AMB_MLAT_BLOCK + threadIdx.x;
    unsigned total;
    amb_mlat_block_rank(amb_mlat_raw(c, g, nullptr), s_w, &total);
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(AMB_MLAT_BLOCK) amb_mlat_items(AmbMlatCall c, const unsigned long long* __restrict__ boff,
                                                                 int C, AmbMlatItem* __restrict__ items)
{
    __shared__ unsigned s_w[AMB_MLAT_BLOCK / 32];
    const int g = blockIdx.x * AMB_MLAT_BLOCK + threadIdx.x;
    AmbMlatItem it;
    const int el = amb_mlat_raw(c, g, &it);
    unsigned total;
    const unsigned at = amb_mlat_block_rank(el, s_w, &total);
    if (el) items[C + boff[blockIdx.x] + at] = it;
}

// items i < C: the carried list, in time order; items of station k's list: [lo_k, hi_k) from the raw offsets
__device__ __forceinline__ void amb_mlat_list(const AmbMlatCall& c, const unsigned long long* boff, int C, int L, int* lo,
                                              int* hi)
{
    if (L == 0) { *lo = 0; *hi = C; return; }
    *lo = C + (int)boff[c.base[L - 1] / AMB_MLAT_BLOCK];
    *hi = C + (int)boff[c.base[L] / AMB_MLAT_BLOCK];
}

// (t_j, s_j, Lj) < (t_x, s_x, Lx)
__device__ __forceinline__ bool amb_mlat_before(const AmbMlatItem& j, int Lj, const AmbMlatItem& x, int Lx)
{
    const double d = amb_mlat_dt(j, x);
    if (d < 0.0) return true;
    if (d > 0.0) return false;
    if (j.station != x.station) return j.station < x.station;
    return Lj < Lx;
}

__global__ void __launch_bounds__(256) amb_mlat_rank(AmbMlatCall c, const unsigned long long* __restrict__ boff, int C, int N,
                                                     int npad, const AmbMlatItem* __restrict__ items,
                                                     unsigned long long* __restrict__ key, unsigned* __restrict__ val,
                                                     unsigned* __restrict__ rank, unsigned long long* __restrict__ ctr)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= npad) return;
    val[i] = (unsigned)i;
    if (i >= N) { key[i] = ~0ull; return; }
    const AmbMlatItem x = items[i];
    const int L = i < C ? 0 : x.station + 1;
    int lo, hi, a0;
    amb_mlat_list(c, boff, C, L, &lo, &hi);
    if (L > 0 && i + 1 < hi && amb_mlat_dt(items[i + 1], x) < 0.0) ctr[AMB_MC_UNORDERED] = 1;
    unsigned r = (unsigned)(i - lo);
    for (int L2 = 0; L2 <= c.K; L2++) {
        if (L2 == L) continue;
        int a, b;
        amb_mlat_list(c, boff, C, L2, &a, &b);
        a0 = a;
        while (a < b) {                                     // the first of the list not before x
            const int m = a + (b - a) / 2;
            if (amb_mlat_before(items[m], L2, x, L)) a = m + 1; else b = m;
        }
        r += (unsigned)(a - a0);
    }
    rank[i] = r;
    key[i] = ((unsigned long long)amb_mlat_hash(x) << 32) | r;
}

__global__ void __launch_bounds__(256) amb_mlat_link(const unsigned long long* __restrict__ key, const unsigned* __restrict__ val,
                                                     int N, const AmbMlatItem* __restrict__ items, double W,
                                                     int* __restrict__ next, uint8_t* __restrict__ start)
{
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p >= N) return;
    const uint32_t h = (uint32_t)(key[p] >> 32);
    const AmbMlatItem& x = items[val[p]];
    int prev = -1, nx = -1;
    for (int q = p - 1; q >= 0 && (uint32_t)(key[q] >> 32) == h; q--)
        if (amb_mlat_same_payload(items[val[q]], x)) { prev = q; break; }
    for (int q = p + 1; q < N && (uint32_t)(key[q] >> 32) == h; q++)
        if (amb_mlat_same_payload(items[val[q]], x)) { nx = q; break; }
    next[p] = nx;
    start[p] = prev < 0 || amb_mlat_dt(x, items[val[prev]]) > W;
}

__global__ void __launch_bounds__(256) amb_mlat_runs(const unsigned* __restrict__ val, int N, const AmbMlatItem* __restrict__ items,
                                                     const unsigned* __restrict__ rank, const int* __restrict__ next,
                                                     const uint8_t* __restrict__ start, double W,
                                                     unsigned long long end_secs, double end_frac, int flush,
                                                     unsigned* __restrict__ gsel, unsigned* __restrict__ csel,
                                                     int* __restrict__ runlen, unsigned long long* __restrict__ ctr)
{
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p >= N || !start[p]) return;
    const AmbMlatItem& first = items[val[p]];
    uint32_t mask = 1u << first.station;
    int dup = 0, m = 1, cur = p;
    for (int q = next[p]; q >= 0 && amb_mlat_dt(items[val[q]], items[val[cur]]) <= W; q = next[q]) {
        const uint32_t bit = 1u << items[val[q]].station;
        dup |= (mask & bit) != 0;
        mask |= bit; m++; cur = q;
    }
    const AmbMlatItem& last = items[val[cur]];
    if (!flush && !(amb_mlat_diff(end_secs, end_frac, last.secs, last.frac) >= W)) {
        for (int q = p, j = 0; j < m; j++, q = next[q]) csel[rank[val[q]]] = val[q] + 1;
        atomicAdd(&ctr[AMB_MC_CARRIED], (unsigned long long)m);
        return;
    }
    if (dup) atomicAdd(&ctr[AMB_MC_DUPLICATE], 1ull);
    else if (m < AMB_MLAT_MIN_STATIONS) atomicAdd(&ctr[AMB_MC_TOO_FEW], 1ull);
    else if (amb_mlat_dt(last, first) > W) atomicAdd(&ctr[AMB_MC_SPAN], 1ull);
    else { gsel[rank[val[p]]] = (unsigned)p + 1; runlen[p] = m; }
}

__global__ void __launch_bounds__(AMB_MLAT_BLOCK) amb_mlat_select_count(const unsigned* __restrict__ gsel,
                                                                        const unsigned* __restrict__ csel, int N,
                                                                        uint32_t* __restrict__ gsum, uint32_t* __restrict__ csum)
{
    __shared__ unsigned s_w[AMB_MLAT_BLOCK / 32];
    const int i = blockIdx.x * AMB_MLAT_BLOCK + threadIdx.x;
    unsigned tg, tc;
    amb_mlat_block_rank(i < N && gsel[i] != 0, s_w, &tg);
    __syncthreads();
    amb_mlat_block_rank(i < N && csel[i] != 0, s_w, &tc);
    if (threadIdx.x == 0) { gsum[blockIdx.x] = tg; csum[blockIdx.x] = tc; }
}

__global__ void __launch_bounds__(AMB_MLAT_BLOCK) amb_mlat_select(const unsigned* __restrict__ gsel, const unsigned* __restrict__ csel,
                                                                  int N, const unsigned long long* __restrict__ goff,
                                                                  const unsigned long long* __restrict__ coff,
                                                                  const AmbMlatItem* __restrict__ items,
                                                                  unsigned* __restrict__ groups, AmbMlatItem* __restrict__ carry)
{
    __shared__ unsigned s_w[AMB_MLAT_BLOCK / 32];
    const int i = blockIdx.x * AMB_MLAT_BLOCK + threadIdx.x;
    const unsigned g = i < N ? gsel[i] : 0u, cs = i < N ? csel[i] : 0u;
    unsigned total;
    const unsigned ag = amb_mlat_block_rank(g != 0, s_w, &total);
    __syncthreads();
    const unsigned ac = amb_mlat_block_rank(cs != 0, s_w, &total);
    if (g) groups[goff[blockIdx.x] + ag] = g - 1;
    if (cs) carry[coff[blockIdx.x] + ac] = items[cs - 1];
}

__global__ void __launch_bounds__(64) amb_mlat_solve(const unsigned* __restrict__ groups, int G, const unsigned* __restrict__ val,
                                                     const AmbMlatItem* __restrict__ items, const int* __restrict__ next,
                                                     const int* __restrict__ runlen, const AmbMlatStation* __restrict__ sta,
                                                     amb_mlat_fix* __restrict__ out, unsigned long long* __restrict__ ctr)
{
    const int g = blockIdx.x * 64 + threadIdx.x;
    if (g >= G) return;
    const int p = (int)groups[g], m = runlen[p];
    const AmbMlatItem& ref = items[val[p]];
    const int r = ref.station;
    double dt[AMB_MLAT_MAX_STATIONS];
    uint32_t mask = 0;
    for (int q = p, j = 0; j < m; j++, q = next[q]) {
        const AmbMlatItem& it = items[val[q]];
        dt[it.station] = amb_mlat_dt(it, ref);
        mask |= 1u << it.station;
    }
    const double h = (double)ref.alt * AMB_MLAT_FT;
    double x[3], rms, dop;
    int steps;
    const int status = amb_mlat_solve_group(sta, mask, r, dt, h, x, &steps, &rms, &dop);
    amb_mlat_fix fx;
    for (int b = 0; b < 14; b++) fx.data[b] = ref.data[b];
    fx.nbits = ref.nbits; fx.df = ref.df; fx.addr = ref.addr;
    fx.status = (uint8_t)status; fx.n = (uint8_t)m; fx.steps = (uint8_t)steps; fx.ref = (uint8_t)r;
    fx.stations = mask; fx.altitude = ref.alt;
    const double* sr = sta[r].s;
    unsigned long long secs = ref.secs;
    double frac = ref.frac - amb_mlat_norm3(x[0] - sr[0], x[1] - sr[1], x[2] - sr[2]) / AMB_MLAT_C;
    if (frac - frac == 0.0) {                               // finite
        while (frac < 0.0) { frac += 1.0; secs -= 1; }
        while (frac >= 1.0) { frac -= 1.0; secs += 1; }
    }
    fx.secs = secs; fx.frac = frac;
    double lat, lon, hh;
    amb_mlat_ecef2llh(x, &lat, &lon, &hh);
    fx.lat = lat * (180.0 / M_PI); fx.lon = lon * (180.0 / M_PI); fx.height = hh;
    fx.x = x[0]; fx.y = x[1]; fx.z = x[2];
    fx.rms = rms; fx.dop = dop;
    out[g] = fx;
    atomicAdd(&ctr[status == AMB_MLAT_SOLVED ? AMB_MC_SOLVED : status == AMB_MLAT_NO_CONVERGENCE ? AMB_MC_NO_CONV
                                                                                                 : AMB_MC_DEGENERATE], 1ull);
}

// ---- the object's device memory --------------------------------------------------------------------------------------
struct AmbMlatState {
    int K = 0;
    double W = 0.0;                                   // s
    double off[AMB_MLAT_MAX_STATIONS] = {};
    AmbMlatStation* sta = nullptr;                    // device, K
    amb_frame* raw = nullptr; size_t raw_cap = 0;     // host frames on their way in
    AmbMlatItem* carry = nullptr; int C = 0; int carry_cap = 0;
    // per call
    uint32_t* bsum[2] = {nullptr, nullptr}; unsigned long long* boff[2] = {nullptr, nullptr}; int nb_cap = 0;
    AmbMlatItem* items = nullptr; unsigned* rank = nullptr; int* next = nullptr; uint8_t* start = nullptr;
    int* runlen = nullptr; unsigned* gsel = nullptr; unsigned* csel = nullptr; unsigned* groups = nullptr;
    int item_cap = 0;
    unsigned long long* key = nullptr; unsigned* val = nullptr; int npad_cap = 0;
    unsigned long long* ctr = nullptr;                // AMB_MC_N
    amb_mlat_fix* fix = nullptr; int fix_cap = 0;     // fixes on their way out
};

static void amb_mlat_free_items(AmbMlatState* s)
{
    void* p[] = {s->items, s->rank, s->next, s->start, s->runlen, s->gsel, s->csel, s->groups};
    for (void* q : p) if (q) cudaFree(q);
    s->items = nullptr; s->rank = nullptr; s->next = nullptr; s->start = nullptr; s->runlen = nullptr;
    s->gsel = nullptr; s->csel = nullptr; s->groups = nullptr; s->item_cap = 0;
}

static void amb_mlat_free(AmbMlatState* s)
{
    amb_mlat_free_items(s);
    void* p[] = {s->sta, s->raw, s->carry, s->bsum[0], s->bsum[1], s->boff[0], s->boff[1], s->key, s->val, s->ctr, s->fix};
    for (void* q : p) if (q) cudaFree(q);
    *s = AmbMlatState();
}

#define AMB_MLAT_GROW(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { *err = e_; return -1; } } while (0)

// capacity for P raw slots (nb = P / 128 blocks)
static int amb_mlat_prepare_raw(AmbMlatState* s, int nb, cudaError_t* err)
{
    if (s->nb_cap < nb + 1) {
        for (int k = 0; k < 2; k++) {
            if (s->bsum[k]) cudaFree(s->bsum[k]);
            if (s->boff[k]) cudaFree(s->boff[k]);
            s->bsum[k] = nullptr; s->boff[k] = nullptr;
        }
        s->nb_cap = 0;
        const int cap = nb + 1 + (nb + 1) / 2;
        for (int k = 0; k < 2; k++) {
            AMB_MLAT_GROW(cudaMalloc(&s->bsum[k], (size_t)cap * sizeof(uint32_t)));
            AMB_MLAT_GROW(cudaMalloc(&s->boff[k], (size_t)(cap + 1) * sizeof(unsigned long long)));
        }
        s->nb_cap = cap;
    }
    if (!s->ctr) AMB_MLAT_GROW(cudaMalloc(&s->ctr, AMB_MC_N * sizeof(unsigned long long)));
    return 0;
}

// capacity for N items (npad = next power of two); the carry keeps its C items when it grows
static int amb_mlat_prepare_items(AmbMlatState* s, int N, int npad, cudaError_t* err)
{
    if (s->item_cap < N) {
        amb_mlat_free_items(s);
        const int cap = N + N / 2;
        AMB_MLAT_GROW(cudaMalloc(&s->items, (size_t)cap * sizeof(AmbMlatItem)));
        AMB_MLAT_GROW(cudaMalloc(&s->rank, (size_t)cap * sizeof(unsigned)));
        AMB_MLAT_GROW(cudaMalloc(&s->next, (size_t)cap * sizeof(int)));
        AMB_MLAT_GROW(cudaMalloc(&s->start, (size_t)cap));
        AMB_MLAT_GROW(cudaMalloc(&s->runlen, (size_t)cap * sizeof(int)));
        AMB_MLAT_GROW(cudaMalloc(&s->gsel, (size_t)cap * sizeof(unsigned)));
        AMB_MLAT_GROW(cudaMalloc(&s->csel, (size_t)cap * sizeof(unsigned)));
        AMB_MLAT_GROW(cudaMalloc(&s->groups, (size_t)cap * sizeof(unsigned)));
        s->item_cap = cap;
    }
    if (s->carry_cap < N) {
        AmbMlatItem* c = nullptr;
        const int cap = N + N / 2;
        AMB_MLAT_GROW(cudaMalloc(&c, (size_t)cap * sizeof(AmbMlatItem)));
        if (s->C) AMB_MLAT_GROW(cudaMemcpy(c, s->carry, (size_t)s->C * sizeof(AmbMlatItem), cudaMemcpyDeviceToDevice));
        if (s->carry) cudaFree(s->carry);
        s->carry = c; s->carry_cap = cap;
    }
    if (s->npad_cap < npad) {
        if (s->key) cudaFree(s->key);
        if (s->val) cudaFree(s->val);
        s->key = nullptr; s->val = nullptr; s->npad_cap = 0;
        AMB_MLAT_GROW(cudaMalloc(&s->key, (size_t)npad * sizeof(unsigned long long)));
        AMB_MLAT_GROW(cudaMalloc(&s->val, (size_t)npad * sizeof(unsigned)));
        s->npad_cap = npad;
    }
    return 0;
}

// The first half of a call: count the eligible frames (E lands in boff[0][nb]). Returns kernels launched.
static int amb_mlat_launch_count(const AmbMlatCall& c, int nb, AmbMlatState* s, cudaStream_t st, cudaError_t* err)
{
    AMB_LAUNCH((amb_mlat_count), nb, AMB_MLAT_BLOCK, 0, st, c, s->bsum[0]);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, st, s->bsum[0], nb, s->boff[0]);
    *err = cudaGetLastError();
    return 2;
}

// The second half, up to the overflow check: items, order, runs, selection counts (groups at boff[0][nbn], the new
// carry at boff[1][nbn], nbn = ceil(N / 128)). Returns kernels launched.
static int amb_mlat_launch_group(const AmbMlatCall& c, int nb, int N, int npad, unsigned order_tile, unsigned long long end_secs,
                                 double end_frac, int flush, AmbMlatState* s, cudaStream_t st, cudaError_t* err)
{
    int launches = 0;
    const int C = s->C, nbn = (N + AMB_MLAT_BLOCK - 1) / AMB_MLAT_BLOCK;
    AMB_MLAT_GROW(cudaMemsetAsync(s->ctr, 0, AMB_MC_N * sizeof(unsigned long long), st));
    AMB_MLAT_GROW(cudaMemsetAsync(s->gsel, 0, (size_t)N * sizeof(unsigned), st));
    AMB_MLAT_GROW(cudaMemsetAsync(s->csel, 0, (size_t)N * sizeof(unsigned), st));
    if (C) AMB_MLAT_GROW(cudaMemcpyAsync(s->items, s->carry, (size_t)C * sizeof(AmbMlatItem), cudaMemcpyDeviceToDevice, st));
    if (nb) { AMB_LAUNCH((amb_mlat_items), nb, AMB_MLAT_BLOCK, 0, st, c, s->boff[0], C, s->items); launches++; }
    AMB_LAUNCH((amb_mlat_rank), (npad + 255) / 256, 256, 0, st, c, s->boff[0], C, N, npad, s->items, s->key, s->val, s->rank,
               s->ctr); launches++;
    launches += amb_launch_bitonic(s->key, s->val, (unsigned)npad, order_tile, st);
    AMB_LAUNCH((amb_mlat_link), (N + 255) / 256, 256, 0, st, s->key, s->val, N, s->items, s->W, s->next, s->start); launches++;
    AMB_LAUNCH((amb_mlat_runs), (N + 255) / 256, 256, 0, st, s->val, N, s->items, s->rank, s->next, s->start, s->W, end_secs,
               end_frac, flush, s->gsel, s->csel, s->runlen, s->ctr); launches++;
    AMB_LAUNCH((amb_mlat_select_count), nbn, AMB_MLAT_BLOCK, 0, st, s->gsel, s->csel, N, s->bsum[0], s->bsum[1]); launches++;
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, st, s->bsum[0], nbn, s->boff[0]); launches++;
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, st, s->bsum[1], nbn, s->boff[1]); launches++;
    *err = cudaGetLastError();
    return launches;
}

// The last part: the selection written (groups, the new carry into s->carry) and G groups solved into out.
static int amb_mlat_launch_solve(int N, int G, amb_mlat_fix* out, AmbMlatState* s, cudaStream_t st, cudaError_t* err)
{
    int launches = 0;
    const int nbn = (N + AMB_MLAT_BLOCK - 1) / AMB_MLAT_BLOCK;
    AMB_LAUNCH((amb_mlat_select), nbn, AMB_MLAT_BLOCK, 0, st, s->gsel, s->csel, N, s->boff[0], s->boff[1], s->items, s->groups,
               s->carry); launches++;
    if (G) {
        AMB_LAUNCH((amb_mlat_solve), (G + 63) / 64, 64, 0, st, s->groups, G, s->val, s->items, s->next, s->runlen, s->sta, out,
                   s->ctr); launches++;
    }
    *err = cudaGetLastError();
    return launches;
}
