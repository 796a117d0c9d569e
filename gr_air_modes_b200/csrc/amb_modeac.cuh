// Mode A/C replies (option "modeac"): the rules are in include/airmodes_b200.h and DESIGN.md §3 "Mode A/C replies".
// Included by amb_kernels.cu. Two launches per call on stream B, after the scan of the same call:
//   amb_modeac_tile_kernel  one CTA per tile of AMB_MODEAC_TILE starts of [j_lo, j_hi): the canonical bb of the tile's
//                           span in shared memory, avg[i] from an fp64 prefix of bb (exact, so equal to the canonical
//                           ascending sum, when every addend's exponent lies within 17 of the others; else the literal
//                           ascending sum), rules 1-5 for the tile and the o(25.1) starts in front of it, rules 6-7 for
//                           the tile; the replies at tile * cap + rank (ascending), the count per tile
//   amb_modeac_emit_kernel  one CTA: the tiles' counts scanned in order, the replies appended to the queue, and the
//                           largest start passing rules 1-5 carried to the next call (rule 7 across calls)
// Stamping happens on poll or, for a device drain, in amb_modeac_stamp_kernel (amb_api.cu).
#pragma once
#include "amb_decode_core.h"

#define AMB_MODEAC_THREADS 256

// Decoded fields of a 13-bit code (rule 6 and the record): squawk, and the altitude when D1 = 0 and the C group is valid.
AMB_HD int32_t amb_modeac_altitude(int code)
{
    const int c = ((code >> 10) & 4) | ((code >> 9) & 2) | ((code >> 8) & 1);     // C1 C2 C4
    if ((code & 0x10) || c == 0 || c == 5 || c == 7) return AMB_NO_ALTITUDE;
    int32_t feet = AMB_NO_ALTITUDE;
    return amb_decode_alt(code, 1, &feet) ? AMB_NO_ALTITUDE : feet;
}

__device__ __forceinline__ float modeac_bb(const float* m2s, int m, int fl, float scale_p, int use_pmf)
{
    if (!use_pmf) return m2s[m];
    double acc = 0.0;
    for (int t = 0; t < fl; t++) acc += (double)m2s[m + t];
    return __fmul_rn((float)acc, scale_p);
}

__global__ void __launch_bounds__(AMB_MODEAC_THREADS) amb_modeac_tile_kernel(const AmbModeacArgs a)
{
    AMB_DYN_SMEM(double, mc_smem, 16);
    __shared__ unsigned s_pass[(AMB_MODEAC_TILE + 1024) / 32 + 2];   // rules 1-5 at e0 + bit (back <= 502 at 20 Msps)
    __shared__ unsigned s_reply[AMB_MODEAC_TILE / 32];                  // rules 1-5 on the tile
    __shared__ unsigned s_keep[AMB_MODEAC_TILE / 32];                   // ... and rule 7
    __shared__ unsigned s_emin[AMB_MODEAC_THREADS / 32], s_emax[AMB_MODEAC_THREADS / 32];
    __shared__ double s_part[AMB_MODEAC_THREADS / 32];
    __shared__ unsigned long long s_cnt[4];
    __shared__ unsigned s_last;                                         // 1 + the tile's last start passing 1-5 - e0
    const AmbParams& P = a.P;
    const AmbModeacGeom& G = a.G;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int L = P.L, fl = P.use_pmf ? P.spc_i : 1;
    const int j0 = a.j_lo + (int)blockIdx.x * AMB_MODEAC_TILE;
    const int j1 = min(j0 + AMB_MODEAC_TILE, a.j_hi);
    const int e0 = max(a.j_lo, j0 - G.back);           // rules 1-5 are evaluated on [e0, j1)
    const int b0 = e0 - L;                             // bb on [b0, b1): floor windows, in[i-1] .. in[i+spi+1]
    const int b1 = j1 + G.spi + 2;
    const int nb = b1 - b0, na = j1 - b0;             // prefix over bb[b0 .. j1)
    double* pre = mc_smem;                             // pre[k] = sum of bb[b0 .. b0+k-1], k = 0..na
    float* bbs = reinterpret_cast<float*>(pre + a.na_cap + 1);
    float* m2s = reinterpret_cast<float*>(pre);        // m2 on [b0 - fl + 1, b1), dead once bb is formed
    if (tid < 4) s_cnt[tid] = 0;
    if (tid == 0) s_last = 0u;
    for (int k = tid; k < (int)(sizeof s_pass / 4); k += AMB_MODEAC_THREADS) s_pass[k] = 0u;
    for (int k = tid; k < AMB_MODEAC_TILE / 32; k += AMB_MODEAC_THREADS) { s_reply[k] = 0u; s_keep[k] = 0u; }
    const int nm = nb + fl - 1, m0 = b0 - fl + 1;
    const float2* span = seg_span(a.S, m0, nm);        // block-uniform: the span inside one segment (the common case)
    if (span) {
        for (int i0 = 0; i0 < nm; i0 += 8 * AMB_MODEAC_THREADS) {                           // 8 loads in flight
            float2 v[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i = i0 + u * AMB_MODEAC_THREADS + tid;
                v[u] = i < nm ? span[i] : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i = i0 + u * AMB_MODEAC_THREADS + tid;
                if (i < nm) m2s[i] = canon_m2_of(v[u]);
            }
        }
    } else {
        for (int k = tid; k < nm; k += AMB_MODEAC_THREADS) m2s[k] = canon_m2(a.S, m0 + k);
    }
    __syncthreads();
    unsigned emax = 0u, emin = 255u;
    for (int k = tid; k < nb; k += AMB_MODEAC_THREADS) {
        const float v = modeac_bb(m2s, k, fl, P.scale_p, P.use_pmf);
        bbs[k] = v;
        const unsigned bits = __float_as_uint(v) & 0x7fffffffu;
        if (k < na && bits) { unsigned e = bits >> 23; e = e ? e : 1u; emax = max(emax, e); emin = min(emin, e); }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        emax = max(emax, __shfl_xor_sync(FULL, emax, d));
        emin = min(emin, __shfl_xor_sync(FULL, emin, d));
    }
    if (lane == 0) { s_emax[warp] = emax; s_emin[warp] = emin; }
    __syncthreads();
    emax = 0u; emin = 255u;
    for (int w = 0; w < AMB_MODEAC_THREADS / 32; w++) { emax = max(emax, s_emax[w]); emin = min(emin, s_emin[w]); }
    // <= 2^12 addends within 2^17 of each other: every partial sum is an integer multiple of the smallest ulp below
    // 2^(24 + 17 + 12) = 2^53, so it is exact in fp64 in any order, and so is a difference of two of them
    const bool exact = emax < 255u && emax <= emin + 17u && na <= 4096;
    if (exact) {                                       // thread t sums its run, a shuffle scan orders the runs
        const int per = (na + AMB_MODEAC_THREADS - 1) / AMB_MODEAC_THREADS;
        const int k0 = min(na, tid * per), k1 = min(na, k0 + per);
        double s = 0.0;
        for (int k = k0; k < k1; k++) s += (double)bbs[k];
        double inc = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const double v = __shfl_up_sync(FULL, inc, d); if (lane >= d) inc += v; }
        if (lane == 31) s_part[warp] = inc;
        __syncthreads();
        double base = inc - s;
        for (int w = 0; w < warp; w++) base += s_part[w];
        if (tid == 0) pre[0] = 0.0;
        for (int k = k0; k < k1; k++) { base += (double)bbs[k]; pre[k + 1] = base; }
    }
    __syncthreads();
    const float* in = bbs - b0;                        // in[j] = bb at chain position j
    auto floor_at = [&](int e) -> float {              // avg[e], canonical
        double w;
        if (exact) w = pre[e - b0 + 1] - pre[e - b0 + 1 - L];
        else { w = 0.0; for (int t = e - L + 1; t <= e; t++) w += (double)in[t]; }
        return __fmul_rn((float)w, P.scale_a);
    };
    unsigned long long n_cand = 0, n_rep = 0, n_drop = 0, n_alt = 0;
    unsigned my_last = 0u;
    for (int e = e0 + tid; e < j1; e += AMB_MODEAC_THREADS) {
        const float x = in[e];
        if (!(in[e - 1] < x) || in[e + 1] > x) continue;                                    // rule 1 (peak part)
        const float av = floor_at(e);
        const float thr_lvl = __fmul_rn(av, P.thr);
        if (!(x > thr_lvl)) continue;                                                       // rule 1
        const float f2 = in[e + G.slot[14]];
        if (f2 < thr_lvl) continue;                                                         // rule 2
        if (e >= j0) n_cand++;
        const float avgpeak = __fdiv_rn(__fadd_rn(x, f2), 2.0f);                            // rule 3
        const float space = __fadd_rn(av, __fdiv_rn(__fsub_rn(avgpeak, av), P.thr));
        const float clear = __fmul_rn(thr_lvl, P.thr);                                       // rule 4
        if (!(x > space) || !(f2 > space) || !(x > clear) || !(f2 > clear) || in[e + G.slot[7]] > space) continue;
        bool quiet = true;
#pragma unroll
        for (int g = 0; g < 14; g++) quiet = quiet && !(in[e + G.gap[g]] > space);          // rule 5
        if (!quiet) continue;
        my_last = (unsigned)(e - e0) + 1u;
        atomicOr(&s_pass[(e - e0) >> 5], 1u << ((e - e0) & 31));
        if (e >= j0) atomicOr(&s_reply[(e - j0) >> 5], 1u << ((e - j0) & 31));
    }
    if (my_last) atomicMax(&s_last, my_last);
    __syncthreads();
    for (int e = j0 + tid; e < j1; e += AMB_MODEAC_THREADS) {                             // rule 7
        if (!((s_reply[(e - j0) >> 5] >> ((e - j0) & 31)) & 1u)) continue;
        const int lo = e - G.back;
        bool drop = false;
        for (int j = max(lo, e0); j < e && !drop; j++) drop = (s_pass[(j - e0) >> 5] >> ((j - e0) & 31)) & 1u;
        if (!drop && lo < a.j_lo && *a.last_prev)
            drop = (long long)(*a.last_prev) - 1 >= a.org + lo;
        if (drop) n_drop++;
        else atomicOr(&s_keep[(e - j0) >> 5], 1u << ((e - j0) & 31));
    }
    __syncthreads();
    for (int e = j0 + tid; e < j1; e += AMB_MODEAC_THREADS) {                             // rule 6, records
        const int r = e - j0;
        if (!((s_keep[r >> 5] >> (r & 31)) & 1u)) continue;
        int rank = __popc(s_keep[r >> 5] & ((1u << (r & 31)) - 1u));
        for (int w = 0; w < (r >> 5); w++) rank += __popc(s_keep[w]);
        const float x = in[e], av = floor_at(e), f2 = in[e + G.slot[14]];
        const float avgpeak = __fdiv_rn(__fadd_rn(x, f2), 2.0f);
        const float space = __fadd_rn(av, __fdiv_rn(__fsub_rn(avgpeak, av), P.thr));
        int code = 0;
        for (int k = 1; k <= 13; k++) code |= (in[e + G.slot[k]] > space ? 1 : 0) << (13 - k);
        amb_modeac m{};
        m.sample_index = (uint64_t)(a.org + e);
        m.peak = avgpeak; m.floor = av;
        m.code = (uint16_t)code; m.squawk = (uint16_t)amb_decode_id(code);
        m.altitude = amb_modeac_altitude(code);
        m.spi = in[e + G.spi] > space ? 1 : 0;
        a.rec[(size_t)blockIdx.x * a.cap_tile + rank] = m;
        n_rep++;
        if (m.altitude != AMB_NO_ALTITUDE) n_alt++;
    }
    unsigned long long cnt[4] = {n_cand, n_rep, n_drop, n_alt};
#pragma unroll
    for (int k = 0; k < 4; k++) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) cnt[k] += __shfl_xor_sync(FULL, cnt[k], d);
        if (lane == 0 && cnt[k]) atomicAdd(&s_cnt[k], cnt[k]);
    }
    __syncthreads();
    if (tid == 0) {
        a.tile_count[blockIdx.x] = (unsigned)s_cnt[1];
        if (s_last) atomicMax(a.last_cur, (unsigned long long)(a.org + e0 + (int)s_last));
        for (int k = 0; k < 4; k++) if (s_cnt[k]) atomicAdd(&a.stats[k], s_cnt[k]);
    }
}

// One CTA of 32 warps: the call's replies, tile by tile in order, appended to the queue; the carried last start of
// rules 1-5. Warp w owns a contiguous run of tiles: it sums their counts (coalesced), the 32 sums give each run its
// offset, and the warp then walks its run 32 tiles at a time with a shuffle scan, each lane copying one tile's replies.
#define AMB_MODEAC_EMIT_THREADS 1024
__global__ void __launch_bounds__(AMB_MODEAC_EMIT_THREADS) amb_modeac_emit_kernel(const AmbModeacArgs a, int n_tiles)
{
    __shared__ unsigned s_warp[AMB_MODEAC_EMIT_THREADS / 32];
    __shared__ unsigned s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int per = (n_tiles + AMB_MODEAC_EMIT_THREADS / 32 - 1) / (AMB_MODEAC_EMIT_THREADS / 32);
    const int t_lo = min(n_tiles, warp * per), t_hi = min(n_tiles, t_lo + per);
    unsigned tot = 0;
    for (int t = t_lo + lane; t < t_hi; t += 32) tot += a.tile_count[t];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) tot += __shfl_xor_sync(FULL, tot, d);
    if (lane == 0) s_warp[warp] = tot;
    if (threadIdx.x == 0) {
        s_base = *a.q_count;
        if (*a.last_cur > *a.last_prev) *a.last_prev = *a.last_cur;
        *a.last_cur = 0ull;
    }
    __syncthreads();
    unsigned base = s_base;
    for (int w = 0; w < warp; w++) base += s_warp[w];
    for (int t0 = t_lo; t0 < t_hi; t0 += 32) {
        const int t = t0 + lane;
        const unsigned c = t < t_hi ? a.tile_count[t] : 0u;
        unsigned inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const unsigned v = __shfl_up_sync(FULL, inc, d); if (lane >= d) inc += v; }
        for (unsigned r = 0; r < c; r++) a.queue[base + inc - c + r] = a.rec[(size_t)t * a.cap_tile + r];
        base += __shfl_sync(FULL, inc, 31);
    }
    if (threadIdx.x == AMB_MODEAC_EMIT_THREADS - 1) *a.q_count = base;     // the last warp's run ends the call's replies
}

size_t amb_modeac_smem_bytes(const AmbModeacArgs& a)
{
    // m2 (nb_cap + AMB_MAX_SPC floats) lives where the prefix (na_cap + 1 doubles) goes later
    return (size_t)(a.na_cap + 1) * sizeof(double) + (size_t)a.nb_cap * sizeof(float);
}

int amb_launch_modeac(const AmbModeacArgs& a, cudaStream_t s, cudaError_t* err)
{
    const int n_tiles = (a.j_hi - a.j_lo + AMB_MODEAC_TILE - 1) / AMB_MODEAC_TILE;
    const size_t smem = amb_modeac_smem_bytes(a);
    *err = cudaFuncSetAttribute(amb_modeac_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (*err != cudaSuccess) return 0;
    AMB_LAUNCH((amb_modeac_tile_kernel), n_tiles, AMB_MODEAC_THREADS, smem, s, a);
    AMB_LAUNCH((amb_modeac_emit_kernel), 1, AMB_MODEAC_EMIT_THREADS, 0, s, a, n_tiles);
    *err = cudaGetLastError();
    return 2;
}
