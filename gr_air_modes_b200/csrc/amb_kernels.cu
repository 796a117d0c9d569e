// sm_90a kernels of the Mode S receive hot path. Citations are file:line under gr-air-modes.
//
// Pipeline per amb_process() call (all on one CUDA stream, nothing round-trips to the host):
//   scan     amb_scan_kernel      streaming pass over IQ (8 B/sample, the HBM-bound kernel): |x|^2, pulse
//                                 matched filter, noise-floor window and the first four pulse tests of
//                                 preamble_impl.cc:173-179 as a CONSERVATIVE fp32 pre-filter -> candidate bitmap
//   compact  amb_compact_kernel   bitmap -> ordered candidate list
//   exact    amb_exact_kernel     one warp per candidate: canonical arithmetic (bit-for-bit the checker's),
//                                 re-checks :173-179, late-gate :182-192, quiet zones :198-209
//   resolve  amb_walk_*           reproduces the visit order of the sequential scan loop (:172, :190, :209,
//                                 :212-216, :237) over the sparse candidate list
//   slice    amb_slice_kernel     one warp per accepted preamble: 240-chip extraction :219-221, llslicer
//                                 slicer_impl.cc:67-100, packet rules :117-182, CRC modes_crc.cc:55-63
#include "amb_internal.h"

#define FULL 0xffffffffu

__constant__ unsigned int c_crc_rem[96]; // x^(t+24) mod 0xFFF409, t = distance of a message bit from the parity field

// ------------------------------------------------------------------------------------------------
// small PTX helpers: mbarrier + TMA tensor copy (SASS: UTMALDG / SYNCS)
// ------------------------------------------------------------------------------------------------
// int(j * d_samples_per_chip) of preamble_impl.cc:220: int -> float, float multiply, truncation (per context, so no
// shared table: two contexts with different rates can coexist on one device)
__device__ __forceinline__ int chip_off(int j, float spc_f) { return __float2int_rz(__fmul_rn((float)j, spc_f)); }

#ifndef AMB_SIMT_EMUL   // PTX (mbarrier / TMA): tests/simt supplies host stand-ins for these six helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// 2-D tiled TMA load: box {32 floats, 32 lines} = 4 KiB = 512 complex samples, 128B-swizzled in shared memory
__device__ __forceinline__ void tma_tile_g2s(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ bool elect_one() {   // one lane of the (converged) warp; lets ptxas keep TMA operands uniform
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

#endif

__device__ __forceinline__ const float2* seg_ptr(const AmbSegs& S, int j) {
    if (j < S.n_carry) return S.carry + j;
    j -= S.n_carry;
    if (j < S.n_main) return S.main_ + j;
    return S.tail + (j - S.n_main);
}

// ------------------------------------------------------------------------------------------------
// scan kernel
// ------------------------------------------------------------------------------------------------
// Work decomposition: the evaluated range is cut into contiguous spans of rows_per_span rows; a row is
// 256 samples = one 2 KiB TMA tile, EIGHT consecutive samples per lane. ONE WARP owns a span and streams
// through it on its own with a private 4-deep tile ring (lane 0 issues cp.async.bulk.tensor, all lanes wait
// on the tile's mbarrier). There is no block-level barrier; a CTA is four independent warps.
//
// Shared-memory layouts are all bank-conflict free for 32 B-per-lane accesses:
//   * IQ tiles are written by TMA with the 128B swizzle (16 B chunk index ^= 128 B line index mod 8); a lane
//     reads its 64 B (8 samples) as 4 LDS.128 from pre-computed swizzled offsets.
//   * the warp's own arrays (filtered samples `bb`, row-local prefix `pr`) store 16 B chunk c at c ^ ((c>>3)&1).
//
// Arithmetic (deliberately NOT the canonical one - this is a filter, the exact stage decides):
//   m2 = re*re + im*im (fma); bbs = sum of the last FL m2 (all-positive adds, unscaled PMF);
//   Pr = row-local inclusive prefix of bbs (warp scan), Rt = row total;
//   W[n] = sum of the last L bbs = (A - Pr_kd[posd]) + Pr_k[pos], A = totals of the rows in between.
//   Exact test (preamble_impl.cc:173-174) is  bb > fl(avg*T)  with bb = fl(S1)*sp, avg = fl(sum bb)*sa;
//   sp cancels, so it is implied by  bbs >= cT*W - G  with cT = T*sa*(1-eps)^2 and the absolute guard
//   G = cT*gfac*(Rt+A) >= cT * (accumulated rounding of W): every operand of W is <= Rt+A and fewer than
//   32 roundings of 2^-24 enter it, gfac = 2^-19. (The ring actually holds cT*Pr so that cT*W - G costs two adds.) Tests :177-179 use the same lowered threshold; the
//   peak test in[i+1] > in[i] (:175) is relaxed by (1+eps); eps = 2^-15 dwarfs the <= 2^-19 relative error
//   of bbs. Result: a superset of the reference's candidates, typically < 0.01 % larger.
// PREF (compile-time pulse offsets 2,7,9*SPC): 2 = all four pulses from registers + shuffles, no look-ahead ring
// (best for short filters, where noise crosses the threshold often); 1 = second pulse from registers as a quick
// per-lane reject, the others from the shared-memory ring (best for SPC >= 4); 0 = run-time offsets, ring only.
template <int SPC, bool PMF, int PREF> struct ScanCfg {
    static constexpr int FL = PMF ? SPC : 1;       // pulse-matched-filter length (rx_path.py:48-51)
    static constexpr int L = 48 * SPC;             // noise-floor window (rx_path.py:54)
    static constexpr int LW = L / 8;               // ... in lanes
    static constexpr int RB = L / AMB_ROW;
    static constexpr int LMOD = L % AMB_ROW;
    static constexpr int PRR = RB + 2;             // prefix ring rows: k, ..., k-RB-1
    static constexpr int NST = 2;                  // TMA tile ring depth per warp (tile = 2 rows = 4 KiB)
    static constexpr int WARM = (RB + 2 + 1) & ~1;
    static constexpr int IQ_BYTES = NST * 4096;                    // per warp, 1 KiB aligned
    static constexpr int BB_FLOATS = (PREF == 2) ? 0 : 512;               // look-ahead ring only when pulse offsets are run-time values
    static constexpr int WORK_BYTES = BB_FLOATS * 4 + PRR * 1024 + 64;  // [bb ring,] pr ring, mbarriers
    static constexpr int CTA_BYTES = 4 * (IQ_BYTES + WORK_BYTES);
};

// float index p (0..255 within a row slot) -> swizzled float index
__device__ __forceinline__ int swz(int p) { return p ^ ((p >> 3) & 4); }

struct RowRegs { float b[8]; float t[8]; };

template <int SPC, bool PMF, int PREF>
struct ScanWarp {
    using C = ScanCfg<SPC, PMF, PREF>;
    int lane;
    const AmbScanArgs* a;
    unsigned char* iq;      // tile ring
    float* bbr;             // 2 rows x 256 floats
    float* prr;             // PRR rows x 256 floats
    uint32_t iq_s, bar0;
    int off[4];             // swizzled byte offsets of this lane's 4 IQ chunks within a row of a tile
    int own;                // swizzled float offset of this lane's first own chunk (chunks own, own^4)
    int ownd;               // same for the lane LW lanes back (window tail)
    bool hi; int rows_back;
    float rth[C::RB + 1];
    float lastm[8];         // previous row's m2 of this lane (PMF look-back across the row boundary)
    uint32_t cw, cnt;
    int ra, rb;
    int ppos;               // slot of the current row in the prefix ring = row index mod PRR

    // tile t = rows 2t, 2t+1 = 512 samples = 32 lines of 128 B. Three separate issues so that each uses a
    // compile-time descriptor address (a run-time selected pointer makes ptxas emit a uniformisation loop).
    __device__ __forceinline__ void issue(int t, int slot) const {
        const AmbSegs& S = a->S;
        const int j = t * AMB_TILE;
        const uint32_t bar = bar0 + 8 * slot, dst = iq_s + 4096 * slot;
        mbar_expect_tx(bar, 4096);
        if (j >= S.n_carry && j < S.n_carry + S.n_main) tma_tile_g2s(dst, &a->tm_main, 0, (j - S.n_carry) >> 4, bar);
        else if (j < S.n_carry) tma_tile_g2s(dst, &a->tm_carry, 0, j >> 4, bar);
        else tma_tile_g2s(dst, &a->tm_tail, 0, (j - S.n_carry - S.n_main) >> 4, bar);
    }

    // element (8*lane + r + PO) of the previous row, continuing into the current row: registers + one shuffle
    template <int PO>
    __device__ __forceinline__ float ahead(int r, const float* pb, const float* cb) const {
        const int d = (r + PO) >> 3, reg = (r + PO) & 7;      // compile-time once r is unrolled
        if (d == 0) return pb[reg];
        const float src = (lane >= d) ? pb[reg] : cb[reg];
        return __shfl_sync(FULL, src, (lane + d) & 31);
    }

    // one row: compute cur from the tile half at `st`, evaluate prev (row k-1)
    __device__ __forceinline__ void step(int k, const unsigned char* st, RowRegs& cur, const RowRegs& prev) {
        float m[8];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const float4 v = *reinterpret_cast<const float4*>(st + off[q]);
            m[2 * q] = fmaf(v.x, v.x, v.y * v.y);
            m[2 * q + 1] = fmaf(v.z, v.z, v.w * v.w);
        }
        // ---- pulse matched filter: unscaled sum of the last FL samples, all-positive adds
        float* b = cur.b;
        if (C::FL > 1) {
            float v[C::FL - 1 + 8];
#pragma unroll
            for (int r = 0; r < 8; r++) v[C::FL - 1 + r] = m[r];
#pragma unroll
            for (int t = 1; t < C::FL; t++) {
                const int d = (t + 7) / 8;                 // lanes back
                const int ridx = (8 * d - t);              // register of that lane
                const float src = (lane > 31 - d) ? lastm[ridx] : m[ridx];
                v[C::FL - 1 - t] = __shfl_sync(FULL, src, (lane - d) & 31);
            }
            if (C::FL >= 8) {
                // the 8 windows v[r .. r+FL-1] share the core v[7 .. FL-1]; what differs is a suffix of v[0..6] and a
                // prefix of v[FL .. FL+6]: FL + 18 all-positive adds instead of 4 FL + 8 (same error bound: <= FL roundings)
                float core = v[7];
#pragma unroll
                for (int i = 8; i < C::FL; i++) core += v[i];
                float lft[8], rgt[8];
                lft[7] = 0.f; lft[6] = v[6];
#pragma unroll
                for (int i = 5; i >= 0; i--) lft[i] = v[i] + lft[i + 1];
                rgt[0] = 0.f; rgt[1] = v[C::FL];
#pragma unroll
                for (int i = 2; i < 8; i++) rgt[i] = rgt[i - 1] + v[C::FL + i - 1];
                b[0] = lft[0] + core; b[7] = core + rgt[7];
#pragma unroll
                for (int r = 1; r < 7; r++) b[r] = (lft[r] + core) + rgt[r];
            } else if (C::FL >= 4) {
                // pair sums shared between neighbouring outputs: s2[i] = v[i] + v[i+1]; all-positive, same bound
                float s2[C::FL - 1 + 8 - 1];
#pragma unroll
                for (int i = 0; i < C::FL - 1 + 8 - 1; i++) s2[i] = v[i] + v[i + 1];
#pragma unroll
                for (int r = 0; r < 8; r++) {          // window v[r .. r+FL-1]
                    float s = s2[r];
#pragma unroll
                    for (int t = 2; t + 1 < C::FL; t += 2) s += s2[r + t];
                    if (C::FL & 1) s += v[r + C::FL - 1];
                    b[r] = s;
                }
            } else {
#pragma unroll
                for (int r = 0; r < 8; r++) {
                    float s = v[C::FL - 1 + r];
#pragma unroll
                    for (int t = 1; t < C::FL; t++) s += v[C::FL - 1 + r - t];
                    b[r] = s;
                }
            }
#pragma unroll
            for (int r = 0; r < 8; r++) lastm[r] = m[r];
        } else {
#pragma unroll
            for (int r = 0; r < 8; r++) b[r] = m[r];
        }
        // ---- row-local inclusive prefix
        float p[8];
        p[0] = b[0];
#pragma unroll
        for (int r = 1; r < 8; r++) p[r] = p[r - 1] + b[r];
        float inc = p[7];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const float y = __shfl_up_sync(FULL, inc, d);
            if (lane >= d) inc += y;
        }
        float exc = __shfl_up_sync(FULL, inc, 1);
        if (lane == 0) exc = 0.f;
        const float Rt = __shfl_sync(FULL, inc, 31);
        // the ring stores q = cT * prefix, so that the thresholds need two adds per sample (below)
        const float cT = a->P.cT;
        const float cexc = cT * exc;
#pragma unroll
        for (int r = 0; r < 8; r++) p[r] = fmaf(cT, p[r], cexc);
        float* bslot = bbr + (k & 1) * 256;
        float* pslot = prr + ppos * 256;                       // ppos == k % PRR, carried (no division in the loop)
        if (PREF != 2) {
            *reinterpret_cast<float4*>(bslot + own) = make_float4(b[0], b[1], b[2], b[3]);
            *reinterpret_cast<float4*>(bslot + (own ^ 4)) = make_float4(b[4], b[5], b[6], b[7]);
        }
        *reinterpret_cast<float4*>(pslot + own) = make_float4(p[0], p[1], p[2], p[3]);
        *reinterpret_cast<float4*>(pslot + (own ^ 4)) = make_float4(p[4], p[5], p[6], p[7]);
        __syncwarp();
        // ---- noise-floor window sums and lowered thresholds of row k
        float A = 0.f;
#pragma unroll
        for (int mm = 0; mm < C::RB; mm++) A += rth[mm];
        if (hi) A += rth[C::RB];
        int dpos = ppos - rows_back; dpos += dpos < 0 ? C::PRR : 0;
        const float* dslot = prr + dpos * 256;
        ppos = ppos + 1 == C::PRR ? 0 : ppos + 1;
        const float4 d0 = *reinterpret_cast<const float4*>(dslot + ownd);
        const float4 d1 = *reinterpret_cast<const float4*>(dslot + (ownd ^ 4));
        // t = cT*W - G with cT*W = (cT*A - q_kd[posd]) + q_k[pos]; every term is a product of cT and a partial sum
        // <= Rt+A, so the absolute guard G = cT*gfac*(Rt+A) still covers all roundings (two more than before).
        const float cA = cT * A;
        const float g = fmaf(cT * a->P.gfac, Rt + A, 1e-42f);   // + absolute slack for sums of denormals
        const float cAg = cA - g;
        cur.t[0] = (cAg - d0.x) + p[0]; cur.t[1] = (cAg - d0.y) + p[1];
        cur.t[2] = (cAg - d0.z) + p[2]; cur.t[3] = (cAg - d0.w) + p[3];
        cur.t[4] = (cAg - d1.x) + p[4]; cur.t[5] = (cAg - d1.y) + p[5];
        cur.t[6] = (cAg - d1.z) + p[6]; cur.t[7] = (cAg - d1.w) + p[7];
        // ---- evaluate row k-1 (its look-ahead reaches into row k, now in registers / the ring)
        const int ke = k - 1;
        if (ke >= ra) {
            // A candidate needs all four preamble pulses above the (lowered) threshold of its start sample
            // (:174, :177-179). With integer samples/chip the pulse offsets are the compile-time 2,7,9*SPC and
            // the look-ahead comes from registers + one shuffle each; otherwise only the first pulse is
            // tested here and the rest from the shared-memory ring below.
            float u[8];
#pragma unroll
            for (int r = 0; r < 8; r++) u[r] = prev.b[r];
            bool first = true;
            if (PREF == 1 && C::FL >= 8) {   // long filters: noise rarely crosses the threshold (1.5e-3 per sample at 10 samples/chip,
                                             // 1.3e-2 at 5), so two rows in three end here after 8 compares and a vote
                bool h0 = false;
#pragma unroll
                for (int r = 0; r < 8; r++) h0 = h0 || !(u[r] < prev.t[r]);
                first = __any_sync(FULL, h0);
            }
            if (!first) {
            } else
            if (PREF == 2) {
#pragma unroll
                for (int r = 0; r < 8; r++)
                    u[r] = fminf(fminf(u[r], ahead<2 * SPC>(r, prev.b, b)),
                                 fminf(ahead<7 * SPC>(r, prev.b, b), ahead<9 * SPC>(r, prev.b, b)));
            } else if (PREF == 1) {
#pragma unroll
                for (int r = 0; r < 8; r++) u[r] = fminf(u[r], ahead<2 * SPC>(r, prev.b, b));
            }
            bool hot = false;
#pragma unroll
            for (int r = 0; r < 8; r++) hot = hot || !(u[r] < prev.t[r]);   // negated '<': a NaN/Inf-contaminated threshold must not hide candidates
            if (first && __any_sync(FULL, hot)) {
                const float nx = ahead<1>(7, prev.b, b);       // first sample of the next lane / row
                uint32_t msk = 0;
                if (hot) {
                    const float oe = a->P.one_eps;
#pragma unroll
                    for (int r = 0; r < 8; r++) {
                        const float nxt = (r < 7) ? prev.b[r + 1] : nx;
                        // an all-zero stretch has b == 0 and must not flood the list although 0 >= lowered threshold;
                        // peak test :175 with relative + absolute (denormal) slack
                        // (b > 0 is necessary for :174 because the threshold is never negative)
                        // comparisons are written the way the reference's are (:175 '>' and :177-179 '<' are false on NaN)
                        if (prev.b[r] > 0.f && !(u[r] < prev.t[r]) && !(nxt > fmaf(prev.b[r], oe, 1e-42f))) msk |= 1u << r;
                    }
                    const int jb = ke * AMB_ROW + 8 * lane;
                    if (jb < a->j_lo || jb + 8 > a->j_hi) {   // only the first / last row of a call
#pragma unroll
                        for (int r = 0; r < 8; r++) if (jb + r < a->j_lo || jb + r >= a->j_hi) msk &= ~(1u << r);
                    }
                    if (PREF != 2) {
                        const int rbase = (ke & 1) * 256 + 8 * lane;
                        const int po1 = a->P.po1, po2 = a->P.po2, po3 = a->P.po3;
                        uint32_t todo = msk;
                        while (todo) {                         // tests :177-179 from the shared-memory ring
                            const int r = __ffs(todo) - 1;
                            todo &= todo - 1;
                            float th = prev.t[0];
#pragma unroll
                            for (int rr = 1; rr < 8; rr++) th = (r == rr) ? prev.t[rr] : th;
                            const int q = rbase + r;
                            const float x1 = bbr[swz((q + po1) & 511)];
                            const float x2 = bbr[swz((q + po2) & 511)];
                            const float x3 = bbr[swz((q + po3) & 511)];
                            if (fminf(fminf(x1, x2), x3) < th) msk &= ~(1u << r);
                        }
                    }
                }
                if (__any_sync(FULL, msk != 0)) {
                    // natural bit order: word w covers samples 32w..32w+31 of the row = lanes 4w..4w+3
                    uint32_t e[8];
#pragma unroll
                    for (int r = 0; r < 8; r++) e[r] = __ballot_sync(FULL, (msk >> r) & 1u);
                    if (lane < 8) {
                        uint32_t w = 0;
#pragma unroll
                        for (int r = 0; r < 8; r++) {
                            const uint32_t x = (e[r] >> (4 * lane)) & 0xFu;
                            w |= ((x & 1u) | ((x & 2u) << 7) | ((x & 4u) << 14) | ((x & 8u) << 21)) << r;
                        }
                        a->fine[(size_t)ke * 8 + lane] = w;
                    }
#pragma unroll
                    for (int r = 0; r < 8; r++) cnt += __popc(e[r]);
                    cw |= 1u << (ke & 31);
                }
            }
            if ((ke & 31) == 31 || ke == rb - 1) {
                if (lane == 0) a->coarse[ke >> 5] = cw;
                cw = 0;
            }
        }
#pragma unroll
        for (int mm = C::RB; mm > 0; mm--) rth[mm] = rth[mm - 1];
        rth[0] = Rt;
        __syncwarp();
    }
};

// Register cap of the scan kernel. Four of its CTAs are resident per SM for the whole pass (one wave); at 112 registers
// they leave 8 K registers (and ~60 KiB of shared memory) per SM free, which is what lets the sparse kernels of the
// previous call (<= 128 threads x 64 registers, or 64 x 128) run UNDER the scan instead of after it. 112 is applied
// where it costs no spills (spc <= 2). spc 3..5: 120 registers leave 4 K registers (and 25 KiB of shared memory) for the
// sparse kernels, so that they overlap the scan. spc >= 6: the prefix ring leaves too little shared memory for anything
// to be resident beside the scan, so it keeps every register. (The SM's 64 K registers and 228 KiB of shared memory are
// the same on sm_90 and sm_100.)
template <int SPC, bool PMF, int PREF>
__global__ void __maxnreg__((SPC) <= 2 ? 112 : (SPC) <= 5 ? 120 : 128) amb_scan_kernel(const __grid_constant__ AmbScanArgs a)
{
    using C = ScanCfg<SPC, PMF, PREF>;
    AMB_DYN_SMEM(unsigned char, smem, 1024);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int span = blockIdx.x * 4 + warp;
    if (span >= a.n_spans) return;

    ScanWarp<SPC, PMF, PREF> w;
    w.lane = lane; w.a = &a;
    w.iq = smem + warp * C::IQ_BYTES;
    unsigned char* work = smem + 4 * C::IQ_BYTES + warp * C::WORK_BYTES;
    w.bbr = reinterpret_cast<float*>(work);
    w.prr = w.bbr + C::BB_FLOATS;
    w.iq_s = smem_u32(w.iq);
    w.bar0 = smem_u32(w.prr + C::PRR * 256);
    {   // TMA 128B swizzle: 16 B chunk index (bits 4-6) ^= 128 B line index (bits 7-9)
        const int line = lane >> 1, c0 = 4 * (lane & 1);
#pragma unroll
        for (int q = 0; q < 4; q++) w.off[q] = line * 128 + (((c0 + q) ^ (line & 7)) << 4);
    }
    w.own = swz(8 * lane);
    w.ownd = swz(8 * ((lane - C::LW) & 31));
    w.hi = (C::LMOD != 0) && (8 * lane < C::LMOD);
    w.rows_back = C::RB + (w.hi ? 1 : 0);
#pragma unroll
    for (int m = 0; m <= C::RB; m++) w.rth[m] = 0.f;
#pragma unroll
    for (int r = 0; r < 8; r++) w.lastm[r] = 0.f;
    w.cw = 0; w.cnt = 0;
    w.ra = a.row_lo + span * a.rows_per_span;              // evaluate rows [ra, rb)
    w.rb = min(w.ra + a.rows_per_span, a.row_hi);
    const int rs = max(w.ra - C::WARM, 0);                 // first row computed (even; window warm-up)
    const int t0 = rs >> 1;
    w.ppos = (2 * t0) % C::PRR;
    const int ntiles = (w.rb >> 1) - t0 + 1;               // row rb is computed as look-ahead only

    for (int i = lane; i < C::BB_FLOATS; i += 32) w.bbr[i] = 0.f;
    for (int i = lane; i < C::PRR * 256; i += 32) w.prr[i] = 0.f;
    if (lane == 0) {
        for (int s = 0; s < C::NST; s++) mbar_init(w.bar0 + 8 * s, 1);
        fence_mbar_init();
    }
    __syncwarp();
    if (lane == 0) {
        const int pre = ntiles < C::NST ? ntiles : C::NST;
        for (int s = 0; s < pre; s++) w.issue(t0 + s, s);
    }
    RowRegs ra_, rb_;
#pragma unroll
    for (int r = 0; r < 8; r++) { ra_.b[r] = ra_.t[r] = rb_.b[r] = rb_.t[r] = 0.f; }
    int slot = 0; uint32_t par = 0;
    for (int tl = 0; tl < ntiles; tl++) {
        while (!mbar_try_wait(w.bar0 + 8 * slot, par)) {}
        const unsigned char* st = w.iq + slot * 4096;
        const int k = (t0 + tl) << 1;
        w.step(k, st, ra_, rb_);
        if (k + 1 <= w.rb) w.step(k + 1, st + 2048, rb_, ra_);
        __syncwarp();
        if (tl + C::NST < ntiles) {                         // refill this slot with tile tl+NST (warp-uniform condition)
            if (elect_one()) w.issue(t0 + tl + C::NST, slot);
        }
        if (++slot == C::NST) { slot = 0; par ^= 1u; }
    }
    if (lane == 0) {
        a.span_count[span] = w.cnt;
        if (w.cnt) atomicAdd(&a.group_count[span >> 6], w.cnt);
    }
}

size_t amb_scan_smem_bytes(int spc_i)
{
    switch (spc_i) {
#define CASE(n) case n: return (size_t)ScanCfg<n, true, 0>::CTA_BYTES;
        CASE(1) CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10)
#undef CASE
    }
    return 0;
}

template <int SPC, bool PMF, int PREF>
static cudaError_t launch_scan_t(const AmbScanArgs& a, cudaStream_t s)
{
    const size_t smem = (size_t)ScanCfg<SPC, PMF, PREF>::CTA_BYTES;
    cudaError_t e = cudaFuncSetAttribute(amb_scan_kernel<SPC, PMF, PREF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    // whole L1 as shared memory: the scan does not use L1 (TMA), and the ~60 KiB its four CTAs leave over are what the
    // sparse kernels of the previous call need to be resident beside them (the split is only reconfigured on an idle SM)
    e = cudaFuncSetAttribute(amb_scan_kernel<SPC, PMF, PREF>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (e != cudaSuccess) return e;
    const int blocks = (a.n_spans + 3) / 4;
    AMB_LAUNCH((amb_scan_kernel<SPC, PMF, PREF>), blocks, 128, smem, s, a);
    return cudaGetLastError();
}

cudaError_t amb_launch_scan(const AmbScanArgs& a, int, cudaStream_t s)
{
    // integer samples/chip: pulse offsets are the compile-time 2,7,9*SPC (register/shuffle look-ahead)
    const bool pref = a.P.po1 == 2 * a.P.spc_i && a.P.po2 == 7 * a.P.spc_i && a.P.po3 == 9 * a.P.spc_i;
    switch (a.P.spc_i) {
#define CASE(n) case n: return a.P.use_pmf ? (pref ? launch_scan_t<n, true, (n <= 3 ? 2 : 1)>(a, s) : launch_scan_t<n, true, 0>(a, s)) \
                                          : (pref ? launch_scan_t<n, false, 2>(a, s) : launch_scan_t<n, false, 0>(a, s));
        CASE(1) CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10)
#undef CASE
        default: break;
    }
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------
// compaction: (coarse, fine) bitmap -> ordered candidate list. One warp per scan span, so the order is
// span order x row order x bit order = ascending sample index. Offsets come from the per-span counts.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) amb_compact_kernel(const __grid_constant__ AmbScanArgs a, int* __restrict__ cand_j,
                                                          unsigned int cap, AmbCounters* ctr,
                                                          unsigned long long* scratch64, int n_scratch64)
{
    // per-call resets of what the later kernels of this call accumulate into
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_scratch64; k += gridDim.x * blockDim.x) scratch64[k] = 0ull;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        ctr->ndet_call = 0; ctr->npassed_call = 0; ctr->nreal_call = 0; ctr->ndet_list = 0; ctr->nec_fixed = 0;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int span = blockIdx.x * 4 + warp;
    if (span >= a.n_spans) return;
    unsigned int off = 0;                                   // candidates before this span: whole groups of 64 spans + the rest
    for (int g = lane; g < (span >> 6); g += 32) off += a.group_count[g];
    for (int w = (span & ~63) + lane; w < span; w += 32) off += a.span_count[w];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) off += __shfl_xor_sync(FULL, off, d);
    const int ra = a.row_lo + span * a.rows_per_span;
    const int rb = min(ra + a.rows_per_span, a.row_hi);
    const int cw_end = (rb + 31) >> 5;
    unsigned int running = off;
    for (int cwb = ra >> 5; cwb < cw_end; cwb += 32) {
        const int idx = cwb + lane;
        const uint32_t cw = idx < cw_end ? a.coarse[idx] : 0u;
        unsigned int cnt = 0;
        for (uint32_t m = cw; m; m &= m - 1) {
            const int row = idx * 32 + (__ffs(m) - 1);
            const uint4 f0 = *reinterpret_cast<const uint4*>(a.fine + (size_t)row * 8);
            const uint4 f1 = *reinterpret_cast<const uint4*>(a.fine + (size_t)row * 8 + 4);
            cnt += __popc(f0.x) + __popc(f0.y) + __popc(f0.z) + __popc(f0.w) +
                   __popc(f1.x) + __popc(f1.y) + __popc(f1.z) + __popc(f1.w);
        }
        unsigned int inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned int y = __shfl_up_sync(FULL, inc, d);
            if (lane >= d) inc += y;
        }
        unsigned int o = running + inc - cnt;
        for (uint32_t m = cw; m; m &= m - 1) {
            const int row = idx * 32 + (__ffs(m) - 1);
            for (int q = 0; q < 8; q++)
                for (uint32_t w = a.fine[(size_t)row * 8 + q]; w; w &= w - 1) {
                    if (o < cap) cand_j[o] = row * AMB_ROW + q * 32 + (__ffs(w) - 1);
                    o++;
                }
        }
        running += __shfl_sync(FULL, inc, 31);
    }
    if (span == a.n_spans - 1 && lane == 0) {
        ctr->ncand = running < cap ? running : cap;
        if (running > cap) ctr->overflow = 1;
    }
}

cudaError_t amb_launch_compact(const AmbScanArgs& a, int* cand_j, unsigned int cand_cap, AmbCounters* ctr,
                               void* walk_scratch, long long n_samples, cudaStream_t s)
{
    const int n64 = walk_scratch ? (int)(32 + (n_samples >> 20) + 8) : 0;   // AmbParScratch header + time buckets
    AMB_LAUNCH((amb_compact_kernel), (a.n_spans + 3) / 4, 128, 0, s, a, cand_j, cand_cap, ctr,
                                                           reinterpret_cast<unsigned long long*>(walk_scratch), n64);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// canonical arithmetic (the definition DESIGN.md gives; the CPU checker used by tests/ states the same):
//   m2  = fl(fl(re*re) + fl(im*im))                         complex_to_mag_squared, no FMA
//   bb  = fl( (float)(fp64 ascending sum of spc_i m2) * scale_p )   moving_average_ff(spc, 1/spc)   rx_path.py:49
//   avg = fl( (float)(fp64 ascending sum of L bb)   * scale_a )     moving_average_ff(48 spc, ...)  rx_path.py:54
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float canon_m2(const AmbSegs& S, int j)
{
    if (j < 0 || j >= S.n_carry + S.n_main + S.n_tail) return 0.f;
    const float2 v = *seg_ptr(S, j);
    return __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
}
// pointer to the logical samples [j, j+count) when they lie inside ONE segment (the common case), else nullptr
__device__ __forceinline__ const float2* seg_span(const AmbSegs& S, int j, int count)
{
    if (j < 0) return nullptr;
    if (j + count <= S.n_carry) return S.carry + j;
    const int t0 = S.n_carry + S.n_main;
    if (j >= S.n_carry && j + count <= t0) return S.main_ + (j - S.n_carry);
    if (j >= t0 && j + count <= t0 + S.n_tail) return S.tail + (j - t0);
    return nullptr;
}
__device__ __forceinline__ float canon_m2_of(float2 v) { return __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)); }

// split form: the caller supplies the two float streams; x is in reported coordinates (history-biased)
__device__ __forceinline__ float stream_at(const float* in, long long n, int H, long long x)
{
    const long long k = x - H;
    return (k >= 0 && k < n) ? in[k] : 0.f;
}


// ---- exact stage ----------------------------------------------------------------------------------
// A warp takes G consecutive candidates (G = 32 / 16 / 8 by samples per chip) in two phases:
//   gather    all 32 lanes copy every candidate's span of the recording - the L + maxlate + fwd + fl samples its
//             verdict depends on - into that candidate's ROW of shared memory as m2 = |x|^2: 16-byte loads from
//             even sample positions, neighbouring lanes read neighbouring addresses, 8 loads in flight per lane (and up to 12 warps per SM), so
//             a group costs a handful of memory round trips whatever its size;
//   evaluate  lane t owns candidate t and walks its row alone: pulse matched filter in place (row[i] <- bb), the fp64
//             ascending sum of bb[c-L+1 .. c] = LITERALLY the canonical noise-floor window of the start c, then the
//             pulse tests, the late gate and the quiet zones from the row. Rows have an odd stride, so 32 lanes
//             walking 32 rows in step never collide on a bank. No shuffles, no votes: 32 candidates advance per warp
//             instruction (the warp-per-candidate kernel spends a whole warp and five barriers on ONE candidate,
//             which makes it instruction-bound in dense traffic).
// After a late shift the window of c+i is acc - head + tail when every addend's exponent lies within 19 of the
// others (then every partial sum of <= 1024 such floats is exact in fp64, 24+19+10 = 53 bits, so any association
// gives the canonical bits); otherwise that window is summed again, literally ascending.
// Writes info = late | real<<8 | valid<<9 and avg at the shifted index.
// SPC > 0: integer samples/chip geometry known at compile time (loops fold); SPC == 0: run-time values.
template <int SPC, bool PMF>
__global__ void __launch_bounds__(64) amb_exact_kernel(const AmbExactArgs a, const int G, const int ROW)
{
    AMB_DYN_SMEM(float, ex_smem, 16);
    const AmbParams& P = a.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int spc = SPC ? SPC : P.spc_i;
    const int L = 48 * spc, maxlate = SPC ? SPC : P.maxlate;
    const int po1 = SPC ? 2 * SPC : P.po1, po2 = SPC ? 7 * SPC : P.po2, po3 = SPC ? 9 * SPC : P.po3;
    const int qa0 = SPC ? 3 * SPC : P.qa0, qa1 = SPC ? 6 * SPC : P.qa1, qb0 = SPC ? 10 * SPC : P.qb0, qb1 = SPC ? 15 * SPC : P.qb1;
    const int fwd = SPC ? 15 * SPC + 2 : P.fwd;
    constexpr int FLC = (PMF && SPC > 1) ? SPC : 1;          // compile-time filter length (1 = none / run-time)
    const int fl = PMF ? spc : 1;                            // pulse matched filter length
    const int nf = maxlate + fwd + 2;                        // forward values: bb[c .. c+nf-1]
    const int NB = L + nf - 1;                               // bb values per candidate: bb[c-L+1 .. c+nf-1]
    const int NM = NB + fl - 1;                              // m2 values behind them
    const int P2 = (NM + 2) / 2;                             // 16-byte pairs per row (rows start at an even sample)
    float* rows = ex_smem + (size_t)warp * ((size_t)G * ROW + 64);
    const float4** ptrs = reinterpret_cast<const float4**>(rows + (size_t)G * ROW);   // G span pointers (8 B each, <= 32)
    const unsigned int ncand = a.ctr->ncand;
    if (ncand <= a.dense_threshold) return;                  // sparse traffic: amb_exact_warp_kernel's regime
    const float scale_p = P.scale_p, scale_a = P.scale_a;
    const unsigned int ngroups = (ncand + G - 1) / G;
    for (unsigned int grp = blockIdx.x * 2 + warp; grp < ngroups; grp += gridDim.x * 2) {
        const unsigned int ci = grp * G + lane;
        const bool valid = lane < G && ci < ncand;
        const int c = valid ? a.cand_j[ci] : 0;
        const int b_m2 = c - L + 1 - (fl - 1);               // logical index of the first m2 sample
        const int be = b_m2 & ~1;                            // even start (also for negative indices)
        if (lane < G) {
            const float2* sp = valid ? seg_span(a.S, be, 2 * P2) : nullptr;
            ptrs[lane] = reinterpret_cast<const float4*>(sp);      // 16-byte aligned: segment bases are, `be` is even
        }
        __syncwarp();
        // ---- gather: element e of the group = pair p of row q; a lane's elements are e = lane, lane + 32, ...
        const int total = G * P2;
        int gq = lane / P2, gp = lane - gq * P2;               // P2 >= 34: at most one row change per step of 32
        for (int e0 = 0; e0 < total; e0 += 32 * 8) {
            float4 v[8];
            int q = gq, p = gp;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (e0 + 32 * u + lane < total) {
                    const float4* sp = ptrs[q];
                    if (sp) v[u] = __ldg(sp + p);
                }
                p += 32; if (p >= P2) { p -= P2; q++; }
            }
            q = gq; p = gp;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                if (e0 + 32 * u + lane < total && ptrs[q]) {   // rows without a pointer are filled below
                    float* r = rows + (size_t)q * ROW + 2 * p;
                    r[0] = __fadd_rn(__fmul_rn(v[u].x, v[u].x), __fmul_rn(v[u].y, v[u].y));
                    r[1] = __fadd_rn(__fmul_rn(v[u].z, v[u].z), __fmul_rn(v[u].w, v[u].w));
                }
                p += 32; if (p >= P2) { p -= P2; q++; }
            }
            gq = q; gp = p;
        }
        __syncwarp();
        // rows whose span is not inside one segment (first / last samples of a call): filled sample by sample
        for (unsigned todo = __ballot_sync(FULL, valid && lane < G && !ptrs[lane < G ? lane : 0]); todo; todo &= todo - 1) {
            const int q = __ffs(todo) - 1;
            const int bq = __shfl_sync(FULL, be, q);
            float* r = rows + (size_t)q * ROW;
            for (int k = lane; k < 2 * P2; k += 32) r[k] = canon_m2(a.S, bq + k);
        }
        __syncwarp();
        // ---- evaluate: lane t, candidate t
        if (valid) {
            float* r = rows + (size_t)lane * ROW + (b_m2 - be);     // r[k] = m2[b_m2 + k]; becomes bb[c-L+1+k] in place
            double acc = 0.0;
            float mx = 0.f, mn = 3.0e38f;                     // largest / smallest non-zero bb that can enter a window
            auto consume = [&](int i, float bb) {             // bb = bb[c - L + 1 + i] (never negative)
                if (i < L + maxlate) { mx = fmaxf(mx, bb); mn = bb > 0.f ? fminf(mn, bb) : mn; }
                if (i < L) acc += (double)bb;
            };
            if (FLC > 1) {
                float w[FLC];                                  // the last FLC m2 values; slot of m2 sample k: k % FLC
#pragma unroll
                for (int t = 0; t < FLC - 1; t++) w[t] = r[t];
                for (int i0 = 0; i0 < NB; i0 += FLC) {         // FLC outputs per round: ring positions are static
#pragma unroll
                    for (int u = 0; u < FLC; u++) {
                        const int i = i0 + u;
                        if (i < NB) {
                            w[(u + FLC - 1) % FLC] = r[i + FLC - 1];
                            double sum = 0.0;                  // ascending: oldest sample first
#pragma unroll
                            for (int t = 0; t < FLC; t++) sum += (double)w[(u + t) % FLC];
                            const float bb = __fmul_rn((float)sum, scale_p);
                            r[i] = bb;                         // m2[i] is not needed again
                            consume(i, bb);
                        }
                    }
                }
            } else if (PMF && fl > 1) {                       // run-time filter length
                for (int i = 0; i < NB; i++) {
                    double sum = 0.0;
                    for (int t = 0; t < fl; t++) sum += (double)r[i + t];
                    const float bb = __fmul_rn((float)sum, scale_p);
                    r[i] = bb;
                    consume(i, bb);
                }
            } else {
#pragma unroll 4
                for (int i = 0; i < NB; i++) {
                    const float bb = PMF ? __fmul_rn((float)(double)r[i], scale_p) : r[i];   // filter length 1: scale 1.0
                    if (PMF) r[i] = bb;
                    consume(i, bb);
                }
            }
            unsigned emax = __float_as_uint(mx) >> 23, emin = __float_as_uint(mn) >> 23;
            emax = emax ? emax : 1u; emin = emin ? emin : 1u;  // denormals share the quantum of exponent field 1
            if (mx == 0.f) { emax = 1u; emin = 1u; }           // all zero: trivially exact
            const float* in = r + (L - 1);                    // in[x] == reference in[i+x] at the candidate start
            const float avg0 = __fmul_rn((float)acc, scale_a);
            const float pulse_threshold = __fmul_rn(avg0, P.thr);                       // :173
            bool real = in[0] > pulse_threshold;                                        // :174
            if (real && (in[1] > in[0])) real = false;                                  // :175
            if (real && (in[po1] < pulse_threshold)) real = false;                      // :177
            if (real && (in[po2] < pulse_threshold)) real = false;                      // :178
            if (real && (in[po3] < pulse_threshold)) real = false;                      // :179
            uint32_t info = 0;
            float avg_fin = avg0;
            if (real) {
                auto corr = [&](int k) -> double {                                      // correlate_preamble :88-98 at c+k
                    double v = 0.0;
                    for (int t = 0; t < spc; t++) v += (double)in[k + t];
                    for (int t = 0; t < spc; t++) v += (double)in[k + 2 * spc + t];
                    for (int t = 0; t < spc; t++) v += (double)in[k + 7 * spc + t];
                    for (int t = 0; t < spc; t++) v += (double)in[k + 9 * spc + t];
                    return v;
                };
                int i = 0, how_late = 0;
                bool late;
                double now_corr = corr(0);
                do {                                                                    // :184-192
                    const double late_corr = corr(i + 1);
                    late = late_corr > now_corr;
                    if (late) { i++; how_late++; now_corr = late_corr; }
                } while (late && (SPC ? how_late < SPC : (float)how_late < P.spc_f));
                if (i > 0) {
                    double w = 0.0;
                    if (emax < 255u && emax <= emin + 19u) {
                        w = acc;
                        for (int k = 1; k <= i; k++) w = (w - (double)r[k - 1]) + (double)in[k];
                    } else {                                                            // literal ascending window of c+i
                        for (int t = 0; t < L; t++) w += (double)r[i + t];
                    }
                    avg_fin = __fmul_rn((float)w, scale_a);
                }
                const float sum4 = __fadd_rn(__fadd_rn(__fadd_rn(in[i], in[i + po1]), in[i + po2]), in[i + po3]);
                const float avgpeak = (float)((double)sum4 / 4.0);                      // :198-201
                const float space_threshold =
                    __fadd_rn(avg_fin, __fdiv_rn(__fsub_rn(avgpeak, avg_fin), P.thr));  // :203
                bool viol = false;
                for (int j = qa0; j <= qa1 && !viol; j++) viol = in[i + j] > space_threshold;   // :205-206
                for (int j = qb0; j <= qb1 && !viol; j++) viol = in[i + j] > space_threshold;   // :207-208
                info = (uint32_t)i | (1u << 8) | (!viol ? (1u << 9) : 0u);
            }
            a.cand_info[ci] = info;
            a.cand_avg[ci] = avg_fin;
        }
        __syncwarp();
    }
}

// ---- exact stage, sparse traffic: one WARP per candidate (round-1 kernel) -----------------------------------------
// With a few thousand candidates per call what counts is the latency of ONE candidate, not throughput: here the 32
// lanes share a candidate's window sums (order-independent when every addend's exponent lies within 19 of the others,
// else the literal ascending loop), so a candidate is decided in one memory round trip. It needs hundreds of warp
// instructions per candidate, though, which is what made dense traffic instruction-bound: beyond dense_threshold
// candidates per call amb_exact_kernel (rows + one lane per candidate) takes over. Both kernels are launched; the one
// whose regime it is not returns at once. Writes info = late | real<<8 | valid<<9 and avg at the shifted index.
// SPC > 0: integer samples/chip geometry known at compile time (loops unroll, offsets fold); SPC == 0: run-time values.
template <int SPC>
__global__ void __launch_bounds__(128) amb_exact_warp_kernel(const AmbExactArgs a)
{
    AMB_DYN_SMEM(float, ex_smem, 4);                 // per warp: m2s[NMp] then bbs[NMp], sized by the launcher
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const AmbParams& P = a.P;
    const int spc = SPC ? SPC : P.spc_i;
    const int L = 48 * spc, maxlate = SPC ? SPC : P.maxlate;
    const int po1 = SPC ? 2 * SPC : P.po1, po2 = SPC ? 7 * SPC : P.po2, po3 = SPC ? 9 * SPC : P.po3;
    const int qa0 = SPC ? 3 * SPC : P.qa0, qa1 = SPC ? 6 * SPC : P.qa1, qb0 = SPC ? 10 * SPC : P.qb0, qb1 = SPC ? 15 * SPC : P.qb1;
    const int fwd = SPC ? 15 * SPC + 2 : P.fwd;
    const int fl = P.use_pmf ? spc : 1;
    const int NB = L + maxlate + fwd + 1;
    const int NM = NB + fl - 1;
    const int NMp = (NM + 31) & ~31;
    float* m2s = ex_smem + (size_t)warp * 2 * NMp;
    float* bbs = m2s + NMp;
    const int c0off = L - 1;                        // bbs index of the candidate start
    const unsigned int ncand = a.ctr->ncand;
    if (ncand > a.dense_threshold) return;
    const int nwarps = gridDim.x * 4;
    for (unsigned int ci = blockIdx.x * 4 + warp; ci < ncand; ci += nwarps) {
        const int c = a.cand_j[ci];
        float avgk = 0.f;
        {
            const int b_bb = c - L + 1;               // bbs[i] <-> bb[b_bb + i]
            const int b_m2 = b_bb - (fl - 1);
            const float2* span = seg_span(a.S, b_m2, NM);     // warp-uniform
            if (span) {
                for (int i0 = 0; i0 < NM; i0 += 256) {        // 8 independent loads in flight per lane
                    float2 v[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) { const int i = i0 + 32 * u + lane; v[u] = i < NM ? span[i] : make_float2(0.f, 0.f); }
#pragma unroll
                    for (int u = 0; u < 8; u++) { const int i = i0 + 32 * u + lane; if (i < NM) m2s[i] = canon_m2_of(v[u]); }
                }
            } else {
                for (int i = lane; i < NM; i += 32) m2s[i] = canon_m2(a.S, b_m2 + i);   // straddles a segment boundary
            }
            __syncwarp();
            for (int i = lane; i < NB; i += 32) {
                if (P.use_pmf) {
                    double acc = 0.0;
                    for (int t = 0; t < fl; t++) acc += (double)m2s[i + t];
                    bbs[i] = __fmul_rn((float)acc, P.scale_p);
                } else {
                    bbs[i] = m2s[i];
                }
            }
            __syncwarp();
            // inavg at c+k, k <= maxlate: fp64 ascending sum of bb[c+k-L+1 .. c+k] (canonical definition).
            // If every non-zero addend's exponent lies within 19 of the others, every partial sum of <= 1024 such
            // floats is exactly representable in fp64 (24 + 19 + 10 = 53 bits), so ANY summation order - incl. a
            // lane-parallel one and the sliding update - gives the canonical bits. Otherwise (huge dynamic range,
            // Inf/NaN) fall back to the literal ascending loop.
            unsigned emax = 0u, emin = 255u;
            for (int i = lane; i < L + maxlate; i += 32) {
                const unsigned bits = __float_as_uint(bbs[i]) & 0x7fffffffu;
                if (bits) { unsigned e = bits >> 23; e = e ? e : 1u; emax = max(emax, e); emin = min(emin, e); }
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                emax = max(emax, __shfl_xor_sync(FULL, emax, d));
                emin = min(emin, __shfl_xor_sync(FULL, emin, d));
            }
            if (emax < 255u && emax <= emin + 19u) {
                double part = 0.0;
                for (int i = lane; i < L; i += 32) part += (double)bbs[i];
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) part += __shfl_xor_sync(FULL, part, d);
                double w = part;                                  // window of k = 0, identical in all lanes
                if (lane == 0) avgk = __fmul_rn((float)w, P.scale_a);
                for (int k = 1; k <= maxlate; k++) {
                    w = (w - (double)bbs[k - 1]) + (double)bbs[k + L - 1];
                    if (lane == k) avgk = __fmul_rn((float)w, P.scale_a);
                }
            } else if (lane <= maxlate) {
                double acc = 0.0;
                for (int t = 0; t < L; t++) acc += (double)bbs[lane + t];
                avgk = __fmul_rn((float)acc, P.scale_a);
            }
        }
        // correlate_preamble (preamble_impl.cc:88-98) at c+k, k = lane-16 in [0, maxlate+1]
        double corrk = 0.0;
        if (lane >= 16 && lane - 16 <= maxlate + 1) {
            const float* q = bbs + c0off + (lane - 16);
            for (int t = 0; t < spc; t++) corrk += (double)q[t];
            for (int t = 0; t < spc; t++) corrk += (double)q[2 * spc + t];
            for (int t = 0; t < spc; t++) corrk += (double)q[7 * spc + t];
            for (int t = 0; t < spc; t++) corrk += (double)q[9 * spc + t];
        }
        const float* in = bbs + c0off;                // in[x] == reference in[i+x] at the candidate start
        const float avg0 = __shfl_sync(FULL, avgk, 0);
        const float pulse_threshold = __fmul_rn(avg0, P.thr);                       // :173
        bool real = in[0] > pulse_threshold;                                        // :174
        if (real && (in[1] > in[0])) real = false;                                  // :175
        if (real && (in[po1] < pulse_threshold)) real = false;                    // :177
        if (real && (in[po2] < pulse_threshold)) real = false;                    // :178
        if (real && (in[po3] < pulse_threshold)) real = false;                    // :179
        uint32_t info = 0;
        float avg_fin = avg0;
        if (real) {
            int i = 0, how_late = 0;
            bool late;
            do {                                                                    // :184-192
                const double now_corr = __shfl_sync(FULL, corrk, 16 + i);
                const double late_corr = __shfl_sync(FULL, corrk, 16 + i + 1);
                late = late_corr > now_corr;
                if (late) { i++; how_late++; }
            } while (late && (SPC ? how_late < SPC : (float)how_late < P.spc_f));
            avg_fin = __shfl_sync(FULL, avgk, i);
            const float* s = in + i;
            const float sum4 = __fadd_rn(__fadd_rn(__fadd_rn(s[0], s[po1]), s[po2]), s[po3]);
            const float avgpeak = (float)((double)sum4 / 4.0);                      // :198-201
            const float space_threshold =
                __fadd_rn(avg_fin, __fdiv_rn(__fsub_rn(avgpeak, avg_fin), P.thr));  // :203
            bool viol = false;
            for (int j = qa0 + lane; j <= qa1; j += 32) viol |= (s[j] > space_threshold);  // :205-206
            for (int j = qb0 + lane; j <= qb1; j += 32) viol |= (s[j] > space_threshold);  // :207-208
            const bool valid = !__any_sync(FULL, viol);
            info = (uint32_t)i | (1u << 8) | (valid ? (1u << 9) : 0u);
        }
        if (lane == 0) { a.cand_info[ci] = info; a.cand_avg[ci] = avg_fin; }
        __syncwarp();
    }
}


// Split form (caller-supplied float streams): same decisions, in0/in1 play bb/avg; one thread per candidate.
__global__ void __launch_bounds__(128) amb_exact_streams_kernel(const AmbExactArgs a)
{
    const AmbParams& P = a.P;
    const int spc = P.spc_i, maxlate = P.maxlate;
    const unsigned int ncand = a.ctr->ncand;
    for (unsigned int ci = blockIdx.x * blockDim.x + threadIdx.x; ci < ncand; ci += gridDim.x * blockDim.x) {
        const long long c = a.cand_j[ci];
        auto in = [&](int x) -> float { return stream_at(a.in0, a.n_streams, P.H, c + x); };
        const float avg0 = stream_at(a.in1, a.n_streams, P.H, c);
        const float pulse_threshold = __fmul_rn(avg0, P.thr);                       // :173
        const float in0 = in(0);
        bool real = in0 > pulse_threshold;                                          // :174
        if (real && (in(1) > in0)) real = false;                                    // :175
        if (real && (in(P.po1) < pulse_threshold)) real = false;                    // :177
        if (real && (in(P.po2) < pulse_threshold)) real = false;                    // :178
        if (real && (in(P.po3) < pulse_threshold)) real = false;                    // :179
        uint32_t info = 0;
        float avg_fin = avg0;
        if (real) {
            auto corr = [&](int k) -> double {
                double v = 0.0;
                for (int t = 0; t < spc; t++) v += (double)in(k + t);
                for (int t = 0; t < spc; t++) v += (double)in(k + 2 * spc + t);
                for (int t = 0; t < spc; t++) v += (double)in(k + 7 * spc + t);
                for (int t = 0; t < spc; t++) v += (double)in(k + 9 * spc + t);
                return v;
            };
            int i = 0, how_late = 0;
            bool late;
            double now_corr = corr(0);
            do {                                                                    // :184-192
                const double late_corr = corr(i + 1);
                late = late_corr > now_corr;
                if (late) { i++; how_late++; now_corr = late_corr; }
            } while (late && (float)how_late < P.spc_f);
            (void)maxlate;
            avg_fin = stream_at(a.in1, a.n_streams, P.H, c + i);
            const float sum4 = __fadd_rn(__fadd_rn(__fadd_rn(in(i), in(i + P.po1)), in(i + P.po2)), in(i + P.po3));
            const float avgpeak = (float)((double)sum4 / 4.0);                      // :198-201
            const float space_threshold =
                __fadd_rn(avg_fin, __fdiv_rn(__fsub_rn(avgpeak, avg_fin), P.thr));  // :203
            bool viol = false;
            for (int j = P.qa0; j <= P.qa1 && !viol; j++) viol = in(i + j) > space_threshold;   // :205-206
            for (int j = P.qb0; j <= P.qb1 && !viol; j++) viol = in(i + j) > space_threshold;   // :207-208
            info = (uint32_t)i | (1u << 8) | (!viol ? (1u << 9) : 0u);
        }
        a.cand_info[ci] = info;
        a.cand_avg[ci] = avg_fin;
    }
}

template <int SPC>
static cudaError_t launch_exact_t(const AmbExactArgs& a, int blocks, int G, int ROW, size_t smem, cudaStream_t s)
{
    cudaError_t e;
    if (a.P.use_pmf) {
        e = cudaFuncSetAttribute(amb_exact_kernel<SPC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(amb_exact_kernel<SPC, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        if (e != cudaSuccess) return e;
        AMB_LAUNCH((amb_exact_kernel<SPC, true>), blocks, 64, smem, s, a, G, ROW);
    } else {
        e = cudaFuncSetAttribute(amb_exact_kernel<SPC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(amb_exact_kernel<SPC, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        if (e != cudaSuccess) return e;
        AMB_LAUNCH((amb_exact_kernel<SPC, false>), blocks, 64, smem, s, a, G, ROW);
    }
    return cudaGetLastError();
}

cudaError_t amb_launch_exact(const AmbExactArgs& a, int sm_count, cudaStream_t s)
{
    const AmbParams& P = a.P;
    if (a.in0) {
        AMB_LAUNCH((amb_exact_streams_kernel), sm_count * 8, 128, 0, s, a);
        return cudaGetLastError();
    }
    // integer samples/chip: everything the kernel needs is a multiple of spc (see compute_params)
    const int k = P.spc_i;
    const bool integral = P.spc_f == (float)k && P.maxlate == k && P.po1 == 2 * k && P.po2 == 7 * k && P.po3 == 9 * k &&
                          P.qa0 == 3 * k && P.qa1 == 6 * k && P.qb0 == 10 * k && P.qb1 == 15 * k && P.fwd == 15 * k + 2;
    const int fl = P.use_pmf ? k : 1;
    const int NM = P.L + (P.maxlate + P.fwd + 2) - 1 + fl - 1;
    const int ROW = (2 * ((NM + 2) / 2)) | 1;                        // floats per row: whole 16-byte pairs, odd stride
    const int G = ROW <= 160 ? 32 : ROW <= 340 ? 16 : 8;              // candidates per warp: <= ~21 KiB of rows per warp
    // two warps per CTA: <= 43 KiB of rows and <= 8 K registers, so that a CTA fits beside the four resident scan CTAs
    const size_t smem = (size_t)2 * ((size_t)G * ROW + 64) * sizeof(float);
    int per_sm = (int)((200 * 1024) / smem);
    if (per_sm > 6) per_sm = 6;
    if (per_sm < 1) per_sm = 1;
    const int blocks = sm_count * per_sm;
    // the warp-per-candidate kernel (sparse traffic): per warp m2s[NMp] + bbs[NMp]
    const int NBw = P.L + P.maxlate + P.fwd + 1;
    const int NMpw = (NBw + fl - 1 + 31) & ~31;
    const size_t smem_w = (size_t)4 * 2 * NMpw * sizeof(float);          // <= 22 KiB at 20 Msps, ~1.3 KiB at 4 Msps
    const int blocks_w = sm_count * 12;
    cudaError_t e;
#define AMB_EXACT_BOTH(N)                                                                         \
    AMB_LAUNCH((amb_exact_warp_kernel<N>), blocks_w, 128, smem_w, s, a);                          \
    e = cudaGetLastError();                                                                       \
    if (e != cudaSuccess) return e;                                                               \
    return launch_exact_t<N>(a, blocks, G, ROW, smem, s);
    if (integral) {
        switch (k) {
            case 1: { AMB_EXACT_BOTH(1) }
            case 2: { AMB_EXACT_BOTH(2) }
            case 5: { AMB_EXACT_BOTH(5) }
            case 10: { AMB_EXACT_BOTH(10) }
            default: break;
        }
    }
    { AMB_EXACT_BOTH(0) }
#undef AMB_EXACT_BOTH
}

// ------------------------------------------------------------------------------------------------
// resolver: exact sequential restatement of the scan loop's control flow over the candidate list.
// State (pos, p) persists across calls in AmbWalkState. See DESIGN.md "visit order".
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ long long ninputs_of(long long ntot, long long pos, int spc_i)
{
    long long R = ntot - pos;                       // items the scheduler stand-in hands over
    if (R > 0x7fffffffLL) R = 0x7fffffffLL;
    long long n = R - (R % spc_i) - spc_i;          // preamble_impl.cc:150
    return n > 0 ? n : 0;
}

// Exact sequential walk from candidate cursor `idx` with state `st`; returns detections flagged.
__device__ unsigned int seq_walk(const AmbWalkArgs& a, AmbWalkState& st, int idx, int n)
{
    const AmbParams& P = a.P;
    unsigned int ndet = 0;
    while (!st.done) {
        long long ninputs = 0, limit;
        if (a.flush) {
            ninputs = ninputs_of(a.ntot, st.pos, P.spc_i);
            if (ninputs <= 0) { st.done = 1; break; }            // :151 consume_each(0); return 0
            limit = st.pos + ninputs;                            // loop bound i < ninputs (:172)
        } else {
            limit = a.r_safe;
        }
        // first real candidate with start >= p (p can step back by one after a "no room" retry)
        while (idx > 0 && a.org + a.cand_j[idx - 1] >= st.p) idx--;
        while (idx < n && (!(a.cand_info[idx] & (1u << 8)) || a.org + a.cand_j[idx] < st.p)) idx++;
        if (idx >= n || a.org + a.cand_j[idx] >= limit) {
            if (a.flush) { st.pos += ninputs; st.p = st.pos; continue; }   // :244 consume_each(ninputs)
            if (st.p < limit) st.p = limit;                      // everything before r_safe has been looked at
            break;
        }
        const uint32_t info = a.cand_info[idx];
        const long long fin = a.org + a.cand_j[idx] + (long long)(info & 0xffu);
        if (!(info & (1u << 9))) { st.p = fin + 1; idx++; continue; }      // :209 continue -> i++
        const long long i_rel = fin - st.pos;
        if (a.flush && (float)(ninputs - i_rel) < P.skip_f) {              // :212 no room
            const long long consumed = i_rel - 1 > 0 ? i_rel - 1 : 0;      // :213
            if (consumed == 0) { st.done = 1; break; }
            st.pos += consumed; st.p = st.pos;
            continue;
        }
        a.cand_info[idx] = info | (1u << 10);                              // accepted: 240-chip packet
        a.det_list[atomicAdd(&a.ctr->ndet_list, 1u)] = idx;
        ndet++;
        const long long consumed = (long long)(int)((float)i_rel + P.skip_f);  // :237 float arithmetic
        st.pos += consumed; st.p = st.pos;
        idx++;
    }
    return ndet;
}

// Sequential resolver (always correct; one thread). Used on request ("resolver" option = 1).
__global__ void amb_walk_seq_kernel(const AmbWalkArgs a)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    AmbWalkState st = *a.st;
    const int n = (int)a.ctr->ncand;
    a.ctr->ndet_list = 0;                       // (the compaction kernel does not run in front of a tiny closing call)
    unsigned int nreal = 0;
    for (int k = 0; k < n; k++) if (a.cand_info[k] & (1u << 8)) nreal++;
    const unsigned int ndet = seq_walk(a, st, 0, n);
    st.ncand_real += nreal; st.ndet += ndet;
    *a.st = st;
    a.ctr->ndet_call = ndet;
    a.ctr->nreal_call = nreal;
    a.ctr->frame_base = a.ctr->nframes;            // the slicer's frame slots: frame_base + position in det_list
    a.ctr->nframes += a.ctr->ndet_list;
}

cudaError_t amb_launch_walk_seq(const AmbWalkArgs& a, cudaStream_t s)
{
    AMB_LAUNCH((amb_walk_seq_kernel), 1, 32, 0, s, a);
    return cudaGetLastError();
}

// ---- parity dumps of the front end (amb_dump_stage): canonical m2 / bb / avg at EVERY sample of a short buffer ---
// Brute force on purpose: this is the definition the exact stage evaluates at candidates only, written the plain way.
__global__ void amb_dump_bb_kernel(const float2* iq, long long n, AmbParams P, int stage, float* out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (stage == 0 || !P.use_pmf) { out[i] = canon_m2_of(iq[i]); return; }
    double acc = 0.0;                                           // zeros before the stream start add nothing
    for (long long k = i - P.spc_i + 1; k <= i; k++) if (k >= 0) acc += (double)canon_m2_of(iq[k]);
    out[i] = __fmul_rn((float)acc, P.scale_p);
}
__global__ void amb_dump_avg_kernel(const float* bb, long long n, AmbParams P, float* out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double acc = 0.0;
    for (long long k = i - P.L + 1; k <= i; k++) if (k >= 0) acc += (double)bb[k];
    out[i] = __fmul_rn((float)acc, P.scale_a);
}

cudaError_t amb_launch_dump(const float2* iq, long long n, const AmbParams& P, int stage, float* tmp, float* out, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    AMB_LAUNCH((amb_dump_bb_kernel), blocks, 256, 0, s, iq, n, P, stage, stage == 2 ? tmp : out);
    if (stage == 2) AMB_LAUNCH((amb_dump_avg_kernel), blocks, 256, 0, s, tmp, n, P, out);
    return cudaGetLastError();
}

// Entry state of a time-sharded span (amb_seek / amb_resolve): only where the loop stands, counters stay.
__global__ void amb_set_state_kernel(AmbWalkState* st, long long pos, long long p)
{
    st->pos = pos; st->p = p; st->done = 0;
}

cudaError_t amb_launch_set_state(AmbWalkState* st, long long pos, long long p, cudaStream_t s)
{
    AMB_LAUNCH((amb_set_state_kernel), 1, 1, 0, s, st, pos, p);
    return cudaGetLastError();
}

// ---- parallel resolver ----------------------------------------------------------------------------
// Two candidates further apart than GAP = maxlate + skip0 + 4 samples cannot influence each other through the
// scan position p: whatever happens at the earlier one, the loop index is back to plain i++ before it reaches
// the later one (an accepted packet skips at most fin + skip0 + 1, :237). So the candidate list splits into
// independent CLUSTERS at such gaps, and every cluster is walked sequentially by its own thread (pass 1).
// The one thing that crosses clusters is `pos` (nitems_read at the start of the current general_work call):
// :237 adds 240*spc to i in FLOAT, which is exact only while i = fin - pos < P.i_exact (about 2^24). Pass 1
// records every packet's consume point in 2^20-sample time buckets; pass 2 checks, for each cluster whose first
// packet was walked without knowing pos, that some earlier packet lies less than i_exact samples back (a
// non-empty bucket among the preceding (i_exact>>20)-1 ones, or the previous call's pos). If that cannot be
// shown (no packet for > ~15 M samples) the finalize kernel redoes the whole call with the exact sequential walk.
// Finalize also applies the end-of-stream rules (:150, :212-216) to the last 240*spc samples when flushing.
#define AMB_BUCKET_SHIFT 20
struct AmbParScratch {
    AmbWalkState saved;
    unsigned long long max_pos_rel1;   // 1 + (largest consume point - org), 0 = none
    unsigned long long max_p_rel1;     // 1 + (largest exit p - org)
    unsigned int violation;
    unsigned int zone_idx1;            // 1 + index of the first candidate with start >= zone (0 = none)
};

// Pass 1 keeps everything that would be a same-address atomic per packet or per cluster in registers and folds it
// once per warp at the end (with 236 k packets and 224 k clusters per call in dense traffic those atomics would be the
// kernel's whole cost); the slicer's work list is built by pass 2 from the verdict bits.
__global__ void __launch_bounds__(64) amb_walk_par1_kernel(const AmbWalkArgs a, AmbParScratch* sc, long long* first_fin,
                                                            unsigned long long* buckets, long long zone)
{
    const AmbParams& P = a.P;
    const int n = (int)a.ctr->ncand;
    const long long gap = (long long)P.maxlate + P.skip0 + 4;
    unsigned int ndet = 0, nreal = 0;
    unsigned long long my_max_pos = 0ull, my_max_p = 0ull;      // 1 + (value - org), 0 = none
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int jc = a.cand_j[c];
        const int jp = c ? a.cand_j[c - 1] : 0;
        const long long s0 = a.org + jc;
        if (a.cand_info[c] & (1u << 8)) nreal++;
        const bool head = (c == 0) || (jc - jp >= gap);
        if (s0 >= zone && (c == 0 || a.org + jp < zone)) sc->zone_idx1 = (unsigned)c + 1u;
        long long ff = -1;
        if (head && s0 < zone) {
            long long pos = -1, p = -1;                     // unknown / "not beyond this cluster's start"
            if (c == 0) { pos = a.st->pos; p = a.st->p; }   // the first cluster continues the previous call
            bool pos_known = (c == 0), any = false;
            long long last_pos = -1;
            // walk the cluster; candidate records are fetched 8 at a time (independent loads)
            int k = c, prevj = jc;
            bool more = true;
            while (more) {
                int jj[8]; uint32_t ii[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int q = k + u < n ? k + u : n - 1;
                    jj[u] = a.cand_j[q]; ii[u] = a.cand_info[q];
                }
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    if (!more) break;
                    if (k + u >= n) { more = false; break; }
                    if ((k + u > c) && (jj[u] - prevj >= gap)) { more = false; break; }   // next cluster's head
                    prevj = jj[u];
                    const long long s = a.org + jj[u];
                    if (s >= zone) { more = false; break; }
                    const uint32_t info = ii[u];
                    if ((info & (1u << 8)) && s >= p) {
                        const long long fin = s + (long long)(info & 0xffu);
                        any = true;
                        if (!(info & (1u << 9))) p = fin + 1;
                        else {
                            long long consumed;
                            if (pos_known) consumed = (long long)(int)((float)(fin - pos) + P.skip_f) - (fin - pos);
                            else { consumed = P.skip0; ff = fin; }
                            a.cand_info[k + u] = info | (1u << 10);
                            ndet++;
                            pos = fin + consumed; p = pos; pos_known = true;
                            last_pos = pos;
                            buckets[(fin - a.org) >> AMB_BUCKET_SHIFT] = 1ull;   // "a packet was consumed in this stretch": idempotent store
                        }
                    }
                }
                k += 8;
            }
            if (last_pos >= 0) my_max_pos = max(my_max_pos, (unsigned long long)(last_pos - a.org + 1));
            if (any && p >= a.org) my_max_p = max(my_max_p, (unsigned long long)(p - a.org + 1));
        }
        first_fin[c] = ff;
    }
    for (int d = 16; d > 0; d >>= 1) {
        ndet += __shfl_xor_sync(FULL, ndet, d); nreal += __shfl_xor_sync(FULL, nreal, d);
        my_max_pos = max(my_max_pos, __shfl_xor_sync(FULL, my_max_pos, d));
        my_max_p = max(my_max_p, __shfl_xor_sync(FULL, my_max_p, d));
    }
    if ((threadIdx.x & 31) == 0) {
        if (ndet) atomicAdd(&a.ctr->ndet_call, ndet);
        if (nreal) atomicAdd(&a.ctr->nreal_call, nreal);
        if (my_max_pos) atomicMax(&sc->max_pos_rel1, my_max_pos);
        if (my_max_p) atomicMax(&sc->max_p_rel1, my_max_p);
    }
}

// Pass 2: (a) the float-rounding check described above; (b) the slicer's work list = every candidate pass 1 accepted
// (verdict bit 10), appended with one atomic per block and iteration.
__global__ void __launch_bounds__(128) amb_walk_par2_kernel(const AmbWalkArgs a, AmbParScratch* sc, const long long* first_fin,
                                                            const unsigned long long* buckets)
{
    __shared__ unsigned int s_cnt[4], s_base;
    const AmbParams& P = a.P;
    const int n = (int)a.ctr->ncand;
    const int back = (int)(P.i_exact >> AMB_BUCKET_SHIFT) - 1;     // buckets wholly inside the exact range
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    bool viol = false;
    const int stride = gridDim.x * blockDim.x;
    for (int c0 = blockIdx.x * blockDim.x; c0 < n; c0 += stride) {           // block-uniform trip count
        const int c = c0 + threadIdx.x;
        bool det = false;
        if (c < n) {
            det = (a.cand_info[c] & (1u << 10)) != 0;
            const long long ff = first_fin[c];
            if (ff >= 0) {
                const int b = (int)((ff - a.org) >> AMB_BUCKET_SHIFT);
                bool safe = false;
                int lo = b - back; if (lo < 0) lo = 0;
                for (int q = b - 1; q >= lo && !safe; q--) safe = buckets[q] != 0;
                if (!safe && b - back <= 0) safe = (ff - a.st->pos) < P.i_exact;   // nothing earlier in this call: pos is the carried one (or later)
                if (!safe) viol = true;
            }
        }
        const unsigned int bal = __ballot_sync(FULL, det);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int tot = 0;
#pragma unroll
            for (int w = 0; w < 4; w++) { const unsigned int v = s_cnt[w]; s_cnt[w] = tot; tot += v; }
            s_base = tot ? atomicAdd(&a.ctr->ndet_list, tot) : 0u;
        }
        __syncthreads();
        if (det) a.det_list[s_base + s_cnt[warp] + __popc(bal & ((1u << lane) - 1u))] = c;
        __syncthreads();
    }
    if (__any_sync(FULL, viol) && lane == 0) sc->violation = 1;
}

__global__ void amb_walk_finalize_kernel(const AmbWalkArgs a, AmbParScratch* sc)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    AmbWalkState st = *a.st;
    const int n = (int)a.ctr->ncand;
    if (sc->violation) {                 // float rounding at :237 may matter: exact sequential walk of the whole call
        for (int k = 0; k < n; k++) a.cand_info[k] &= ~(1u << 10);
        a.ctr->ndet_list = 0;
        st.fallback = 1;
        const unsigned int ndet = seq_walk(a, st, 0, n);
        st.ndet += ndet; st.ncand_real += a.ctr->nreal_call;
        a.ctr->ndet_call = ndet;
        *a.st = st;
        a.ctr->frame_base = a.ctr->nframes;
        a.ctr->nframes += a.ctr->ndet_list;
        return;
    }
    st.fallback = 0;
    if (sc->max_pos_rel1) { const long long v = (long long)sc->max_pos_rel1 - 1 + a.org; if (v > st.pos) st.pos = v; }
    if (sc->max_p_rel1) { const long long v = (long long)sc->max_p_rel1 - 1 + a.org; if (v > st.p) st.p = v; }
    unsigned int extra = 0;
    if (a.flush) {
        const int lo = sc->zone_idx1 ? (int)sc->zone_idx1 - 1 : n;   // first candidate with start >= zone (from pass 1)
        extra = seq_walk(a, st, lo, n);
    } else if (st.p < a.r_safe) {
        st.p = a.r_safe;
    }
    st.ndet += a.ctr->ndet_call + extra; st.ncand_real += a.ctr->nreal_call;
    a.ctr->ndet_call += extra;
    *a.st = st;
    a.ctr->frame_base = a.ctr->nframes;            // the slicer's frame slots: frame_base + position in det_list
    a.ctr->nframes += a.ctr->ndet_list;
}

size_t amb_walk_scratch_bytes(unsigned int cand_cap, long long n_samples)
{
    return 256 + (size_t)cand_cap * sizeof(long long) + ((size_t)(n_samples >> AMB_BUCKET_SHIFT) + 8) * sizeof(unsigned long long);
}

cudaError_t amb_launch_walk_par(const AmbWalkArgs& a, void* scratch, unsigned int cand_cap, long long n_samples, cudaStream_t s)
{
    AmbParScratch* sc = reinterpret_cast<AmbParScratch*>(scratch);
    unsigned long long* buckets = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(scratch) + 256);
    const size_t nb = (size_t)(n_samples >> AMB_BUCKET_SHIFT) + 8;
    long long* first_fin = reinterpret_cast<long long*>(buckets + nb);
    (void)cand_cap;
    cudaError_t e;                                          // scratch header + buckets were zeroed by the prologue kernel
    const long long guard = (long long)a.P.maxlate + a.P.skip0 + 2 * a.P.spc_i + 8;
    const long long zone = a.flush ? (a.ntot - guard) : a.r_safe;
    // latency-bound (dependent loads per candidate): many small CTAs (<= 4 K registers each) so that dense traffic has
    // ~300 k threads in flight; with a few thousand candidates almost all of them exit at once
    const int sms = a.sm_count > 0 ? a.sm_count : 8;
    AMB_LAUNCH((amb_walk_par1_kernel), sms * 32, 64, 0, s, a, sc, first_fin, buckets, zone);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    AMB_LAUNCH((amb_walk_par2_kernel), sms * 16, 128, 0, s, a, sc, first_fin, buckets);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    AMB_LAUNCH((amb_walk_finalize_kernel), 1, 32, 0, s, a, sc);
    return cudaGetLastError();
}

// ---- time-sharded spans resolved speculatively (amb_resolve twice, amb_get_walk_summary) ------------------------
// Forget a previous resolution of the same call: verdict bits, work list, frames, resolver scratch.
__global__ void amb_walk_reset_kernel(const AmbWalkArgs a, unsigned long long* scratch64, int n64)
{
    const int n = (int)a.ctr->ncand;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) a.cand_info[c] &= ~(1u << 10);
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n64; k += gridDim.x * blockDim.x) scratch64[k] = 0ull;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.ctr->ndet_call = 0; a.ctr->npassed_call = 0; a.ctr->nreal_call = 0; a.ctr->ndet_list = 0; a.ctr->nframes = 0;
        a.ctr->nec_fixed = 0;
        a.st->done = 0; a.st->fallback = 0;
    }
}

cudaError_t amb_launch_walk_reset(const AmbWalkArgs& a, void* scratch, long long n_samples, cudaStream_t s)
{
    const int n64 = scratch ? (int)(32 + (n_samples >> AMB_BUCKET_SHIFT) + 8) : 0;   // as the compaction kernel clears it
    AMB_LAUNCH((amb_walk_reset_kernel), a.sm_count > 0 ? a.sm_count : 8, 256, 0, s, a,
               reinterpret_cast<unsigned long long*>(scratch), n64);
    return cudaGetLastError();
}

// What the NEXT resolution of this call could be sensitive to: the first candidate that passes the pulse tests
// (an entry p beyond it changes the walk) and the first accepted preamble (its skip is computed in float from pos).
__global__ void amb_walk_summary_kernel(const AmbWalkArgs a)
{
    const int n = (int)a.ctr->ncand;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const uint32_t info = a.cand_info[c];
        if (!(info & (1u << 8))) continue;
        const unsigned long long s0 = (unsigned long long)(a.org + a.cand_j[c]);
        atomicMin(&a.st->first_real, s0);
        if (info & (1u << 10)) atomicMin(&a.st->first_packet, s0 + (info & 0xffu));
    }
}

cudaError_t amb_launch_walk_summary(const AmbWalkArgs& a, cudaStream_t s)
{
    cudaError_t e = cudaMemsetAsync(&a.st->first_real, 0xff, 2 * sizeof(unsigned long long), s);
    if (e != cudaSuccess) return e;
    AMB_LAUNCH((amb_walk_summary_kernel), a.sm_count > 0 ? a.sm_count : 8, 256, 0, s, a);
    return cudaGetLastError();
}

// ---- time-sharded spans, hand-over without the host (amb_walk_summary_async / amb_compose_entries_async /
// amb_resolve_device): the six numbers of a span's speculative resolution go to device memory, every rank composes the
// true entries of all spans from the all-gathered table in a one-thread kernel, and the last span (never speculated on)
// takes its entry state straight from that kernel's output.
__global__ void amb_pack_summary_kernel(const AmbWalkState* st, const AmbCounters* ctr, long long i_exact, int have, long long* out)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    out[0] = st->pos; out[1] = st->p;
    out[2] = (have && st->first_real != ~0ull) ? (long long)st->first_real : -1;
    out[3] = (have && st->first_packet != ~0ull) ? (long long)st->first_packet : -1;
    out[4] = i_exact;
    out[5] = have ? (long long)ctr->npassed_call : 0;
}
// out[0] = first span whose speculation does not hold (n_spans - 1 if all hold); out[1 + 2k], out[2 + 2k] = true entry
// (pos, p) of span k; out[1 + 2 n_spans + k] = messages queued before span k - all valid for k <= out[0].
__global__ void amb_compose_kernel(const long long* g, int n_spans, long long* out)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int last = n_spans - 1;
    long long pos_in = 0, p_in = 0, queued = 0;
    long long* ent = out + 1; long long* qd = out + 1 + 2 * n_spans;
    ent[0] = 0; ent[1] = 0; qd[0] = 0;
    int bad = last;
    for (int k = 0; k < last; k++) {
        const long long pos = g[6 * k], p = g[6 * k + 1], first_real = g[6 * k + 2], first_packet = g[6 * k + 3];
        const long long exact_span = g[6 * k + 4], passed = g[6 * k + 5];
        const bool ok = (first_real < 0 || p_in <= first_real) && (first_packet < 0 || first_packet - pos_in < exact_span);
        if (!ok) { bad = k; break; }
        pos_in = first_packet >= 0 ? pos : pos_in;
        p_in = p > p_in ? p : p_in;
        queued += passed;
        ent[2 * (k + 1)] = pos_in; ent[2 * (k + 1) + 1] = p_in; qd[k + 1] = queued;
    }
    out[0] = bad;
}
__global__ void amb_set_state_dev_kernel(AmbWalkState* st, const long long* entry)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    st->pos = entry[0]; st->p = entry[1]; st->done = 0;
}
cudaError_t amb_launch_pack_summary(const AmbWalkArgs& a, long long i_exact, int have, long long* out, cudaStream_t s)
{
    AMB_LAUNCH((amb_pack_summary_kernel), 1, 32, 0, s, a.st, a.ctr, i_exact, have, out);
    return cudaGetLastError();
}
cudaError_t amb_launch_compose(const long long* gathered, int n_spans, long long* out, cudaStream_t s)
{
    AMB_LAUNCH((amb_compose_kernel), 1, 32, 0, s, gathered, n_spans, out);
    return cudaGetLastError();
}
cudaError_t amb_launch_set_state_dev(AmbWalkState* st, const long long* entry, cudaStream_t s)
{
    AMB_LAUNCH((amb_set_state_dev_kernel), 1, 32, 0, s, st, entry);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// slicer: one warp per accepted preamble
// ------------------------------------------------------------------------------------------------
// llslicer (slicer_impl.cc:67-100): bit 0 = decision, bit 1 = confidence. The three limits depend only on the
// packet's reference level, so they are computed once per packet: highlimit = (float)(ref*1.414) (:71),
// lowlimit = (float)(ref*0.707) (:72), and the fp64 product lowlimit*0.5 of :91/:94.
__device__ __forceinline__ int llslice(float bit0, float bit1, float highlimit, float lowlimit, double lowhalf)
{
    const bool f = (bit0 > lowlimit) && (bit0 < highlimit);
    const bool s = (bit1 > lowlimit) && (bit1 < highlimit);
    if (f && !s) return 1 | 2;
    if (s && !f) return 0 | 2;
    if (f && s) return (bit0 > bit1) ? 1 : 0;
    const bool d = bit0 > bit1;
    const bool c = d ? ((double)bit1 < lowhalf) : ((double)bit0 < lowhalf);   // :91 / :94
    return (d ? 1 : 0) | (c ? 2 : 0);
}

// Packet rules of slicer_impl::work (slicer_impl.cc:117-182). Executed by a full warp; bit j of the packet belongs
// to lane j % 32. `pair(j, b0, b1)` yields chips 16+2j and 17+2j (:133,:147); p0/p2/p7/p9 are the preamble chips of
// the reference level. The second half of the packet is only fetched and sliced when the header says it is a long
// one (:140), which is all the reference looks at, too. Lane 0..31 fill *f (sample_index/secs/frac are the caller's).
template <class PairFn>
__device__ __forceinline__ bool slice_packet_warp(float p0, float p2, float p7, float p9, PairFn pair, amb_frame* f,
                                                  int lane, const unsigned int* crc_rem)
{
    const float ref = (float)((double)__fadd_rn(__fadd_rn(__fadd_rn(p0, p2), p7), p9) / 4.0);   // :128-131
    const float highlimit = (float)((double)ref * 1.414);                     // :71
    const float lowlimit = (float)((double)ref * 0.707);                      // :72
    const double lowhalf = (double)lowlimit * 0.5;
    uint32_t dw[4] = {0u, 0u, 0u, 0u}, lw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int k = 0; k < 2; k++) {                      // bits 0..63
        float b0, b1;
        pair(32 * k + lane, b0, b1);
        const int r = llslice(b0, b1, highlimit, lowlimit, lowhalf);
        dw[k] = __brev(__ballot_sync(FULL, r & 1));    // MSB-first: bit 31 <-> j = 32k
        lw[k] = __ballot_sync(FULL, !(r & 2));         // bit lane <-> low confidence at j
    }
    const unsigned hdr = dw[0] >> 27;                                         // :135-139
    const bool is_long = (hdr == 16 || hdr == 17 || hdr == 20 || hdr == 21); // :140
    const int nbits = is_long ? 112 : 56;                                     // :142
    if (is_long) {                                     // warp-uniform
#pragma unroll
        for (int k = 2; k < 4; k++) {
            const int j = 32 * k + lane;
            int r = 2;
            if (j < 112) { float b0, b1; pair(j, b0, b1); r = llslice(b0, b1, highlimit, lowlimit, lowhalf); }
            dw[k] = __brev(__ballot_sync(FULL, r & 1));
            lw[k] = __ballot_sync(FULL, !(r & 2));
        }
        dw[3] &= 0xFFFF0000u; lw[3] &= 0x0000FFFFu;
    } else {
        dw[1] &= 0xFFFFFF00u; lw[1] &= 0x00FFFFFFu;
    }
    // CRC over the first nbits-24 bits (modes_crc.cc:55-63) as an XOR fold of per-bit remainders
    uint32_t crc = 0;
    const int nmsg = nbits - 24;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int j = 32 * k + lane;
        if (j < nmsg && ((dw[k] >> (31 - lane)) & 1u)) crc ^= crc_rem[nmsg - 1 - j];   // shared memory: per-lane index
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) crc ^= __shfl_xor_sync(FULL, crc, d);
    // ---- packet rules, evaluated by every lane on warp-uniform values; the stores are spread over lanes
    const uint32_t lowtot = __popc(lw[0]) + __popc(lw[1]) + __popc(lw[2]) + __popc(lw[3]);
    const unsigned numlow = lowtot < 24u ? lowtot : 24u;                      // :157 saturates at 24
    const unsigned df = dw[0] >> 27;                                          // :168 (data[0] >> 3) & 0x1F
    // last three bytes = bits nbits-24 .. nbits-1
    const uint32_t ap = is_long ? (((dw[2] & 0xFFu) << 16) | (dw[3] >> 16)) : (dw[1] >> 8) & 0xFFFFFFu;
    const bool zeroes = (dw[0] | dw[1] | dw[2] | dw[3]) == 0;                 // :162-166
    bool passed = !zeroes;
    if (passed && !is_long && df != 11 && numlow > 0) passed = false;         // :170
    if (passed && df == 11 && numlow >= 10) passed = false;                   // :171
    uint32_t syn = 0;
    if (passed) {
        syn = crc ^ ap;                                                       // :173-177
        if (syn && (df == 11 || df == 17)) passed = false;                    // :182
    }
    if (lane < 14) f->data[lane] = (uint8_t)(dw[lane >> 2] >> (24 - 8 * (lane & 3)));
    if (lane < 24 && (unsigned)lane >= numlow) f->lowconfbits[lane] = 0;      // :152-158: ascending j, first 24
    if (lowtot) {
        unsigned before = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if ((lw[k] >> lane) & 1u) {
                const unsigned rank = before + __popc(lw[k] & ((1u << lane) - 1u));
                if (rank < 24u) f->lowconfbits[rank] = (uint8_t)(32 * k + lane);
            }
            before += __popc(lw[k]);
        }
    }
    if (lane == 24) f->ec = 0;                                                // the error correction fills these (amb_ec_kernel)
    if (lane == 25) f->ec_flips = 0;
    if (lane >= 26 && lane < 30) f->pad_[lane - 26] = 0;
    if (lane == 31) {
        f->ref_level = ref;
        f->crc = syn;
        f->nbits = (uint8_t)nbits;
        f->df = (uint8_t)df;
        f->numlowconf = (uint8_t)numlow;
        f->passed = passed ? 1 : 0;
    }
    return passed;
}

// One warp per accepted preamble. Chip j of the packet is in[fin + int(j*spc)] - inavg[fin] (preamble_impl.cc:219-221).
// The packet's span of the recording (240*spc + fl samples) is copied into shared memory as m2 by ONE batch of
// 16-byte loads per lane; the work-list entry and candidate record of the NEXT packet are fetched while the current
// one is sliced, so a packet costs one memory round trip. The frame slot is frame_base + position in the work list
// (no atomics), bits are sliced straight from the staged samples (no chip array unless the caller asked for chips).
// SPC > 0: integer samples/chip (chip offsets j*SPC and the filter loop fold at compile time); SPC == 0: run-time values.
template <bool STREAMS, int SPC, bool PMF>
__global__ void __launch_bounds__(64) amb_slice_kernel(const AmbSliceArgs a, const int spanp)
{
    __shared__ unsigned int s_crc[96];
    AMB_DYN_SMEM(float, sl_smem, 16);                        // per warp: m2 of the packet span (not in STREAMS mode)
    for (int i = threadIdx.x; i < 96; i += blockDim.x) s_crc[i] = c_crc_rem[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const AmbParams& P = a.P;
    const unsigned int ndet = a.ctr->ndet_list;                // accepted preambles of this call (any order)
    const unsigned int base = a.ctr->frame_base;               // frames queued before this call
    const unsigned int nwarps = gridDim.x * 2;
    constexpr int FLC = (PMF && SPC > 0) ? SPC : 1;            // compile-time filter length (SPC == 0: run-time `fl`)
    const int fl = PMF ? (SPC ? SPC : P.spc_i) : 1;
    auto off = [&](int j) -> int { return SPC ? j * SPC : chip_off(j, P.spc_f); };   // int(j * spc) of preamble_impl.cc:220
    const int span = off(239) + fl;                            // m2 samples a packet touches
    float* m2s = sl_smem + (size_t)warp * spanp;
    unsigned int npassed = 0;
    unsigned int di = blockIdx.x * 2 + warp;
    int n_j = 0; uint32_t n_info = 0; float n_avg = 0.f;       // record of the packet about to be processed
    if (di < ndet) { const int ci = a.det_list[di]; n_j = a.cand_j[ci]; n_info = a.cand_info[ci]; n_avg = a.cand_avg[ci]; }
    for (; di < ndet; di += nwarps) {
        const int fin = n_j + (int)(n_info & 0xffu);
        const float avg_fin = n_avg;
        if (di + nwarps < ndet) {                              // prefetch the next record (independent of the work below)
            const int ci = a.det_list[di + nwarps]; n_j = a.cand_j[ci]; n_info = a.cand_info[ci]; n_avg = a.cand_avg[ci];
        }
        const int b0 = fin - fl + 1;                           // m2 index behind chip offset 0
        const int be = b0 & ~1;                                // even start: 16-byte loads
        const int sh = b0 - be;
        if (!STREAMS) {
            const int pairs = (span + sh + 1) / 2;
            const float4* src = reinterpret_cast<const float4*>(seg_span(a.S, be, 2 * pairs));   // warp-uniform
            if (src) {
                for (int p0 = 0; p0 < pairs; p0 += 256) {      // 8 independent loads in flight per lane
                    float4 v[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) { const int p = p0 + 32 * u + lane; v[u] = p < pairs ? __ldg(src + p) : make_float4(0.f, 0.f, 0.f, 0.f); }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int p = p0 + 32 * u + lane;
                        if (p < pairs) {
                            m2s[2 * p] = __fadd_rn(__fmul_rn(v[u].x, v[u].x), __fmul_rn(v[u].y, v[u].y));
                            m2s[2 * p + 1] = __fadd_rn(__fmul_rn(v[u].z, v[u].z), __fmul_rn(v[u].w, v[u].w));
                        }
                    }
                }
            } else {
                for (int i = lane; i < 2 * pairs; i += 32) m2s[i] = canon_m2(a.S, be + i);   // straddles a segment boundary
            }
            __syncwarp();
        }
        auto chip = [&](int j) -> float {
            const int o = off(j);
            if (STREAMS) return __fsub_rn(stream_at(a.in0, a.n_streams, P.H, (long long)fin + o), avg_fin);
            float bb;
            if (PMF) {                                         // bb[fin + o] = PMF over m2[fin+o-fl+1 .. fin+o]
                double acc = 0.0;
                if (SPC) {
#pragma unroll
                    for (int t = 0; t < FLC; t++) acc += (double)m2s[sh + o + t];
                } else {
                    for (int t = 0; t < fl; t++) acc += (double)m2s[sh + o + t];
                }
                bb = __fmul_rn((float)acc, P.scale_p);
            } else {
                bb = m2s[sh + o];
            }
            return __fsub_rn(bb, avg_fin);
        };
        const unsigned int slot = base + di;
        if (slot < a.frame_cap) {
            amb_frame* f = a.frames + slot;
            const bool passed = slice_packet_warp(chip(0), chip(2), chip(7), chip(9),
                                                  [&](int j, float& x0, float& x1) { x0 = chip(16 + 2 * j); x1 = chip(17 + 2 * j); },
                                                  f, lane, s_crc);
            if (lane == 0) {
                f->sample_index = (uint64_t)(a.org + fin);
                f->secs = 0; f->frac = 0.0;
                if (passed) npassed++;
            }
            if (a.chips_out) for (int j = lane; j < 240; j += 32) a.chips_out[(size_t)slot * 240 + j] = chip(j);
        } else if (lane == 0) {
            a.ctr->frame_overflow = 1;
        }
        __syncwarp();
    }
    if (lane == 0 && npassed) atomicAdd(&a.ctr->npassed_call, npassed);
}

template <int SPC, bool PMF>
static cudaError_t launch_slice_t(const AmbSliceArgs& a, int blocks, size_t smem, int spanp, cudaStream_t s)
{
    cudaError_t e = cudaFuncSetAttribute(amb_slice_kernel<false, SPC, PMF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(amb_slice_kernel<false, SPC, PMF>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (e != cudaSuccess) return e;
    AMB_LAUNCH((amb_slice_kernel<false, SPC, PMF>), blocks, 64, smem, s, a, spanp);
    return cudaGetLastError();
}

cudaError_t amb_launch_slice(const AmbSliceArgs& a, int sm_count, cudaStream_t s)
{
    const AmbParams& P = a.P;
    const int fl = P.use_pmf ? P.spc_i : 1;
    const int spanp = ((int)(239 * P.spc_f) + fl + 3 + 31) & ~31;       // span + the alignment sample(s), rounded
    const size_t smem = a.in0 ? 0 : (size_t)2 * spanp * sizeof(float);  // two warps per CTA (<= 4 K registers): 19 KiB at 20 Msps, 4 KiB at 4 Msps
    int per_sm = smem ? (int)((200 * 1024) / smem) : 32;
    if (per_sm > 32) per_sm = 32;
    if (per_sm < 1) per_sm = 1;
    const int blocks = sm_count * per_sm;
    if (a.in0) {
        AMB_LAUNCH((amb_slice_kernel<true, 0, false>), blocks, 64, smem, s, a, spanp);
        return cudaGetLastError();
    }
    const int k = P.spc_i;
    if (P.spc_f == (float)k) {                                           // integer samples/chip: int(j * spc) == j * k
        switch (k) {
#define CASE(N) case N: return P.use_pmf ? launch_slice_t<N, true>(a, blocks, smem, spanp, s) : launch_slice_t<N, false>(a, blocks, smem, spanp, s);
            CASE(1) CASE(2) CASE(5) CASE(10)
#undef CASE
            default: break;
        }
    }
    return P.use_pmf ? launch_slice_t<0, true>(a, blocks, smem, spanp, s) : launch_slice_t<0, false>(a, blocks, smem, spanp, s);
}

// slicer only (split-form block): packets of 240 chips already in device memory
__global__ void __launch_bounds__(128) amb_slice_chips_kernel(const float* __restrict__ chips_in, int ndet, amb_frame* frames)
{
    __shared__ unsigned int s_crc[96];
    if (threadIdx.x < 96) s_crc[threadIdx.x] = c_crc_rem[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = blockIdx.x * 4 + warp; d < ndet; d += gridDim.x * 4) {
        const float* c = chips_in + (size_t)d * 240;
        slice_packet_warp(c[0], c[2], c[7], c[9], [&](int j, float& x0, float& x1) { x0 = c[16 + 2 * j]; x1 = c[17 + 2 * j]; },
                          frames + d, lane, s_crc);
    }
}
cudaError_t amb_launch_slice_chips(const float* chips, int ndet, amb_frame* frames, cudaStream_t s)
{
    if (ndet <= 0) return cudaSuccess;
    int blocks = (ndet + 3) / 4; if (blocks > 2048) blocks = 2048;
    AMB_LAUNCH((amb_slice_chips_kernel), blocks, 128, 0, s, chips, ndet, frames);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// error correction (option "ec" = K, off by default): the frames slicer_impl.cc:182 drops - passed == 0 with crc != 0,
// i.e. DF11 / DF17 with a non-zero syndrome - are searched for the subsets S of their low-confidence bits L
// (lowconfbits minus the DF field, bits 0-4) whose flips zero the syndrome. The syndrome is linear over GF(2): flipping
// message bit j XORs crc_rem[nbits-25-j] into it, flipping parity bit j XORs 1 << (nbits-1-j). So instead of trying
// 2^|L| subsets, a 24-step elimination spread over the warp decides the system: lane i holds the syndrome vector of
// L[i] and the subset (a mask of lanes) it currently stands for, pivots travel by shuffle. The syndrome outside the span
// of L: no solution; inside it with rank < |L|: several solutions; otherwise exactly one, which is applied.
// A warp reads 32 frame headers, ballots the candidates and solves them one after the other (O(24 |L|) each).
//
// Second phase (option "ec_any" = M in {1, 2}, off by default): a DF17 frame still dropped after the first phase is
// searched for the patterns of at most M bits anywhere in 5..111 whose flips zero the syndrome, whatever their
// confidence. The 107 one-bit syndromes s_i and the 5,671 two-bit syndromes s_i ^ s_j are non-zero and pairwise
// distinct over these positions, so a fit is unique when it exists. Lane l owns positions 5+l, 37+l, 69+l, 101+l: it
// tests syn == s_i, and looks syn ^ s_i up in a CTA-wide hash of (s_j -> j) for a partner j > i. DF11 is left alone:
// its parity carries the interrogator code (II/SI) on top of the CRC, so a small syndrome is often not an error.
// ------------------------------------------------------------------------------------------------
constexpr int EC_HASH = 512;                                   // slots of the (s_j -> j) table: 107 keys, load 0.21
__device__ __forceinline__ unsigned ec_hash(uint32_t s) { return (s * 0x9E3779B1u) >> 23; }
__device__ __forceinline__ uint32_t ec_bit_syndrome(const unsigned int* s_crc, int i)   // a 112-bit frame's bit i
{
    return i < 88 ? s_crc[87 - i] : 1u << (111 - i);
}

// XOR the flips into f->data: each lane contributes the bits of its four MSB-first words of the packet (bit 31 of word
// k = bit 32k); they are OR-reduced over the warp.
__device__ __forceinline__ void ec_apply_flips(amb_frame* f, int lane, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3)
{
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        x0 |= __shfl_xor_sync(FULL, x0, d); x1 |= __shfl_xor_sync(FULL, x1, d);
        x2 |= __shfl_xor_sync(FULL, x2, d); x3 |= __shfl_xor_sync(FULL, x3, d);
    }
    if (lane < 14) {
        const uint32_t w = lane < 4 ? x0 : lane < 8 ? x1 : lane < 12 ? x2 : x3;
        f->data[lane] ^= (uint8_t)(w >> (24 - 8 * (lane & 3)));
    }
}
__device__ __forceinline__ void ec_word_bit(int pos, uint32_t& x0, uint32_t& x1, uint32_t& x2, uint32_t& x3)
{
    const uint32_t bit = 1u << (31 - (pos & 31));
    if ((pos >> 5) == 0) x0 |= bit; else if ((pos >> 5) == 1) x1 |= bit; else if ((pos >> 5) == 2) x2 |= bit; else x3 |= bit;
}

__global__ void __launch_bounds__(64) amb_ec_kernel(amb_frame* __restrict__ frames, unsigned int frame_cap, AmbCounters* ctr,
                                                    int n_host, int k_max, int m_any)
{
    __shared__ unsigned int s_crc[96];
    __shared__ unsigned int s_hash[EC_HASH];                   // (s_j << 8) | j, 0 = empty (no s_j is 0); m_any == 2 only
    for (int i = threadIdx.x; i < 96; i += blockDim.x) s_crc[i] = c_crc_rem[i];
    if (m_any > 1) for (int i = threadIdx.x; i < EC_HASH; i += blockDim.x) s_hash[i] = 0u;
    __syncthreads();
    if (m_any > 1 && threadIdx.x == 0) {                       // linear probing, once per CTA
        for (int j = 5; j < 112; j++) {
            const uint32_t s = ec_bit_syndrome(s_crc, j);
            unsigned h = ec_hash(s);
            while (s_hash[h]) h = (h + 1) & (EC_HASH - 1);
            s_hash[h] = (s << 8) | (unsigned)j;
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    unsigned int base = 0, n = (unsigned)n_host;
    if (ctr) {                                                 // this call's slots; those past the capacity were never written
        base = ctr->frame_base;
        n = base < frame_cap ? min(ctr->ndet_list, frame_cap - base) : 0u;
    }
    unsigned int nfixed = 0;
    const unsigned int nwarps = gridDim.x * (blockDim.x >> 5);
    for (unsigned int w0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32u; w0 < n; w0 += nwarps * 32u) {
        bool cand = false;
        if (w0 + lane < n) { const amb_frame* f = frames + base + w0 + lane; cand = !f->passed && f->crc != 0u; }
        unsigned int todo = __ballot_sync(FULL, cand);
        while (todo) {                                         // warp-uniform from here on
            amb_frame* f = frames + base + w0 + (__ffs(todo) - 1);
            todo &= todo - 1u;
            const uint32_t syn0 = f->crc;
            if (k_max > 0) {                                   // first phase: the low-confidence bits
                const unsigned nlow = f->numlowconf;
                unsigned status = AMB_EC_TOO_MANY;
                if (nlow <= (unsigned)k_max) {
                    const int nbits = f->nbits;
                    const int pos = lane < (int)nlow ? (int)f->lowconfbits[lane] : 0;
                    const bool in_l = pos >= 5;                // the DF field is never flipped
                    uint32_t v = 0u, m = in_l ? 1u << lane : 0u;
                    if (in_l) v = pos < nbits - 24 ? s_crc[nbits - 25 - pos] : 1u << (nbits - 1 - pos);
                    const int size_l = __popc(__ballot_sync(FULL, in_l));
                    uint32_t syn = syn0, sol = 0u;
                    bool pivot = false;
                    int rank = 0;
                    for (int b = 23; b >= 0; b--) {
                        const unsigned int rows = __ballot_sync(FULL, !pivot && ((v >> b) & 1u));
                        if (!rows) continue;
                        const int p = __ffs(rows) - 1;
                        const uint32_t pv = __shfl_sync(FULL, v, p), pm = __shfl_sync(FULL, m, p);
                        if (lane == p) pivot = true;
                        else if ((v >> b) & 1u) { v ^= pv; m ^= pm; }
                        if ((syn >> b) & 1u) { syn ^= pv; sol ^= pm; }
                        rank++;
                    }
                    status = syn ? AMB_EC_NO_SOLUTION : rank < size_l ? AMB_EC_AMBIGUOUS : AMB_EC_FIXED;
                    if (status == AMB_EC_FIXED) {
                        uint32_t x0 = 0u, x1 = 0u, x2 = 0u, x3 = 0u;
                        if ((sol >> lane) & 1u) ec_word_bit(pos, x0, x1, x2, x3);
                        ec_apply_flips(f, lane, x0, x1, x2, x3);
                        if (lane == 31) {
                            f->crc = 0u; f->passed = 1;
                            f->ec = AMB_EC_FIXED; f->ec_flips = (uint8_t)__popc(sol);
                        }
                        nfixed++;
                        continue;                              // a frame the first phase fixed is not tried again
                    }
                }
                if (lane == 0) f->ec = (uint8_t)status;
            }
            if (m_any <= 0 || f->df != 17) continue;
            // second phase: every pattern of at most m_any bits in 5..111
            int i1 = 0, j1 = 0;                                // this lane's fit: position(s), 0 = none
            int nfit = 0;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int i = 5 + lane + 32 * q;
                if (i >= 112) break;
                const uint32_t si = ec_bit_syndrome(s_crc, i);
                if (si == syn0) { i1 = i; j1 = 0; nfit++; }
                if (m_any > 1) {
                    const uint32_t want = syn0 ^ si;
                    for (unsigned h = ec_hash(want);; h = (h + 1) & (EC_HASH - 1)) {
                        const uint32_t e = s_hash[h];
                        if (!e) break;
                        if ((e >> 8) == want) {
                            if ((int)(e & 0xFFu) > i) { i1 = i; j1 = (int)(e & 0xFFu); nfit++; }
                            break;
                        }
                    }
                }
            }
            const unsigned fit_lanes = __ballot_sync(FULL, nfit > 0);
            if (__popc(fit_lanes) != 1 || __any_sync(FULL, nfit > 1)) {          // none, or (never seen) not unique
                if (lane == 0) AMB_FRAME_EC_ANY(f) = AMB_EC_NO_SOLUTION;
                continue;
            }
            uint32_t x0 = 0u, x1 = 0u, x2 = 0u, x3 = 0u;
            if (nfit) { ec_word_bit(i1, x0, x1, x2, x3); if (j1) ec_word_bit(j1, x0, x1, x2, x3); }
            ec_apply_flips(f, lane, x0, x1, x2, x3);
            if (lane == __ffs(fit_lanes) - 1) {
                f->crc = 0u; f->passed = 1;
                AMB_FRAME_EC_ANY(f) = AMB_EC_FIXED;
                AMB_FRAME_EC_ANY_BIT(f, 0) = (uint8_t)i1; AMB_FRAME_EC_ANY_BIT(f, 1) = (uint8_t)j1;
            }
            nfixed++;
        }
    }
    if (ctr && lane == 0 && nfixed) { atomicAdd(&ctr->npassed_call, nfixed); atomicAdd(&ctr->nec_fixed, nfixed); }
}

cudaError_t amb_launch_ec(amb_frame* frames, unsigned int frame_cap, AmbCounters* ctr, int n, int k_max, int m_any,
                          int sm_count, cudaStream_t s)
{
    if (!ctr && n <= 0) return cudaSuccess;
    AMB_LAUNCH((amb_ec_kernel), sm_count > 0 ? sm_count : 8, 64, 0, s, frames, frame_cap, ctr, n, k_max, m_any);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Address/parity check (option "ap_filter" = S seconds, off by default), after the error correction. The semantics are
// in include/airmodes_b200.h (AMB_FRAME_AP). Four launches per call, all on the slicer's stream:
//   amb_ap_count_kernel    classify the call's slots; count confirmers and subjects per bucket (a hash of the address)
//   amb_ap_scan_kernel     bucket offsets; re-zeroes the counts for the next call
//   amb_ap_scatter_kernel  classify again, append (sample index, address | kind, slot) to the bucket
//   amb_ap_resolve_kernel  per bucket: sort by (address, sample index) - in shared memory up to AMB_AP_TILE entries,
//                          in place in global memory beyond - then a max-scan over the confirmer positions gives each
//                          subject the latest earlier confirmer of its address in this call (same address = the same
//                          sorted run), else the table's latest confirmer of an earlier call. The last entry of each
//                          address run writes the table: one writer per address, no atomics.
// Every frame of a later call lies after every frame of an earlier one (DESIGN.md section 4), so "latest confirmer
// before this call" is all the table has to hold. Sample indices are unique per stream, so the sort key is a total order
// and the result does not depend on the order the scatter's atomics produced.
// ------------------------------------------------------------------------------------------------
constexpr unsigned AP_NONE = 0, AP_CONF = 1, AP_SUBJECT = 2, AP_IISI = 3;

__device__ __forceinline__ unsigned ap_classify(const amb_frame* f, unsigned& addr)
{
    const unsigned df = f->df;
    const unsigned crc = f->crc;
    const unsigned aa = ((unsigned)f->data[1] << 16) | ((unsigned)f->data[2] << 8) | f->data[3];
    if (f->passed) {
        if (df != 11 && df != 17) { addr = crc & 0xFFFFFFu; return AP_SUBJECT; }
        if (crc == 0u && f->ec != AMB_EC_FIXED && AMB_FRAME_EC_ANY(f) != AMB_EC_FIXED) { addr = aa; return AP_CONF; }
        return AP_NONE;
    }
    if (df == 11 && crc != 0u && crc < 0x80u) { addr = aa; return AP_IISI; }
    return AP_NONE;
}
__device__ __forceinline__ unsigned ap_bucket(unsigned addr) { return (addr * 0x9E3779B1u) >> (32 - AMB_AP_BUCKET_BITS); }
__device__ __forceinline__ void ap_call_slots(const AmbCounters* ctr, unsigned frame_cap, unsigned& base, unsigned& n)
{
    base = ctr->frame_base;                                    // slots past the capacity were never written
    n = base < frame_cap ? min(ctr->ndet_list, frame_cap - base) : 0u;
}

__global__ void __launch_bounds__(128) amb_ap_count_kernel(const amb_frame* __restrict__ frames, unsigned int frame_cap,
                                                          const AmbCounters* ctr, unsigned* __restrict__ count)
{
    unsigned base, n;
    ap_call_slots(ctr, frame_cap, base, n);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        unsigned addr = 0;
        if (ap_classify(frames + base + i, addr) != AP_NONE) atomicAdd(&count[ap_bucket(addr)], 1u);
    }
}

__global__ void __launch_bounds__(128) amb_ap_scan_kernel(unsigned* __restrict__ count, unsigned* __restrict__ off,
                                                         unsigned* __restrict__ cursor)
{
    constexpr unsigned PER = AMB_AP_BUCKETS / 128;
    __shared__ unsigned s_sum[128];
    const unsigned t = threadIdx.x;
    unsigned sum = 0;
    for (unsigned k = 0; k < PER; k++) sum += count[t * PER + k];
    s_sum[t] = sum;
    __syncthreads();
    for (unsigned d = 1; d < 128; d <<= 1) {                   // inclusive scan over the threads' sums
        const unsigned v = t >= d ? s_sum[t - d] : 0u;
        __syncthreads();
        s_sum[t] += v;
        __syncthreads();
    }
    unsigned run = s_sum[t] - sum;
    for (unsigned k = 0; k < PER; k++) {
        const unsigned c = count[t * PER + k];
        off[t * PER + k] = run; cursor[t * PER + k] = run; count[t * PER + k] = 0u;
        run += c;
    }
}

__global__ void __launch_bounds__(128) amb_ap_scatter_kernel(const amb_frame* __restrict__ frames, unsigned int frame_cap,
                                                            const AmbCounters* ctr, unsigned* __restrict__ cursor,
                                                            AmbApEntry* __restrict__ ent)
{
    unsigned base, n;
    ap_call_slots(ctr, frame_cap, base, n);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const amb_frame* f = frames + base + i;
        unsigned addr = 0;
        const unsigned kind = ap_classify(f, addr);
        if (kind == AP_NONE) continue;
        const unsigned pos = atomicAdd(&cursor[ap_bucket(addr)], 1u);
        AmbApEntry e; e.si = f->sample_index; e.key = addr | (kind << 24); e.slot = base + i;
        ent[pos] = e;
    }
}

__device__ __forceinline__ bool ap_less(const AmbApEntry& a, const AmbApEntry& b)
{
    const unsigned ka = a.key & 0xFFFFFFu, kb = b.key & 0xFFFFFFu;
    return ka != kb ? ka < kb : a.si < b.si;
}
// CTA-wide sort of e[0, n) by (address, sample index): a bitonic network in the form whose every compare-exchange puts
// the smaller element at the lower index (a flip stage, then half-cleaners), so the missing elements up to the next
// power of two act as +infinity at the end and their pairs are simply skipped. e may be shared or global memory.
__device__ void ap_sort(AmbApEntry* e, unsigned n)
{
    unsigned npad = 1;
    while (npad < n) npad <<= 1;
    for (unsigned k = 2; k <= npad; k <<= 1) {
        for (unsigned p = threadIdx.x; p < (npad >> 1); p += blockDim.x) {
            const unsigned h = k >> 1, b0 = (p / h) * k, o = p % h;
            const unsigned i = b0 + o, l = b0 + k - 1 - o;
            if (l < n && ap_less(e[l], e[i])) { const AmbApEntry x = e[i]; e[i] = e[l]; e[l] = x; }
        }
        __syncthreads();
        for (unsigned j = k >> 2; j > 0; j >>= 1) {
            for (unsigned p = threadIdx.x; p < (npad >> 1); p += blockDim.x) {
                const unsigned i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;
                if (l < n && ap_less(e[l], e[i])) { const AmbApEntry x = e[i]; e[i] = e[l]; e[l] = x; }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(128, 16) amb_ap_resolve_kernel(amb_frame* __restrict__ frames, AmbCounters* ctr,
                                                                 const unsigned* __restrict__ off,
                                                                 const unsigned* __restrict__ cursor, AmbApEntry* ent,
                                                                 unsigned long long* __restrict__ last,
                                                                 unsigned long long window)
{
    __shared__ AmbApEntry s_ent[AMB_AP_TILE];
    __shared__ int s_wmax[4];
    __shared__ unsigned s_delta;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_delta = 0u;
    __syncthreads();
    int delta = 0;                                           // change of the call's passed count
    for (unsigned b = blockIdx.x; b < AMB_AP_BUCKETS; b += gridDim.x) {
        const unsigned lo = off[b], n = cursor[b] - lo;
        if (n == 0u) continue;
        AmbApEntry* e = ent + lo;
        if (n <= AMB_AP_TILE) {
            for (unsigned t = threadIdx.x; t < n; t += blockDim.x) s_ent[t] = e[t];
            e = s_ent;
        }
        __syncthreads();
        ap_sort(e, n);
        int carry = -1;                                        // position of the latest confirmer before this chunk
        for (unsigned c0 = 0; c0 < n; c0 += AMB_AP_TILE) {
            const unsigned m = min(n - c0, (unsigned)AMB_AP_TILE);
            const unsigned q0 = 2 * threadIdx.x;               // this thread's two positions of the chunk
            const int v0 = q0 < m && (e[c0 + q0].key >> 24) == AP_CONF ? (int)(c0 + q0) : -1;
            const int v1 = max(v0, q0 + 1 < m && (e[c0 + q0 + 1].key >> 24) == AP_CONF ? (int)(c0 + q0 + 1) : -1);
            int x = v1;                                        // inclusive max-scan over the warp
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(FULL, x, d); if ((int)lane >= d) x = max(x, y); }
            const int xprev = __shfl_up_sync(FULL, x, 1);
            if (lane == 31) s_wmax[warp] = x;
            __syncthreads();
            int pre = carry;
            for (unsigned w = 0; w < warp; w++) pre = max(pre, s_wmax[w]);
            if (lane > 0) pre = max(pre, xprev);
            const int incl[2] = {max(pre, v0), max(pre, v1)};  // latest confirmer at or before each position
#pragma unroll
            for (int r = 0; r < 2; r++) {                      // subjects decide (before any table write of this chunk)
                const unsigned q = q0 + r;
                if (q >= m) break;
                const AmbApEntry en = e[c0 + q];
                const unsigned kind = en.key >> 24, addr = en.key & 0xFFFFFFu;
                if (kind == AP_CONF) continue;
                const int p = incl[r];
                const unsigned long long g1 = p >= 0 && (e[p].key & 0xFFFFFFu) == addr ? e[p].si + 1ull : last[addr];
                const bool known = g1 != 0ull && en.si + 1ull - g1 <= window;
                amb_frame* f = frames + en.slot;
                AMB_FRAME_AP(f) = known ? AMB_AP_KNOWN : AMB_AP_UNKNOWN;
                if (kind == AP_SUBJECT && !known) { f->passed = 0; delta--; }
                if (kind == AP_IISI && known) { f->passed = 1; delta++; }
            }
            __syncthreads();
#pragma unroll
            for (int r = 0; r < 2; r++) {                      // the last entry of each address run writes the table
                const unsigned q = q0 + r;
                if (q >= m) break;
                const unsigned addr = e[c0 + q].key & 0xFFFFFFu;
                const bool run_end = c0 + q + 1 == n || (e[c0 + q + 1].key & 0xFFFFFFu) != addr;
                const int p = incl[r];
                if (run_end && p >= 0 && (e[p].key & 0xFFFFFFu) == addr) last[addr] = e[p].si + 1ull;
            }
            for (unsigned w = 0; w < 4; w++) carry = max(carry, s_wmax[w]);
            __syncthreads();
        }
    }
    if (delta) atomicAdd(&s_delta, (unsigned)delta);
    __syncthreads();
    if (threadIdx.x == 0 && s_delta) atomicAdd(&ctr->npassed_call, s_delta);
}

int amb_launch_ap(amb_frame* frames, unsigned int frame_cap, AmbCounters* ctr, const AmbApState& ap,
                  unsigned long long window, int sm_count, cudaStream_t s, cudaError_t* err)
{
    const int g = sm_count > 0 ? sm_count : 8;
    AMB_LAUNCH((amb_ap_count_kernel), g, 128, 0, s, frames, frame_cap, ctr, ap.count);
    AMB_LAUNCH((amb_ap_scan_kernel), 1, 128, 0, s, ap.count, ap.off, ap.cursor);
    AMB_LAUNCH((amb_ap_scatter_kernel), g, 128, 0, s, frames, frame_cap, ctr, ap.cursor, ap.ent);
    AMB_LAUNCH((amb_ap_resolve_kernel), min(AMB_AP_BUCKETS, 4 * g), 128, 0, s, frames, ctr, ap.off, ap.cursor, ap.ent,
               ap.last, window);
    *err = cudaGetLastError();
    return 4;
}

// device CRC parity hook: same XOR fold as the slicer
__global__ void amb_crc_kernel(const uint8_t* __restrict__ data, int n, int length, uint32_t* out)
{
    const int lane = threadIdx.x & 31;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n) return;
    const int nmsg = length * 8;
    uint32_t crc = 0;
    for (int j = lane; j < nmsg; j += 32)
        if ((data[(size_t)w * length + (j >> 3)] >> (7 - (j & 7))) & 1) crc ^= c_crc_rem[nmsg - 1 - j];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) crc ^= __shfl_xor_sync(FULL, crc, d);
    if (lane == 0) out[w] = crc;
}
cudaError_t amb_launch_crc(const uint8_t* data, int n, int length, uint32_t* out, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    AMB_LAUNCH((amb_crc_kernel), (n + 3) / 4, 128, 0, s, data, n, length, out);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// carry: keep the last kc samples of (carry ++ new data) for the next call
// ------------------------------------------------------------------------------------------------
__global__ void amb_carry_kernel(const AmbSegs S, float2* __restrict__ dst, int kc)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kc) return;
    dst[i] = *seg_ptr(S, S.n_valid - kc + i);
}
cudaError_t amb_launch_carry(const AmbSegs& S, float2* dst, int kc, cudaStream_t s)
{
    AMB_LAUNCH((amb_carry_kernel), (kc + 255) / 256, 256, 0, s, S, dst, kc);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// 16-bit IQ ingest: the receivers behind gr-air-modes deliver 16-bit samples on the wire and the host widens them
// to gr_complex (radio.py:163-173 asks UHD for cpu_format="fc32"). Shipping the 16-bit samples and widening them
// here halves the PCIe traffic; x * 2^-15 is exact in float32, so the chain sees the very floats the host-side
// conversion would have produced.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) amb_widen_sc16_kernel(const short2* __restrict__ in, float2* __restrict__ out, long long n)
{
    const float k = 1.0f / 32768.0f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const short2 v = in[i];
        out[i] = make_float2(__fmul_rn((float)v.x, k), __fmul_rn((float)v.y, k));
    }
}
cudaError_t amb_launch_widen_sc16(const void* in, float2* out, long long n, int sm_count, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    long long blocks = (n + 255) / 256;
    if (blocks > (long long)sm_count * 16) blocks = (long long)sm_count * 16;
    AMB_LAUNCH((amb_widen_sc16_kernel), (unsigned)blocks, 256, 0, s, reinterpret_cast<const short2*>(in), out, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// prologue: everything that has to be reset / staged before the scan of one call, in one launch
// ------------------------------------------------------------------------------------------------
__global__ void amb_prologue_kernel(float2* __restrict__ tail, int tail_cap, const float2* __restrict__ src_rem, int n_rem,
                                    uint32_t* group_count, int n_groups)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int stride = gridDim.x * blockDim.x;
    for (int k = i; k < tail_cap; k += stride) tail[k] = k < n_rem ? src_rem[k] : make_float2(0.f, 0.f);
    for (int k = i; k < n_groups; k += stride) group_count[k] = 0;
}
cudaError_t amb_launch_prologue(float2* tail, int tail_cap, const float2* src_rem, int n_rem,
                                uint32_t* group_count, int n_groups, cudaStream_t s)
{
    AMB_LAUNCH((amb_prologue_kernel), 8, 256, 0, s, tail, tail_cap, src_rem, n_rem, group_count, n_groups);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// split-form preamble block: the two float streams are given; the first four tests (:173-179) are evaluated
// exactly per item and written in the same (coarse, fine) bitmap format the scan kernel produces.
// Indices are reported coordinates (item + history-1). coarse / span_count / group_count are pre-zeroed.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) amb_stream_cand_kernel(const __grid_constant__ AmbScanArgs a, const float* __restrict__ in0,
                                                              const float* __restrict__ in1, long long n)
{
    const AmbParams& P = a.P;
    const long long nwords = ((long long)a.row_hi * AMB_ROW) / 32;
    const int lane = threadIdx.x & 31;
    for (long long w = (long long)(blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < nwords; w += (long long)(gridDim.x * blockDim.x) >> 5) {
        const long long r = w * 32 + lane;
        bool c = false;
        if (r >= a.j_lo && r < a.j_hi) {
            const float x = stream_at(in0, n, P.H, r);
            const float thr = __fmul_rn(stream_at(in1, n, P.H, r), P.thr);                 // :173
            c = x > thr;                                                                    // :174
            if (c && (stream_at(in0, n, P.H, r + 1) > x)) c = false;                        // :175
            if (c && (stream_at(in0, n, P.H, r + P.po1) < thr)) c = false;                  // :177
            if (c && (stream_at(in0, n, P.H, r + P.po2) < thr)) c = false;                  // :178
            if (c && (stream_at(in0, n, P.H, r + P.po3) < thr)) c = false;                  // :179
        }
        const uint32_t word = __ballot_sync(FULL, c);
        if (lane == 0) {
            a.fine[w] = word;                                   // row = w / 8, word q = w % 8
            if (word) {
                const int row = (int)(w >> 3);
                atomicOr(&a.coarse[row >> 5], 1u << (row & 31));
                const int span = row / a.rows_per_span;
                atomicAdd(&a.span_count[span], (unsigned)__popc(word));
                atomicAdd(&a.group_count[span >> 6], (unsigned)__popc(word));
            }
        }
    }
}
cudaError_t amb_launch_stream_candidates(const AmbScanArgs& a, const float* in0, const float* in1, long long n, int sm_count,
                                         cudaStream_t s)
{
    AMB_LAUNCH((amb_stream_cand_kernel), 4 * sm_count, 256, 0, s, a, in0, in1, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// optional DC blocker in front of the demodulator: filter.dc_blocker_cc(100*spc, False) (rx_path.py:39-41).
// GNU Radio's short form is  out[n] = x[n-D+1] - MA_D(MA_D(x))[n]  with complex fp32 moving averages. Canonical
// arithmetic (same as the CPU checker): every window sum in fp64, ascending, per component, rounded once to
// fp32 and divided by (float)D. This stage is off by default (radio.py:118-119).
//
// A tile of DC_T outputs needs W = DC_T + D - 1 source elements. If, per component, the largest magnitude and the
// smallest non-zero quantum of the tile are at most `lim` = 29 - ceil(log2 W) binades apart, every sum of up to W of
// these fp32 values is a multiple of that quantum below 2^53 quanta, i.e. exactly representable in fp64: the
// reference order's partial sums never round, and neither do the tile's prefix sums nor their differences. The
// window sums are then P[t+D] - P[t] (O(1) per output, bit-identical). Tiles that fail the test (a strong burst
// next to a near-zero sample, NaN/Inf) take the brute-force path, which keeps the summation order literally.
// `raw` is the logical stream rawcarry(2D-2 samples) ++ new samples, addressed through two pointers.
// ------------------------------------------------------------------------------------------------
#define DC_T 1024
__device__ __forceinline__ float2 dc_raw(const float2* carry, int nc, const float2* fresh, long long r)
{
    return r < nc ? carry[r] : fresh[r - nc];
}
__device__ __forceinline__ double shfl_up_f64(double v, int d)
{
    return __hiloint2double(__shfl_up_sync(0xffffffffu, __double2hiint(v), d), __shfl_up_sync(0xffffffffu, __double2loint(v), d));
}

// ONE pass (round 2): a CTA produces DC_T outputs from W2 = DC_T + 2D - 2 raw samples held in shared memory:
//   raw (W2)  --MA_D-->  ma0 (W1 = DC_T + D - 1)  --MA_D-->  m1 (DC_T);   out[t] = raw[t + D - 1] - m1[t]
// Each moving average is evaluated as P[i+D] - P[i] from a block-wide fp64 prefix sum when the exactness test above
// holds for its input (raw for the first, ma0 for the second), else literally. Traffic: 8 B read + 8 B written per
// sample (the two-pass version moved 40 B: x, ma0 out, ma0 in, x again, out); the 2D-2 halo re-reads hit L2.
// CH = elements per thread in the prefix phase, ceil(W2 / 256) rounded up to an ODD number: a thread's chunk is
// contiguous, so with an odd CH the 8-byte source reads and the 16-byte prefix writes of a warp are bank-conflict free.
struct DcRange { unsigned mxr, mnr, mxi, mni; };          // largest |bits|, smallest non-zero |bits| - 1, per component
__device__ __forceinline__ void dc_range_add(DcRange& g, float2 v)
{
    const unsigned int ux = __float_as_uint(v.x) & 0x7fffffffu, uy = __float_as_uint(v.y) & 0x7fffffffu;
    g.mxr = max(g.mxr, ux); g.mnr = min(g.mnr, ux - 1u);     // zero wraps to 0xffffffff and drops out of the minimum
    g.mxi = max(g.mxi, uy); g.mni = min(g.mni, uy - 1u);
}
// block-wide verdict: every sum of these values is exact in fp64 (see above). s_rng: 8 x 4 words of scratch.
__device__ __forceinline__ bool dc_range_exact(DcRange g, unsigned int (*s_rng)[4], int lim)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    g.mxr = __reduce_max_sync(0xffffffffu, g.mxr); g.mnr = __reduce_min_sync(0xffffffffu, g.mnr);
    g.mxi = __reduce_max_sync(0xffffffffu, g.mxi); g.mni = __reduce_min_sync(0xffffffffu, g.mni);
    __syncthreads();                                         // previous users of s_rng are done
    if (lane == 0) { s_rng[warp][0] = g.mxr; s_rng[warp][1] = g.mnr; s_rng[warp][2] = g.mxi; s_rng[warp][3] = g.mni; }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < 8; w++) { g.mxr = max(g.mxr, s_rng[w][0]); g.mnr = min(g.mnr, s_rng[w][1]); g.mxi = max(g.mxi, s_rng[w][2]); g.mni = min(g.mni, s_rng[w][3]); }
    // exponent fields; denormals share the quantum of exponent field 1
    const int er1 = (int)max(g.mxr >> 23, 1u), er0 = (int)max((g.mnr + 1u) >> 23, 1u);
    const int ei1 = (int)max(g.mxi >> 23, 1u), ei0 = (int)max((g.mni + 1u) >> 23, 1u);
    return (g.mxr == 0 || (er1 < 255 && er1 - er0 <= lim)) && (g.mxi == 0 || (ei1 < 255 && ei1 - ei0 <= lim));
}
// block-wide inclusive fp64 prefix sums of v[0 .. W) into P[1 .. W], P[0] = 0 (every addition exact: association is free)
template <int CH>
__device__ __forceinline__ void dc_prefix(const float2* v, int W, double2* P, double2* s_tot)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k0 = tid * CH;
    double xr[CH], xi[CH];
    double sr = 0.0, si = 0.0;
#pragma unroll
    for (int j = 0; j < CH; j++) {
        const float2 e = (k0 + j < W) ? v[k0 + j] : make_float2(0.f, 0.f);
        xr[j] = (double)e.x; xi[j] = (double)e.y;
        sr += xr[j]; si += xi[j];
    }
    double ar = sr, ai = si;                              // inclusive scan of the per-thread totals within the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double tr = shfl_up_f64(ar, d), ti = shfl_up_f64(ai, d);
        if (lane >= d) { ar += tr; ai += ti; }
    }
    __syncthreads();                                      // previous users of s_tot / P are done
    if (lane == 31) s_tot[warp] = make_double2(ar, ai);
    __syncthreads();
    double offr = ar - sr, offi = ai - si;                // exclusive offset of this thread
#pragma unroll
    for (int w = 0; w < 7; w++) if (w < warp) { offr += s_tot[w].x; offi += s_tot[w].y; }
    if (tid == 0) P[0] = make_double2(0.0, 0.0);
#pragma unroll
    for (int j = 0; j < CH; j++) {
        offr += xr[j]; offi += xi[j];
        if (k0 + j < W) P[k0 + j + 1] = make_double2(offr, offi);
    }
    __syncthreads();
}

// TILE = outputs per CTA: 1024 for D <= 256, 2048 beyond (the 2D-2 halo is recomputed by every tile).
template <int CH, int TILE>
__global__ void __launch_bounds__(256) amb_dcblock_kernel(const float2* __restrict__ carry, int nc, const float2* __restrict__ fresh,
                                                          float2* __restrict__ dst, long long n_out, int D, int lim1, int lim2)
{
    AMB_DYN_SMEM(unsigned char, dc_smem, 16);
    const int W1 = TILE + D - 1, W2 = TILE + 2 * D - 2;
    float2* src = reinterpret_cast<float2*>(dc_smem);                                               // W2 raw samples
    float2* ma0 = src + ((W2 + 1) & ~1);                                                            // W1 first averages
    double2* P = reinterpret_cast<double2*>(ma0 + ((W1 + 1) & ~1));                                 // W2 + 1 prefix sums (re, im)
    __shared__ unsigned int s_rng[8][4];
    __shared__ double2 s_tot[8];
    const long long base = (long long)blockIdx.x * TILE;          // first output of the tile = raw index base
    const int tid = threadIdx.x;
    const long long raw_end = (long long)nc + n_out;              // raw = carry ++ fresh
    const float fD = (float)D;
    // ---- raw samples of the tile (interior tiles: one contiguous run of `fresh`)
    DcRange g = {0u, ~0u, 0u, ~0u};
    const float2* run = (base >= nc && base + W2 <= raw_end) ? fresh + (base - nc) : nullptr;
    for (int i = tid; i < W2; i += 256) {
        float2 v = make_float2(0.f, 0.f);
        if (run) v = run[i];
        else { const long long q = base + i; if (q < raw_end) v = dc_raw(carry, nc, fresh, q); }
        src[i] = v;
        dc_range_add(g, v);
    }
    const bool exact1 = dc_range_exact(g, s_rng, lim2);           // also orders the src[] stores before their readers
    // ---- first moving average: ma0[i] covers raw[base+i .. base+i+D-1]
    if (exact1) dc_prefix<CH>(src, W2, P, s_tot);
    g = {0u, ~0u, 0u, ~0u};
    for (int i = tid; i < W1; i += 256) {
        double ar = 0.0, ai = 0.0;
        if (exact1) { const double2 hi = P[i + D], lo = P[i]; ar = hi.x - lo.x; ai = hi.y - lo.y; }
        else for (int k = 0; k < D; k++) { ar += (double)src[i + k].x; ai += (double)src[i + k].y; }
        const float2 m = make_float2(__fdiv_rn((float)ar, fD), __fdiv_rn((float)ai, fD));
        ma0[i] = m;
        dc_range_add(g, m);
    }
    const bool exact2 = dc_range_exact(g, s_rng, lim1);           // (its barriers also retire the readers of P)
    // ---- second moving average and the output
    if (exact2) dc_prefix<CH>(ma0, W1, P, s_tot);
#pragma unroll
    for (int u = 0; u < TILE / 256; u++) {
        const int t = tid + 256 * u;
        const long long m = base + t;
        if (m >= n_out) break;
        double ar = 0.0, ai = 0.0;
        if (exact2) { const double2 hi = P[t + D], lo = P[t]; ar = hi.x - lo.x; ai = hi.y - lo.y; }
        else for (int k = 0; k < D; k++) { ar += (double)ma0[t + k].x; ai += (double)ma0[t + k].y; }
        const float mr = __fdiv_rn((float)ar, fD), mi = __fdiv_rn((float)ai, fD);
        const float2 d = src[t + D - 1];                              // x[n-D+1]: raw index of new sample m is nc + m = base + t + 2D-2 ... - (D-1)
        dst[m] = make_float2(__fsub_rn(d.x, mr), __fsub_rn(d.y, mi));
    }
}

template <int CH, int TILE>
static cudaError_t launch_dcblock_t(const float2* rawcarry, int nc, const float2* fresh, long long n_new, int D, int lim1, int lim2,
                                    size_t smem, float2* out, cudaStream_t s)
{
    // per device, like the scan kernel: set on every launch (a host-side table write)
    cudaError_t e = cudaFuncSetAttribute(amb_dcblock_kernel<CH, TILE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(amb_dcblock_kernel<CH, TILE>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (e != cudaSuccess) return e;
    AMB_LAUNCH((amb_dcblock_kernel<CH, TILE>), (unsigned)((n_new + TILE - 1) / TILE), 256, smem, s, rawcarry, nc, fresh, out, n_new, D, lim1, lim2);
    return cudaGetLastError();
}

static int dc_lim(int W)
{
    int c = 0;
    while ((1 << c) < W) c++;
    return 29 - c;                                       // see the exactness argument above
}

cudaError_t amb_launch_dcblock(const float2* rawcarry, int nc, const float2* fresh, long long n_new, int D,
                               float2* ma0_tmp, float2* out, float2* rawcarry_next, cudaStream_t s)
{
    (void)ma0_tmp;                                       // the two-pass version's intermediate: not needed any more
    const int T = D <= 256 ? 1024 : 2048;
    const int W1 = T + D - 1, W2 = T + 2 * D - 2;
    const size_t smem = (size_t)(((W2 + 1) & ~1) + ((W1 + 1) & ~1)) * sizeof(float2) + (size_t)(W2 + 1) * sizeof(double2);
    if (smem > 200 * 1024 || W2 > 17 * 256) return cudaErrorInvalidValue;
    if (n_new > 0) {
        cudaError_t e;
        const int l1 = dc_lim(W1), l2 = dc_lim(W2);
        if (T == 1024) {
            if (W2 <= 5 * 256) e = launch_dcblock_t<5, 1024>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
            else e = launch_dcblock_t<7, 1024>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
        } else {
            if (W2 <= 11 * 256) e = launch_dcblock_t<11, 2048>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
            else if (W2 <= 13 * 256) e = launch_dcblock_t<13, 2048>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
            else if (W2 <= 15 * 256) e = launch_dcblock_t<15, 2048>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
            else e = launch_dcblock_t<17, 2048>(rawcarry, nc, fresh, n_new, D, l1, l2, smem, out, s);
        }
        if (e != cudaSuccess) return e;
    }
    // next raw carry = last nc samples of rawcarry ++ fresh
    AmbSegs S; S.carry = rawcarry; S.main_ = fresh; S.tail = fresh; S.n_carry = nc; S.n_main = (int)n_new; S.n_tail = 0;
    S.n_valid = nc + (int)n_new;
    return amb_launch_carry(S, rawcarry_next, nc, s);
}

// Every kernel of the library asks for the same L1 / shared-memory split (all shared). An SM's split is only changed
// while the SM is idle, so a kernel that prefers another split than the one the resident scan CTAs run with is NOT
// co-scheduled with them - it waits for the scan to drain. With one common preference the sparse kernels of call k
// really do run under the scan of call k+1.
template <class K> static cudaError_t prefer_shared(K kernel)
{
    return cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}
template <int SPC> static cudaError_t prefer_shared_spc()
{
    cudaError_t e = prefer_shared(amb_exact_warp_kernel<SPC>);
    if (e == cudaSuccess) e = prefer_shared(amb_exact_kernel<SPC, true>);
    if (e == cudaSuccess) e = prefer_shared(amb_exact_kernel<SPC, false>);
    return e;
}
cudaError_t amb_prefer_max_shared()
{
    cudaError_t e = prefer_shared(amb_compact_kernel);
    if (e == cudaSuccess) e = prefer_shared_spc<0>();
    if (e == cudaSuccess) e = prefer_shared_spc<1>();
    if (e == cudaSuccess) e = prefer_shared_spc<2>();
    if (e == cudaSuccess) e = prefer_shared_spc<5>();
    if (e == cudaSuccess) e = prefer_shared_spc<10>();
    if (e == cudaSuccess) e = prefer_shared(amb_exact_streams_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_seq_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_par1_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_par2_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_finalize_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_reset_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_walk_summary_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_set_state_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_pack_summary_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_compose_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_set_state_dev_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_slice_kernel<true, 0, false>);
    if (e == cudaSuccess) e = prefer_shared(amb_slice_chips_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_ec_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_carry_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_prologue_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_widen_sc16_kernel);
    if (e == cudaSuccess) e = prefer_shared(amb_stream_cand_kernel);
    return e;
}

cudaError_t amb_upload_tables(const int*)
{
    unsigned int rem[96];                               // rate independent: safe to share between contexts
    unsigned int r = 0xFFF409u;                         // x^24 mod G
    for (int t = 0; t < 96; t++) {
        rem[t] = r;
        r = (r & 0x800000u) ? (((r << 1) ^ 0xFFF409u) & 0xFFFFFFu) : ((r << 1) & 0xFFFFFFu);
    }
    return cudaMemcpyToSymbol(c_crc_rem, rem, sizeof(rem));
}

// ------------------------------------------------------------------------------------------------
// Mode A/C replies (option "modeac")
// ------------------------------------------------------------------------------------------------
#include "amb_modeac.cuh"
