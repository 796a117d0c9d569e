// TEST HARNESS (not a product path): the hot path's sparse kernels and their launchers - gr_air_modes_b200/csrc/
// amb_kernels.cu minus the TMA scan kernel (PTX), i.e. candidate bitmap from float streams, compaction, exact preamble
// tests, the sequential and the parallel resolver, the slicer with its CRC - compiled for the host under
// tests/simt/simt_emul.h and driven like amb_preamble_process / amb_slicer_process / amb_device_crc drive them
// (amb_api.cu). tests/test_kernels_simt.py compares the results with the oracle. Built by the test with plain g++.
#include "simt_emul.h"

#include "../../gr_air_modes_b200/csrc/amb_kernels.cu"
#include "../../gr_air_modes_b200/csrc/amb_params.h"

#include <algorithm>
#include <vector>

// One whole stream (first call, flush): amb_preamble_process with sf_total = 0. resolver: 1 sequential, else parallel.
// Returns the number of detections (<= max_det), < 0 on error; chips_out[240 * k], index_out[k] in stream order.
extern "C" int emul_preamble(const float* in0, const float* in1, int n, float rate, float threshold_db, int resolver,
                             int sm_count, float* chips_out, unsigned long long* index_out, int max_det,
                             unsigned* n_candidates)
{
    AmbParams P; int off[240];
    if (compute_params(rate, threshold_db, 0, &P, off) != AMB_OK) return -100;
    if (amb_upload_tables(off) != cudaSuccess) return -101;
    const size_t m = (size_t)n;
    const long long ntot = (long long)n + P.H;
    std::vector<float> d0(m + 1, 0.f), d1(m + 1, 0.f);
    std::copy(in0, in0 + n, d0.begin());
    std::copy(in1, in1 + n, d1.begin());
    AmbScanArgs a{};
    a.P = P; a.j_lo = 0; a.j_hi = (int)ntot; a.row_lo = 0; a.row_hi = (int)((a.j_hi + AMB_ROW - 1) / AMB_ROW);
    const int rows = a.row_hi;
    const int target = sm_count * 16;
    int rps = ((rows + target - 1) / target + AMB_SPAN_ROWS_ALIGN - 1) / AMB_SPAN_ROWS_ALIGN * AMB_SPAN_ROWS_ALIGN;
    if (rps < AMB_SPAN_ROWS_ALIGN) rps = AMB_SPAN_ROWS_ALIGN;
    a.rows_per_span = rps; a.n_spans = std::max(1, (rows + rps - 1) / rps);
    // buffers as ensure_call_buffers sizes them
    const size_t rows_cap = (size_t)a.row_hi + 64 + ((size_t)a.row_hi + 64) / 8;
    const int spans_cap = a.n_spans + 64;
    const unsigned cand_cap = (unsigned)std::max<long long>(1 << 16, (long long)m + P.H + 1024);   // cand_capacity() of amb_api.cu
    const unsigned frame_cap = (unsigned)((long long)m / std::max(P.skip0, 1) + 2) * 2 + 1024;
    std::vector<uint32_t> coarse(rows_cap / 32 + 2, 0), fine(rows_cap * 8, 0), span_count((size_t)spans_cap + 128, 0);
    std::vector<int> cand_j(cand_cap), det_list(cand_cap);
    std::vector<uint32_t> cand_info(cand_cap);
    std::vector<float> cand_avg(cand_cap);
    const long long n_samples = (long long)m + P.H + 4096;
    std::vector<unsigned char> walk_scratch(amb_walk_scratch_bytes(cand_cap, (long long)cand_cap * 8 + 4096), 0);
    std::vector<amb_frame> frames(frame_cap);
    std::vector<float> chips((size_t)frame_cap * 240);
    AmbCounters ctr{}; AmbWalkState st{};
    a.coarse = coarse.data(); a.fine = fine.data(); a.span_count = span_count.data();
    a.group_count = span_count.data() + spans_cap;
    cudaStream_t s = nullptr;
    if (amb_launch_stream_candidates(a, d0.data(), d1.data(), (long long)m, sm_count, s) != cudaSuccess) return -1;
    const bool par = resolver != 1;
    if (amb_launch_compact(a, cand_j.data(), cand_cap, &ctr, par ? walk_scratch.data() : nullptr, n_samples, s) != cudaSuccess) return -2;
    AmbExactArgs ea{};
    ea.P = P; ea.cand_j = cand_j.data(); ea.cand_info = cand_info.data(); ea.cand_avg = cand_avg.data(); ea.ctr = &ctr;
    ea.in0 = d0.data(); ea.in1 = d1.data(); ea.n_streams = (long long)m;
    if (amb_launch_exact(ea, sm_count, s) != cudaSuccess) return -3;
    AmbWalkArgs wa{};
    wa.P = P; wa.org = 0; wa.ntot = ntot; wa.r_safe = 0; wa.flush = 1; wa.ctr = &ctr; wa.st = &st;
    wa.cand_j = cand_j.data(); wa.cand_info = cand_info.data(); wa.det_list = det_list.data();
    if ((par ? amb_launch_walk_par(wa, walk_scratch.data(), cand_cap, n_samples, s) : amb_launch_walk_seq(wa, s)) != cudaSuccess) return -4;
    AmbSliceArgs sl{};
    sl.P = P; sl.cand_j = cand_j.data(); sl.cand_info = cand_info.data(); sl.cand_avg = cand_avg.data(); sl.ctr = &ctr;
    sl.det_list = det_list.data();
    sl.frames = frames.data(); sl.frame_cap = frame_cap; sl.chips_out = chips.data(); sl.org = 0;
    sl.in0 = d0.data(); sl.in1 = d1.data(); sl.n_streams = (long long)m;
    if (amb_launch_slice(sl, sm_count, s) != cudaSuccess) return -5;
    if (ctr.overflow || ctr.frame_overflow) return -6;
    if (n_candidates) { n_candidates[0] = ctr.ncand; n_candidates[1] = ctr.nreal_call; n_candidates[2] = (unsigned)st.fallback; }
    const unsigned nd = ctr.nframes;
    std::vector<unsigned> order(nd);
    for (unsigned k = 0; k < nd; k++) order[k] = k;
    std::sort(order.begin(), order.end(), [&](unsigned x, unsigned y) { return frames[x].sample_index < frames[y].sample_index; });
    if (nd > (unsigned)max_det) return -7;
    for (unsigned k = 0; k < nd; k++) {
        index_out[k] = frames[order[k]].sample_index;
        memcpy(chips_out + (size_t)k * 240, chips.data() + (size_t)order[k] * 240, 240 * sizeof(float));
    }
    return (int)nd;
}

static unsigned emul_last_counts[3];
extern "C" void emul_counts(unsigned* out) { memcpy(out, emul_last_counts, sizeof emul_last_counts); }

// The fused path on IQ (amb_process, one call over a whole stream, flush): the exact and slice kernels in their IQ form
// recompute |x|^2, the pulse matched filter and the noise-floor window from the samples (canonical arithmetic) through
// the carry ++ main ++ tail segment view, the prologue kernel stages the tail. The TMA scan kernel cannot run here; its
// output - the candidate bitmap in segment coordinates - is produced by the stream-candidate kernel from the (bb, avg)
// streams the caller computed with the canonical front end, shifted into the same coordinates. With bb == NULL the
// scan kernel itself runs: its PTX helpers (mbarrier, 2-D TMA tile copy with the 128-byte swizzle) are emulated.
// Returns detections in stream order: index_out, chips_out (240 each), frames_out (unstamped).
extern "C" int emul_process_iq(const float* iq, int n, const float* bb, const float* avg, float rate, float threshold_db,
                               int use_pmf, int resolver, int sm_count, float* chips_out, unsigned long long* index_out,
                               amb_frame* frames_out, int max_det)
{
    AmbParams P; int off[240];
    if (compute_params(rate, threshold_db, use_pmf, &P, off) != AMB_OK) return -100;
    if (amb_upload_tables(off) != cudaSuccess) return -101;
    const int guard = P.maxlate + (int)ceilf(P.skip_f) + 4;                       // setup_rate (amb_api.cu)
    const int kc = (guard + P.L + 2 * P.spc_i + 64 + AMB_STAGE - 1) / AMB_STAGE * AMB_STAGE;
    const int tail_cap = 4 * AMB_STAGE;
    const int n_main = n & ~(AMB_STAGE - 1), n_tv = n - n_main;
    const int n_tail = (n_tv + 512 + AMB_STAGE - 1) / AMB_STAGE * AMB_STAGE;
    std::vector<float2> carry(kc, make_float2(0.f, 0.f)), tail(tail_cap), src(n > 0 ? n : 1);
    memcpy(src.data(), iq, (size_t)n * sizeof(float2));
    AmbSegs S;
    S.carry = carry.data(); S.main_ = src.data(); S.tail = tail.data();
    S.n_carry = kc; S.n_main = n_main; S.n_tail = n_tail; S.n_valid = kc + n;
    const long long org = -(long long)kc + P.H;
    const long long ntot = (long long)n + P.H;
    const long long j_lo = 0 - org, j_hi = S.n_valid;
    AmbScanArgs a{};
    a.P = P; a.S = S; a.j_lo = (int)j_lo; a.j_hi = (int)j_hi;
    a.row_lo = (int)(j_lo / AMB_ROW) & ~(AMB_SPAN_ROWS_ALIGN - 1);
    a.row_hi = (int)((j_hi + AMB_ROW - 1) / AMB_ROW);
    if (a.row_lo != 0) return -102;
    const int rows = a.row_hi - a.row_lo;
    const int target = sm_count * 16;
    int rps = (rows + target - 1) / target;
    rps = (rps + AMB_SPAN_ROWS_ALIGN - 1) / AMB_SPAN_ROWS_ALIGN * AMB_SPAN_ROWS_ALIGN;
    if (rps < AMB_SPAN_ROWS_ALIGN) rps = AMB_SPAN_ROWS_ALIGN;
    a.rows_per_span = rps; a.n_spans = (rows + rps - 1) / rps;
    const size_t rows_cap = (size_t)a.row_hi + 64 + ((size_t)a.row_hi + 64) / 8;
    const int spans_cap = a.n_spans + 64;
    const unsigned cand_cap = (unsigned)std::max<long long>(1 << 16, (j_hi - j_lo) + 1024);      // cand_capacity() of amb_api.cu
    const unsigned frame_cap = (unsigned)((j_hi - j_lo) / std::max(P.skip0, 1) + 2) * 2 + 1024;
    std::vector<uint32_t> coarse(rows_cap / 32 + 2, 0), fine(rows_cap * 8, 0), span_count((size_t)spans_cap + 128, 0);
    std::vector<int> cand_j(cand_cap), det_list(cand_cap);
    std::vector<uint32_t> cand_info(cand_cap);
    std::vector<float> cand_avg(cand_cap);
    const long long n_samples = (long long)S.n_carry + S.n_main + S.n_tail;
    std::vector<unsigned char> walk_scratch(amb_walk_scratch_bytes(cand_cap, (long long)cand_cap * 8 + 4096), 0);
    std::vector<amb_frame> frames(frame_cap);
    std::vector<float> chips((size_t)frame_cap * 240);
    AmbCounters ctr{}; AmbWalkState st{};
    a.coarse = coarse.data(); a.fine = fine.data(); a.span_count = span_count.data();
    a.group_count = span_count.data() + spans_cap;
    cudaStream_t s = nullptr;
    if (amb_launch_prologue(tail.data(), tail_cap, src.data() + n_main, n_tv, a.group_count, 128, s) != cudaSuccess) return -1;
    if (!bb) {      // the real scan kernel: TMA tiles and mbarriers are emulated (simt_emul.h), the kernel source is the product's
        simt_make_tmap(&a.tm_carry, carry.data(), (size_t)kc);
        simt_make_tmap(&a.tm_tail, tail.data(), (size_t)tail_cap);
        if (n_main) simt_make_tmap(&a.tm_main, src.data(), (size_t)n_main); else a.tm_main = a.tm_tail;
        if (amb_launch_scan(a, sm_count, s) != cudaSuccess) return -2;
    } else
    {   // stand-in for the scan kernel: item i of the streams sits at segment coordinate i + kc, i.e. reported r' = i + kc
        const int shift = kc - P.H;
        std::vector<float> s0((size_t)n + shift + 1, 0.f), s1((size_t)n + shift + 1, 0.f);
        std::copy(bb, bb + n, s0.begin() + shift);
        std::copy(avg, avg + n, s1.begin() + shift);
        if (amb_launch_stream_candidates(a, s0.data(), s1.data(), (long long)n + shift, sm_count, s) != cudaSuccess) return -2;
    }
    const bool par = resolver != 1;
    if (amb_launch_compact(a, cand_j.data(), cand_cap, &ctr, par ? walk_scratch.data() : nullptr, n_samples, s) != cudaSuccess) return -3;
    AmbExactArgs ea{};
    ea.P = P; ea.S = S; ea.cand_j = cand_j.data(); ea.cand_info = cand_info.data(); ea.cand_avg = cand_avg.data(); ea.ctr = &ctr;
    // both regimes of the exact stage are exercised: the row-based kernel (threshold 0) unless the test asks for the
    // warp-per-candidate one (AMB_TEST_EXACT_DENSE = a large number)
    { const char* t = getenv("AMB_TEST_EXACT_DENSE"); ea.dense_threshold = t ? (unsigned)strtoul(t, nullptr, 10) : 0u; }
    if (amb_launch_exact(ea, sm_count, s) != cudaSuccess) return -4;
    AmbWalkArgs wa{};
    wa.P = P; wa.org = org; wa.ntot = ntot; wa.r_safe = 0; wa.flush = 1; wa.ctr = &ctr; wa.st = &st;
    wa.cand_j = cand_j.data(); wa.cand_info = cand_info.data(); wa.det_list = det_list.data();
    if ((par ? amb_launch_walk_par(wa, walk_scratch.data(), cand_cap, n_samples, s) : amb_launch_walk_seq(wa, s)) != cudaSuccess) return -5;
    AmbSliceArgs sl{};
    sl.P = P; sl.S = S; sl.cand_j = cand_j.data(); sl.cand_info = cand_info.data(); sl.cand_avg = cand_avg.data();
    sl.det_list = det_list.data(); sl.ctr = &ctr; sl.frames = frames.data(); sl.frame_cap = frame_cap;
    sl.chips_out = chips.data(); sl.org = org;
    if (amb_launch_slice(sl, sm_count, s) != cudaSuccess) return -6;
    if (ctr.overflow || ctr.frame_overflow) return -7;
    emul_last_counts[0] = ctr.ncand; emul_last_counts[1] = ctr.nreal_call; emul_last_counts[2] = (unsigned)st.fallback;
    const unsigned nd = ctr.nframes;
    if (nd > (unsigned)max_det) return -8;
    std::vector<unsigned> order(nd);
    for (unsigned k = 0; k < nd; k++) order[k] = k;
    std::sort(order.begin(), order.end(), [&](unsigned x, unsigned y) { return frames[x].sample_index < frames[y].sample_index; });
    for (unsigned k = 0; k < nd; k++) {
        index_out[k] = frames[order[k]].sample_index;
        frames_out[k] = frames[order[k]];
        memcpy(chips_out + (size_t)k * 240, chips.data() + (size_t)order[k] * 240, 240 * sizeof(float));
    }
    return (int)nd;
}

// amb_slicer_process: ndet packets of 240 chips -> frames (slicer_impl.cc:117-182)
extern "C" int emul_slicer(const float* chips, int ndet, amb_frame* out)
{
    int off[240] = {0};
    if (amb_upload_tables(off) != cudaSuccess) return -1;
    std::vector<float> c(chips, chips + (size_t)ndet * 240);
    return amb_launch_slice_chips(c.data(), ndet, out, nullptr) == cudaSuccess ? 0 : -2;
}

// amb_device_crc: n messages of `length` bytes
extern "C" int emul_crc(const uint8_t* data, int n, int length, uint32_t* out)
{
    int off[240] = {0};
    if (amb_upload_tables(off) != cudaSuccess) return -1;
    return amb_launch_crc(data, n, length, out, nullptr) == cudaSuccess ? 0 : -2;
}

// amb_launch_dcblock on a whole stream (raw-sample history = zeros): out[2n] = x[n-D+1] - MA_D(MA_D(x))[n]
extern "C" int emul_dcblock(const float* iq, int n, int D, float* out)
{
    const int nc = 2 * D - 2;
    std::vector<float2> carry(nc, make_float2(0.f, 0.f)), next(nc), fresh(n > 0 ? n : 1), ma0((size_t)n + D + 1024), o((size_t)n + D + 1024);
    memcpy(fresh.data(), iq, (size_t)n * sizeof(float2));
    if (amb_launch_dcblock(carry.data(), nc, fresh.data(), (long long)n, D, ma0.data(), o.data(), next.data(), nullptr) != cudaSuccess) return -1;
    memcpy(out, o.data(), (size_t)n * sizeof(float2));
    return 0;
}
