// TEST HARNESS (not a product path): the hot path's kernels and their launchers - gr_air_modes_b200/csrc/amb_kernels.cu,
// the TMA scan kernel included (its PTX helpers are emulated) - compiled for the host under tests/simt/simt_emul.h and
// driven by the library's own per-call rules (gr_air_modes_b200/csrc/amb_chain.h): the geometry of a call, the buffers
// (amb_chain_prepare, host memory here) and the sparse sequence compact -> exact -> walk -> slice that amb_process and
// amb_preamble_process run. tests/test_kernels_simt.py compares the results with the oracle. Built by the test with
// plain g++.
#include "simt_emul.h"

#include "../../gr_air_modes_b200/csrc/amb_kernels.cu"
#include "../../gr_air_modes_b200/csrc/amb_params.h"
#include "../../gr_air_modes_b200/csrc/amb_chain.h"

#include <algorithm>
#include <vector>

// A call's buffers, from the library's owner, freed on every way out. Nothing else uses them: growth needs no sync.
struct EmulBufs { AmbChainBufs b; ~EmulBufs() { amb_chain_free(&b); } };
static cudaError_t emul_no_sync() { return cudaSuccess; }

// The call's frames in stream order (the sort of amb_preamble_process and of the poll): index_out, chips_out (240 each)
// and frames_out (unstamped, unless NULL). Returns their number, < 0 on an overflow or when there are more than max_det.
static int emul_stream_order(const AmbChainBufs& b, const AmbCounters& ctr, int max_det, unsigned long long* index_out,
                             float* chips_out, amb_frame* frames_out)
{
    if (ctr.overflow || ctr.frame_overflow) return -6;
    const unsigned nd = ctr.nframes;
    if (nd > (unsigned)max_det) return -7;
    std::vector<unsigned> order(nd);
    for (unsigned k = 0; k < nd; k++) order[k] = k;
    std::sort(order.begin(), order.end(), [&](unsigned x, unsigned y) { return b.frames[x].sample_index < b.frames[y].sample_index; });
    for (unsigned k = 0; k < nd; k++) {
        index_out[k] = b.frames[order[k]].sample_index;
        if (frames_out) frames_out[k] = b.frames[order[k]];
        memcpy(chips_out + (size_t)k * 240, b.chips + (size_t)order[k] * 240, 240 * sizeof(float));
    }
    return (int)nd;
}

// One whole stream (first call, flush): amb_preamble_process with sf_total = 0. resolver: 1 sequential, else parallel.
// Returns the number of detections (<= max_det), < 0 on error; chips_out[240 * k], index_out[k] in stream order.
extern "C" int emul_preamble(const float* in0, const float* in1, int n, float rate, float threshold_db, int resolver,
                             int sm_count, float* chips_out, unsigned long long* index_out, int max_det,
                             unsigned* n_candidates)
{
    AmbParams P; int off[240];
    if (compute_params(rate, threshold_db, 0, &P, off) != AMB_OK) return -100;
    if (amb_upload_tables(off) != cudaSuccess) return -101;
    const long long m = n, ntot = m + P.H;
    std::vector<float> d0((size_t)m + 1, 0.f), d1((size_t)m + 1, 0.f);
    std::copy(in0, in0 + n, d0.begin());
    std::copy(in1, in1 + n, d1.begin());
    AmbScanArgs a{};
    a.P = P;
    amb_chain_geometry(&a, 0, ntot, true, sm_count, 0);
    EmulBufs eb; AmbChainErr er;
    if (amb_chain_prepare(&eb.b, &a, 0, amb_chain_cand_capacity(ntot), amb_chain_frame_bound(P, m), true, emul_no_sync, &er) < 0)
        return -102;
    AmbCounters ctr{}; AmbWalkState st{};
    AmbChainCall call{};
    call.P = P; call.in0 = d0.data(); call.in1 = d1.data(); call.n_streams = m;
    call.org = 0; call.ntot = ntot; call.r_safe = 0; call.flush = 1; call.ctr = &ctr; call.st = &st;
    call.n_samples = m + P.H + 4096;
    AmbChainOpts o{};
    o.sm_count = sm_count; o.par = resolver != 1; o.keep_chips = true;
    AmbChainSpan sp;
    cudaStream_t s = nullptr;
    if (amb_chain_split_scan(a, eb.b, d0.data(), d1.data(), m, &ctr, &st, sm_count, s, &er) < 0) return -1;
    if (amb_chain_launch(a, call, &eb.b, o, false, s, &sp, &er) < 0) return -2;
    if (n_candidates) { n_candidates[0] = ctr.ncand; n_candidates[1] = ctr.nreal_call; n_candidates[2] = (unsigned)st.fallback; }
    return emul_stream_order(eb.b, ctr, max_det, index_out, chips_out, nullptr);
}

static unsigned emul_last_counts[3];
extern "C" void emul_counts(unsigned* out) { memcpy(out, emul_last_counts, sizeof emul_last_counts); }

// The fused path on IQ (amb_process, one call over a whole stream, flush): the exact and slice kernels in their IQ form
// recompute |x|^2, the pulse matched filter and the noise-floor window from the samples (canonical arithmetic) through
// the carry ++ main ++ tail segment view, the prologue kernel stages the tail. With bb == NULL the scan kernel runs: its
// PTX helpers (mbarrier, 2-D TMA tile copy with the 128-byte swizzle) are emulated. Otherwise a stand-in writes its
// output - the candidate bitmap in segment coordinates - with the stream-candidate kernel from the (bb, avg) streams
// the caller computed with the canonical front end, shifted into the same coordinates.
// Returns detections in stream order: index_out, chips_out (240 each), frames_out (unstamped).
extern "C" int emul_process_iq(const float* iq, int n, const float* bb, const float* avg, float rate, float threshold_db,
                               int use_pmf, int resolver, int sm_count, float* chips_out, unsigned long long* index_out,
                               amb_frame* frames_out, int max_det)
{
    AmbParams P; int off[240];
    if (compute_params(rate, threshold_db, use_pmf, &P, off) != AMB_OK) return -100;
    if (amb_upload_tables(off) != cudaSuccess) return -101;
    const int kc = amb_chain_carry(P);
    std::vector<float2> carry(kc, make_float2(0.f, 0.f)), tail(AMB_TAIL_CAP), src(n > 0 ? n : 1);
    memcpy(src.data(), iq, (size_t)n * sizeof(float2));
    const AmbSegs S = amb_chain_segs(carry.data(), kc, src.data(), n, tail.data());
    const long long org = -(long long)kc + P.H, j_lo = -org, j_hi = S.n_valid;
    AmbScanArgs a{};
    a.P = P; a.S = S;
    amb_chain_geometry(&a, j_lo, j_hi, false, sm_count, 0);
    if (a.row_lo != 0) return -102;
    EmulBufs eb; AmbChainErr er;
    if (amb_chain_prepare(&eb.b, &a, 0, amb_chain_cand_capacity(j_hi - j_lo), amb_chain_frame_bound(P, j_hi - j_lo), true,
                          emul_no_sync, &er) < 0) return -103;
    AmbCounters ctr{}; AmbWalkState st{};
    cudaStream_t s = nullptr;
    if (amb_launch_prologue(tail.data(), AMB_TAIL_CAP, src.data() + S.n_main, n - S.n_main, a.group_count, 128, s) != cudaSuccess)
        return -1;
    if (!bb) {      // the real scan kernel: TMA tiles and mbarriers are emulated (simt_emul.h), the kernel source is the product's
        simt_make_tmap(&a.tm_carry, carry.data(), (size_t)kc);
        simt_make_tmap(&a.tm_tail, tail.data(), (size_t)AMB_TAIL_CAP);
        if (S.n_main) simt_make_tmap(&a.tm_main, src.data(), (size_t)S.n_main); else a.tm_main = a.tm_tail;
        if (amb_launch_scan(a, sm_count, s) != cudaSuccess) return -2;
    } else
    {   // stand-in for the scan kernel: item i of the streams sits at segment coordinate i + kc, i.e. reported r' = i + kc
        const int shift = kc - P.H;
        std::vector<float> s0((size_t)n + shift + 1, 0.f), s1((size_t)n + shift + 1, 0.f);
        std::copy(bb, bb + n, s0.begin() + shift);
        std::copy(avg, avg + n, s1.begin() + shift);
        if (amb_chain_split_scan(a, eb.b, s0.data(), s1.data(), (long long)n + shift, &ctr, nullptr, sm_count, s, &er) < 0) return -2;
    }
    AmbChainCall call{};
    call.P = P; call.S = S; call.org = org; call.ntot = (long long)n + P.H; call.r_safe = 0; call.flush = 1;
    call.ctr = &ctr; call.st = &st; call.n_samples = (long long)S.n_carry + S.n_main + S.n_tail;
    AmbChainOpts o{};
    o.sm_count = sm_count; o.par = resolver != 1; o.keep_chips = true;
    // both regimes of the exact stage are exercised: the row-based kernel (threshold 0) unless the test asks for the
    // warp-per-candidate one (AMB_TEST_EXACT_DENSE = a large number)
    { const char* t = getenv("AMB_TEST_EXACT_DENSE"); o.exact_dense = t ? (unsigned)strtoul(t, nullptr, 10) : 0u; }
    AmbChainSpan sp;
    if (amb_chain_launch(a, call, &eb.b, o, false, s, &sp, &er) < 0) return -3;
    emul_last_counts[0] = ctr.ncand; emul_last_counts[1] = ctr.nreal_call; emul_last_counts[2] = (unsigned)st.fallback;
    return emul_stream_order(eb.b, ctr, max_det, index_out, chips_out, frames_out);
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
