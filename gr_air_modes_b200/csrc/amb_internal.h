// Internal definitions shared by the kernels (amb_kernels.cu) and the host API (amb_api.cu).
// Reference citations are file:line under the gr-air-modes tree.
#pragma once
#include "amb_launch.h"
#include <stdint.h>
#include "../../include/airmodes_b200.h"

#define AMB_TILE 512           // samples per TMA tile (4 KiB of float2) = 2 rows
#define AMB_STAGE AMB_TILE      // segment granularity: carry/main/tail are whole tiles
#define AMB_ROW 256            // samples per warp row (8 per lane) = one TMA tile
#define AMB_MAX_SPC 10         // samples per chip supported (20 Msps)
#define AMB_SPAN_ROWS_ALIGN 32 // spans are multiples of 32 rows = one coarse bitmap word

// Everything the kernels need that the reference derives from (rate, threshold):
// preamble_impl.cc:56-68 (set_rate/set_threshold), :158-162 (pulse offsets), :205-208 (quiet zones),
// :192 (late-gate budget), :212,:237 (240*spc), rx_path.py:35,49,54 (window lengths and scales).
struct AmbParams {
    float spc_f, sps_f;   // d_samples_per_chip, d_samples_per_symbol (float!)
    int spc_i;            // int(d_samples_per_chip): PMF length, correlator samples/chip, ninputs rounding
    int L;                // 48*spc_i noise-floor window
    int H;                // history()-1
    int po1, po2, po3;    // int(2*spc), int(7*spc), int(9*spc)
    int qa0, qa1, qb0, qb1; // inclusive j ranges of the two quiet-zone loops
    int maxlate;          // number of late shifts the do/while allows
    int skip0;            // (int)(240*spc_f)
    float skip_f;         // 240*spc_f as the reference computes it
    float thr;            // d_threshold = powf(10, dB/20)
    float scale_p, scale_a; // (float)(1/spc_i), (float)(1/(48*spc_i))
    int use_pmf;
    int rate_int;
    // conservative pre-filter constants (see amb_kernels.cu, scan kernel)
    float cT;             // thr*scale_a*(1-eps)^2   (threshold side, slightly lowered)
    float one_eps;        // 1+eps                    (peak test slack)
    float gfac;           // absolute guard factor on the window sum
    int fwd;              // forward reach of the exact stage from a candidate start (bb samples)
    int64_t i_exact;      // for i_rel < i_exact: (int)((float)i_rel + skip_f) == i_rel + skip0
};

// Logical input of one call = carry ++ main ++ tail, each a multiple of AMB_STAGE samples.
struct AmbSegs {
    const float2* carry; const float2* main_; const float2* tail;
    int n_carry, n_main, n_tail;   // samples
    int n_valid;                   // samples of real data (carry + new); beyond it the tail is zeros
};

// Resolver state carried across calls (absolute reported coordinates r = sample + H).
struct AmbWalkState {
    long long pos;   // nitems_read at the start of the current general_work() call (preamble_impl.cc:164)
    long long p;     // next index the scan loop will look at
    int done;        // stream finished (flush processed)
    int fallback;    // parallel resolver handed over to the sequential one
    unsigned long long ncand_real, ndet;
    unsigned long long first_real, first_packet;   // amb_get_walk_summary: smallest start of a candidate passing :174-179 /
                                                   // smallest index of an accepted preamble in the last call (~0 = none)
};

struct AmbCounters {
    unsigned int ncand;        // candidates produced by the compaction
    unsigned int overflow;     // 1 = candidate capacity exceeded
    unsigned int nframes;      // frames appended (all calls since last poll)
    unsigned int frame_overflow;
    unsigned int ndet_call;    // detections in this call
    unsigned int npassed_call;
    unsigned int nreal_call;
    unsigned int ndet_list;    // entries of the detection list of this call (indices into the candidate arrays)
    unsigned int frame_base;   // frames queued before this call's (set by the resolver; slot = frame_base + list position)
};

struct AmbScanArgs {
    AmbParams P; AmbSegs S;
    int j_lo, j_hi;            // predicate evaluated for j in [j_lo, j_hi)
    int row_lo, row_hi;        // rows covering that range (row_lo multiple of 32)
    int rows_per_span, n_spans;
    uint32_t* coarse; uint32_t* fine; uint32_t* span_count;   // fine: 8 words per row, coarse: 1 bit per row
    uint32_t* group_count;     // candidates per group of 64 spans (zeroed by the prologue)
    alignas(64) CUtensorMap tm_carry;   // 2-D {32 floats, rows of 128 B}, box {32,32}, SWIZZLE_128B
    alignas(64) CUtensorMap tm_main;
    alignas(64) CUtensorMap tm_tail;
};

struct AmbExactArgs {
    AmbParams P; AmbSegs S;
    const int* cand_j; uint32_t* cand_info; float* cand_avg;
    const AmbCounters* ctr;
    unsigned int dense_threshold;   // candidates per call beyond which the row-based kernel decides instead of the warp-per-candidate one
    // split-form (float streams instead of IQ): if in0 != nullptr the exact stage reads these
    const float* in0; const float* in1; long long n_streams;
};

struct AmbWalkArgs {
    AmbParams P;
    const int* cand_j; uint32_t* cand_info;
    int* det_list;        // out: candidate indices of accepted preambles, unordered (the slicer's work list)
    AmbCounters* ctr; AmbWalkState* st;
    long long org;        // absolute reported index of j = 0
    long long ntot;       // flush: total items incl. history (N + H); else unused
    long long r_safe;     // !flush: first reported index that may not be decided yet
    int flush;
    int sm_count;         // grid sizing of the cluster walk (0: a small default)
};

struct AmbSliceArgs {
    AmbParams P; AmbSegs S;
    const int* cand_j; const uint32_t* cand_info; const float* cand_avg;
    const int* det_list;
    AmbCounters* ctr;
    amb_frame* frames; unsigned int frame_cap;
    float* chips_out;     // optional 240 floats per detection (same slot as the frame)
    long long org;
    const float* in0; const float* in1; long long n_streams;
};

// kernel launchers (amb_kernels.cu)
cudaError_t amb_launch_scan(const AmbScanArgs& a, int sm_count, cudaStream_t s);
cudaError_t amb_launch_compact(const AmbScanArgs& a, int* cand_j, unsigned int cand_cap, AmbCounters* ctr,
                               void* walk_scratch, long long n_samples, cudaStream_t s);
cudaError_t amb_launch_exact(const AmbExactArgs& a, int sm_count, cudaStream_t s);
cudaError_t amb_launch_dump(const float2* iq, long long n, const AmbParams& P, int stage, float* tmp, float* out, cudaStream_t s);
cudaError_t amb_launch_walk_reset(const AmbWalkArgs& a, void* scratch, long long n_samples, cudaStream_t s);
cudaError_t amb_launch_walk_summary(const AmbWalkArgs& a, cudaStream_t s);
cudaError_t amb_launch_set_state(AmbWalkState* st, long long pos, long long p, cudaStream_t s);
cudaError_t amb_launch_pack_summary(const AmbWalkArgs& a, long long i_exact, int have, long long* out, cudaStream_t s);
cudaError_t amb_launch_compose(const long long* gathered, int n_spans, long long* out, cudaStream_t s);
cudaError_t amb_launch_set_state_dev(AmbWalkState* st, const long long* entry, cudaStream_t s);
cudaError_t amb_launch_walk_seq(const AmbWalkArgs& a, cudaStream_t s);
cudaError_t amb_launch_walk_par(const AmbWalkArgs& a, void* scratch, unsigned int cand_cap, long long n_samples, cudaStream_t s);
size_t amb_walk_scratch_bytes(unsigned int cand_cap, long long n_samples);
cudaError_t amb_launch_slice(const AmbSliceArgs& a, int sm_count, cudaStream_t s);
cudaError_t amb_launch_carry(const AmbSegs& S, float2* dst, int kc, cudaStream_t s);
cudaError_t amb_launch_stream_candidates(const AmbScanArgs& a, const float* in0, const float* in1, long long n, int sm_count,
                                         cudaStream_t s);
cudaError_t amb_launch_slice_chips(const float* chips, int ndet, amb_frame* frames, cudaStream_t s);
cudaError_t amb_launch_crc(const uint8_t* data, int n, int length, uint32_t* out, cudaStream_t s);
cudaError_t amb_upload_tables(const int* chip_off);
cudaError_t amb_prefer_max_shared();
cudaError_t amb_launch_dcblock(const float2* rawcarry, int nc, const float2* fresh, long long n_new, int D,
                               float2* ma0_tmp, float2* out, float2* rawcarry_next, cudaStream_t s);
cudaError_t amb_launch_prologue(float2* tail, int tail_cap, const float2* src_rem, int n_rem,
                                uint32_t* group_count, int n_groups, cudaStream_t s);
size_t amb_scan_smem_bytes(int spc_i);
cudaError_t amb_launch_widen_sc16(const void* in_sc16, float2* out, long long n, int sm_count, cudaStream_t s);
