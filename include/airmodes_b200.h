/* airmodes_b200.h - C ABI of libairmodes_b200.so: the Mode S / ADS-B receive hot path of
 * gr-air-modes (|x|^2 -> pulse matched filter -> noise floor -> preamble detect -> PPM slice with
 * confidence -> 24-bit CRC) as hand-written sm_90a CUDA.
 *
 * This is the drop-in boundary for that path. The reference exposes it as GNU Radio C++ blocks
 * behind SWIG (swig/air_modes_swig.i:15-16); each entry point below names the reference interface
 * it replaces (file:line relative to the gr-air-modes tree). Plain pointers and sizes only.
 * There is NO CPU fallback: every compute entry point fails with AMB_ERR_NO_DEVICE / a CUDA error
 * when no sm_90 device is usable.
 *
 * Conventions
 *   IQ input    : interleaved float32 I,Q = gr_complex (python/rx_path.py:29), host or device memory.
 *   sample_index: the value the reference stamps, nitems_read(0)+i (lib/preamble_impl.cc:164,224),
 *                 i.e. stream sample number of the preamble peak + history()-1.
 *   Threading   : one amb_ctx per IQ stream, one producer thread (like one GNU Radio block thread).
 */
#ifndef AIRMODES_B200_H
#define AIRMODES_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define AMB_API __attribute__((visibility("default")))
#else
#define AMB_API
#endif

#define AMB_OK 0
#define AMB_ERR_INVALID (-1)      /* bad argument */
#define AMB_ERR_NO_DEVICE (-2)    /* no CUDA device / not sm_90: there is no CPU path */
#define AMB_ERR_CUDA (-3)         /* CUDA runtime error, see amb_last_error() */
#define AMB_ERR_RATE (-4)         /* rate < 2 Msps or samples/chip > 10 (unsupported geometry) */
#define AMB_ERR_OVERFLOW (-5)     /* internal candidate/frame buffers exhausted even after growth */
#define AMB_ERR_UNSUPPORTED (-6)  /* feature not built (use_dcblock) */
#define AMB_ERR_ALIGN (-7)        /* device IQ pointer not 16-byte aligned */
#define AMB_ERR_STATE (-8)        /* call not valid in this state (e.g. process after flush without reset) */

#define AMB_MEM_HOST 0          /* interleaved float32 I,Q in host memory (pinned or pageable) */
#define AMB_MEM_DEVICE 1        /* ... in device memory (read in place when 16-byte aligned) */
#define AMB_MEM_HOST_SC16 2     /* interleaved int16 I,Q in host memory, full scale 32768 (the receivers' wire format) */
#define AMB_MEM_DEVICE_SC16 3   /* ... in device memory */

typedef struct amb_ctx amb_ctx;

/* One detected preamble after slicing. Mirrors struct modes_packet (include/gr_air_modes/types.h:29-41)
 * plus the tag the preamble block attaches (lib/preamble_impl.cc:224-232). `passed` != 0 means the
 * frame survived every drop rule of slicer_impl::work (lib/slicer_impl.cc:162-182) and the reference
 * would have queued a message for it. */
typedef struct amb_frame {
    uint64_t sample_index;   /* abs_sample_cnt + i (preamble_impl.cc:224) */
    uint64_t secs;           /* tag_to_timestamp (preamble_impl.cc:100-137) */
    double frac;
    float ref_level;         /* reference_level (slicer_impl.cc:128-131) */
    uint32_t crc;            /* modes_check_crc ^ last 3 bytes (slicer_impl.cc:173-177) */
    uint8_t nbits;           /* 56 or 112 (slicer_impl.cc:140-142) */
    uint8_t df;              /* message_type (slicer_impl.cc:168) */
    uint8_t numlowconf;      /* saturates at 24 (slicer_impl.cc:157) */
    uint8_t passed;
    uint8_t lowconfbits[24];
    uint8_t data[14];
    uint8_t ec;              /* error correction outcome, AMB_EC_* (option "ec"); 0 unless it was attempted */
    uint8_t ec_flips;        /* bits flipped by a correction (AMB_EC_FIXED), else 0 */
    uint8_t pad_[4];         /* [0] ec_any, [1..2] ec_any_bits (AMB_FRAME_EC_ANY*), [3] ap_filter outcome (AMB_FRAME_AP) */
} amb_frame;                 /* 80 bytes */

/* amb_frame.ec: what the opt-in error correction (amb_set_option(ctx, "ec", K), K in 1..23) made of a DF11/DF17 frame
 * that the reference drops for a non-zero CRC syndrome (slicer_impl.cc:182). It searches the frame's low-confidence
 * bits (lowconfbits, minus the DF field 0-4) for the subsets whose flips zero the syndrome. Names after
 * bruteResultTypeDef (include/gr_air_modes/types.h:27). */
#define AMB_EC_NOT_TRIED 0       /* not a candidate, or the option is off */
#define AMB_EC_FIXED 1           /* Solution_Found: exactly one subset; data corrected, crc = 0, passed = 1 */
#define AMB_EC_TOO_MANY 2        /* Too_Many_LCBs: numlowconf > K (a saturated count of 24 always) */
#define AMB_EC_NO_SOLUTION 3     /* No_Solution: no subset zeroes the syndrome */
#define AMB_EC_AMBIGUOUS 4       /* Multiple_Solutions: more than one does; the frame stays dropped */

/* ec_any: what the opt-in second pass (amb_set_option(ctx, "ec_any", M), M in 1..2) made of a DF17 frame still
 * dropped for its CRC after the "ec" pass (when that is on too). It searches every pattern of at most M bits in
 * positions 5..111, whatever their confidence. The one- and two-bit syndromes there are non-zero and pairwise
 * distinct, so a fit is unique: AMB_EC_FIXED (data corrected, crc = 0, passed = 1, bits recorded) or
 * AMB_EC_NO_SOLUTION; AMB_EC_NOT_TRIED otherwise. DF11 is never tried: its parity may carry the interrogator's II/SI
 * code. The outcome and the flipped positions live in the first three bytes of amb_frame.pad_ (bytes 76-78 of the
 * frame), so the declared layout of amb_frame is the one it had before this pass existed: */
#define AMB_FRAME_EC_ANY(f) ((f)->pad_[0])                  /* AMB_EC_NOT_TRIED, AMB_EC_FIXED or AMB_EC_NO_SOLUTION */
#define AMB_FRAME_EC_ANY_BIT(f, i) ((f)->pad_[1 + (i)])     /* i = 0, 1: flipped positions, ascending; 0 = unused */

/* Address/parity check (amb_set_option(ctx, "ap_filter", S), S in 1..3600 seconds), after both correction passes.
 * A confirmer is a DF11/DF17 frame that passed with crc == 0 and that neither correction pass fixed; its address is
 * AA (data[1..3]). Subjects are never confirmers:
 *   AP subject     passed and df not in {11, 17}; its address is the syndrome in crc (AP xor parity)
 *   II/SI subject  df == 11, not passed, 0 < crc < 0x80 (an interrogator code in the parity); its address is AA
 * A subject is KNOWN when a confirmer g of the same address lies in this stream (since amb_reset / amb_set_rate, in a
 * call made with the option on) with g.sample_index < f.sample_index <= g.sample_index + S * (int)rate. A known AP
 * subject is unchanged and an unknown one gets passed = 0; a known II/SI subject gets passed = 1 (its message shows the
 * code as the crc token) and an unknown one stays dropped. data and crc are never changed. frames_passed counts the
 * result. The outcome lives in the last byte of amb_frame.pad_ (byte 79 of the frame), which the slicer zeroes.
 * The split-form amb_slicer_process carries no stream position and leaves it at AMB_AP_NOT_CHECKED. */
#define AMB_FRAME_AP(f) ((f)->pad_[3])
#define AMB_AP_NOT_CHECKED 0     /* not a subject, or the option was off */
#define AMB_AP_KNOWN 1           /* a confirmer of its address lies in the window */
#define AMB_AP_UNKNOWN 2         /* none does: an AP reply is dropped, an II/SI reply stays dropped */

typedef struct amb_stats {
    uint64_t samples_in;     /* complex samples accepted so far on this stream */
    uint64_t candidates;     /* first-four-test candidates handed to the exact stage (last call) */
    uint64_t candidates_real;/* ... of which pass the exact tests (preamble_impl.cc:174-179) */
    uint64_t detections;     /* accepted preambles = 240-chip packets (last call) */
    uint64_t frames_passed;  /* ... of which pass the slicer rules (last call) */
    uint64_t kernel_launches;/* kernels launched by this ctx since creation */
    float ms_scan;           /* device time of the streaming scan kernel, last call (timing on) */
    float ms_total;          /* device time of the whole call incl. copies on the ctx stream */
    int resolver_fallback;   /* 1 if the exact sequential resolver had to replace the parallel one */
    int ec_fixed;            /* frames the error correction fixed (last call; counted in frames_passed too) */
} amb_stats;

/* ---- lifetime -------------------------------------------------------------------------------
 * Replaces air_modes.rx_path(rate, threshold, queue, use_pmf, use_dcblock) (python/rx_path.py:27)
 * = preamble::make(channel_rate, threshold_db) (include/gr_air_modes/preamble.h:40,
 * lib/preamble_impl.cc:37-54) + slicer::make(queue) (include/gr_air_modes/slicer.h:41) + the
 * GNU Radio front end wired in rx_path.py:38-65. */
AMB_API int amb_create(int device, float rate, float threshold_db, int use_pmf, int use_dcblock, amb_ctx** out);
AMB_API void amb_destroy(amb_ctx* ctx);
/* Forget all stream state (history, scan position, pending frames): next sample is sample 0. */
AMB_API int amb_reset(amb_ctx* ctx);

/* ---- preamble accessors: preamble.h:42-45, preamble_impl.cc:56-76 --------------------------- */
AMB_API int amb_set_rate(amb_ctx* ctx, float channel_rate);     /* also rx_path.set_rate (rx_path.py:67-72); resets the stream */
AMB_API int amb_set_threshold(amb_ctx* ctx, float threshold_db);/* takes effect at the next amb_process */
AMB_API float amb_get_rate(const amb_ctx* ctx);                 /* (float)(int)rate, as preamble_impl.cc:74-76 */
AMB_API float amb_get_threshold(const amb_ctx* ctx);            /* dB, as preamble_impl.cc:70-72 */
AMB_API int amb_get_pmf(const amb_ctx* ctx);                    /* rx_path.get_pmf (rx_path.py:83-84) */
/* The rx_time stream tag a UHD source attaches to item 0 (lib/preamble_impl.cc:104-116,164-170): frames are then
 * stamped tag + sample_index/rate with the reference's `frac > 1.0f` carry (:127-130). Default (0, 0.0) = no tag.
 * Applies to frames collected afterwards. */
AMB_API int amb_set_start_time(amb_ctx* ctx, uint64_t secs, double frac);
/* A later rx_time tag (what a UHD source attaches after an overflow) at absolute item `offset` of the preamble
 * block's input = the coordinate of amb_frame.sample_index. Frames at or after `offset` are stamped against it
 * (tag_to_timestamp, preamble_impl.cc:100-137), earlier ones against the previous tag / the start time. This is what
 * the reference computes whenever no general_work() window straddles the tag; when one does, the reference latches the
 * tag at the START of that window (preamble_impl.cc:164-170) and stamps the window's earlier detections with a wrapped
 * unsigned delay - an artefact of the scheduler's buffer boundaries that is not reproduced. Ascending offsets only;
 * tags are forgotten by amb_reset. Applies to frames collected afterwards. */
AMB_API int amb_add_time_tag(amb_ctx* ctx, uint64_t offset, uint64_t secs, double frac);

/* Host-only (no GPU needed): the geometry preamble_impl derives from (rate, threshold) - preamble_impl.cc:56-68
 * (set_rate/set_threshold), :158-162 (pulse offsets), :205-208 (quiet-zone loop bounds), :184-192 (late-gate
 * budget), :212/:237 (240*spc) - as the kernels will use it. Returns AMB_ERR_RATE for unsupported rates. */
typedef struct amb_geometry {
    float samples_per_chip, samples_per_symbol, threshold;   /* d_samples_per_chip, d_samples_per_symbol, d_threshold */
    int rate_int, history, check_width;                      /* d_sample_rate, history(), d_check_width */
    int pulse_offset[4];
    int quiet_a[2], quiet_b[2];                              /* inclusive j ranges of the two space checks */
    int max_late, packet_skip;                               /* late shifts allowed; (int)(240*spc) */
    int pmf_len, floor_len;                                  /* rx_path.py:49,54 */
    int chip_offset_239;                                     /* int(239*spc), last extracted chip (:220) */
    int shard_back, shard_fwd;                               /* time-sharding halos in samples, see amb_seek */
} amb_geometry;
AMB_API int amb_query_geometry(float rate, float threshold_db, int use_pmf, amb_geometry* out);

/* ---- the hot path -----------------------------------------------------------------------------
 * Feed n_complex samples (2*n_complex floats). Replaces the scheduler calling
 * complex_to_mag_squared/moving_average_ff work() (rx_path.py:38-54),
 * preamble_impl::general_work (preamble_impl.cc:139-246) and slicer_impl::work
 * (slicer_impl.cc:102-198) on this stretch of the stream. flush != 0 marks end of stream: the
 * reference's end-of-input rules are applied and the stream must be reset before more input.
 * Work is enqueued on the ctx's CUDA stream; results are collected by amb_poll_frames. */
AMB_API int amb_process(amb_ctx* ctx, const float* iq_interleaved, size_t n_complex, int mem_kind, int flush);
/* Memory kinds. AMB_MEM_DEVICE (16-byte aligned) is read in place and must stay valid until amb_synchronize /
 * amb_poll_frames / amb_join + a wait on the caller's side. Everything else is consumed before amb_process returns:
 * host memory travels through a library-owned ring of pinned host + device chunk buffers (option "ingest_chunk",
 * default 2^22 samples) on a copy stream, so the H2D copy of one chunk overlaps the kernels of the previous one;
 * pinned caller memory is DMA'd from where it lies, pageable memory is first gathered into the ring by a few copy
 * threads (option "copy_threads"). Calls smaller than option "coalesce" (default 2^18 samples) are gathered and only
 * dispatched once that many samples are pending or when results are asked for (amb_poll_frames, amb_synchronize,
 * flush) - GNU Radio hands a sink at most 32 k items per work() call. The *_SC16 kinds take interleaved int16 I,Q and
 * widen them on the device with x * 2^-15 (exact): half the PCIe bytes of float32, bit-identical results to feeding
 * the float32 the host-side conversion (radio.py:163-173, cpu_format "fc32") would have produced. `iq_interleaved`
 * then points to int16 data. */

/* Wait for enqueued work and copy out up to `max` frames in stream order (all detections; test
 * .passed for what slicer_impl.cc:193-194 would queue). Returns the count, or <0 on error.
 * amb_pending_frames() tells how many are waiting (also synchronises). */
AMB_API int amb_poll_frames(amb_ctx* ctx, amb_frame* out, int max);
AMB_API int amb_pending_frames(amb_ctx* ctx);
/* Non-blocking variant for streaming callers (a GNU Radio work() function): returns the frames of the calls that
 * have already completed on the device, in stream order, and leaves work in flight alone. Host input that is still
 * being gathered (see amb_process) is not forced out. */
AMB_API int amb_poll_ready(amb_ctx* ctx, amb_frame* out, int max);
/* The device-side amb_poll_frames: waits for enqueued work, then writes every frame that has not been handed out yet to
 * DEVICE memory - in stream order and stamped (tag_to_timestamp, preamble_impl.cc:100-137), i.e. byte for byte what
 * amb_poll_frames would have copied to the host - so that a consumer on the same GPU (amb_decode_frames_device) reads
 * them without a PCIe round trip. Only the count crosses to the host. out_dev == NULL: report the count, consume
 * nothing. Returns the count, AMB_ERR_OVERFLOW (nothing consumed) if cap is too small. Frames that an earlier
 * amb_poll_ready moved to the host side stay there. Option "order_tile" (power of two <= 2048, default 2048) sizes the
 * shared-memory tile of the ordering network. */
AMB_API int amb_drain_device(amb_ctx* ctx, amb_frame* out_dev, int cap);

/* Message text exactly as slicer_impl.cc:186-192 builds it: "<hex payload> <crc %06x> <ref> <secs> <frac>".
 * `first` != 0 formats ref with the stream's default precision 6 (the first message a slicer instance
 * emits; setprecision(10) at :192 is sticky afterwards). Returns strlen, <0 if buflen too small. */
AMB_API int amb_format_message(const amb_frame* f, int first, char* buf, size_t buflen);
/* The same for n frames at once: the messages of the frames with passed != 0, in order, joined by '\n' (what
 * slicer_impl::work queues for them, slicer_impl.cc:186-194). `first` != 0: the first message written is the stream's
 * first (precision 6), all later ones use precision 10. Returns the number of messages, <0 if buflen is too small
 * (128 bytes per frame always suffice). */
AMB_API int amb_format_messages(const amb_frame* frames, int n, int first, char* buf, size_t buflen);

/* unsigned int modes_check_crc(unsigned char data[], int length) (include/gr_air_modes/modes_crc.h:26,
 * lib/modes_crc.cc:55-63). Host helper with the same table; the device CRC is a separate kernel path. */
AMB_API uint32_t amb_modes_check_crc(const uint8_t* data, int length);
/* Same CRC computed by the device routine used inside the slicer kernel (parity hook). `n` messages of
 * `length` bytes each, packed; out[n]. */
AMB_API int amb_device_crc(amb_ctx* ctx, const uint8_t* data, int n, int length, uint32_t* out);

/* ---- split-form blocks (stream contract of the two reference blocks) ---------------------------
 * preamble: in0 = signal, in1 = moving-average reference (preamble_impl.cc:43), the next n items of both streams
 * in host memory (flush != 0 marks the end of the stream; the next call then starts a new one); out = 240 chips
 * per detection decided in this call + reported index (tag offset). Returns the number of detections
 * (<= max_det) or <0. */
AMB_API int amb_preamble_process(amb_ctx* ctx, const float* in0, const float* in1, size_t n, int flush,
                         float* chips_out, uint64_t* index_out, int max_det);
/* slicer: ndet packets of 240 chips (slicer_impl.cc:117-182) -> frames (sample_index/secs/frac are
 * taken from the arrays, as the slicer takes them from the tag value, slicer_impl.cc:184). */
AMB_API int amb_slicer_process(amb_ctx* ctx, const float* chips, int ndet, const uint64_t* secs,
                       const double* frac, amb_frame* out);

/* ---- plumbing ---------------------------------------------------------------------------------- */
AMB_API int amb_set_stream(amb_ctx* ctx, void* cuda_stream);   /* run on a caller-owned cudaStream_t */
AMB_API int amb_enable_timing(amb_ctx* ctx, int on);           /* CUDA events around the scan kernel / the call */
AMB_API int amb_get_stats(amb_ctx* ctx, amb_stats* out);       /* synchronises */
/* Device time (ms) of the streaming scan kernel for the most recent calls made with timing on (oldest
 * first, at most 64). Returns how many were written. Synchronises. */
AMB_API int amb_get_scan_times(amb_ctx* ctx, float* ms_out, int max);
/* Timeline of the most recent calls made with timing on (oldest first, at most 63), three floats per call in ms:
 * idle time of the scan stream in front of the call's scan, the scan kernel, and scan end -> end of the call's sparse
 * stages (which run on a second stream under the next call's scan). Returns the number of calls. Synchronises. */
AMB_API int amb_get_timeline(amb_ctx* ctx, float* ms_out, int max_calls);
AMB_API int amb_synchronize(amb_ctx* ctx);
/* amb_process returns with work pending on the caller-visible stream AND on an internal stream (the sparse
 * kernels of call k overlap the streaming pass of call k+1). amb_join makes the caller-visible stream wait for
 * all of it without blocking the host; amb_synchronize / amb_poll_frames block. Input buffers must stay valid
 * until one of them. amb_set_option("overlap", 0) restores strictly stream-ordered behaviour. */
AMB_API int amb_join(amb_ctx* ctx);
/* The converse: make the context's streams wait for everything enqueued so far on `cuda_stream` (the stream that
 * produces a device-resident input buffer) before the next amb_process reads it. No host synchronisation. */
AMB_API int amb_wait_stream(amb_ctx* ctx, void* cuda_stream);
/* Parity dumps of the last amb_process call: candidate start indices (reported coordinates) and their
 * exact-stage verdict: bits 0-7 late shift, bit 8 passes preamble_impl.cc:174-179, bit 9 valid preamble
 * (:205-209), bit 10 visited-and-accepted. Returns count. */
AMB_API int amb_debug_candidates(amb_ctx* ctx, uint64_t* index, uint32_t* info, int max);
/* "resolver": 0 auto, 1 sequential, 2 parallel. "ec": K = 0 (default, off) .. 23, error correction over the
 * low-confidence bits of frames dropped for their CRC (see AMB_EC_*); persists across amb_reset / amb_set_rate.
 * "ec_any": M = 0 (default, off), 1 or 2, correction of DF17 frames by at most M flipped bits anywhere in 5..111, after
 * "ec" (see amb_frame.ec_any); persists likewise. Both apply from the next call.
 * "ap_filter": S = 0 (default, off) .. 3600 seconds, the address/parity check against the aircraft confirmed within
 * the last S seconds (see AMB_FRAME_AP); persists likewise and applies from the next call, while the table of confirmed
 * addresses (128 MiB of device memory, allocated at the first call with the option on) is cleared by amb_reset /
 * amb_set_rate. Not available in time-sharded operation: with S > 0, amb_seek and "defer_resolve" = 1 return
 * AMB_ERR_STATE, and so does setting S > 0 while "defer_resolve" is on or after an amb_seek (until amb_reset). */
AMB_API int amb_set_option(amb_ctx* ctx, const char* name, int value);
/* Parity dump of the GNU Radio front end wired in rx_path.py:38-54, for a short HOST buffer taken as a whole stream
 * (zeros before sample 0): stage M2 = complex_to_mag_squared (:38), BB = the preamble block's in0 (PMF output, :48-51,
 * or m2 when the PMF is off), AVG = its in1 (:54). n_complex floats are written to `out` (2*n_complex for DC). The hot path never
 * materialises these streams; this evaluates the same canonical arithmetic at every sample. */
#define AMB_STAGE_M2 0
#define AMB_STAGE_BB 1
#define AMB_STAGE_AVG 2
#define AMB_STAGE_DC 3   /* output of filter.dc_blocker_cc(100*spc, False) (rx_path.py:39-41): 2*n_complex floats */
AMB_API int amb_dump_stage(amb_ctx* ctx, int stage, const float* iq_interleaved, size_t n_complex, float* out);

/* ---- one stream time-sharded over several contexts / GPUs (no reference equivalent) ----------
 * The only state preamble_impl::general_work carries from one stretch of the stream to the next is where its
 * loop stands: nitems_read at the start of the current call (`pos`, preamble_impl.cc:164) and the next index
 * it will look at (`p`; an accepted packet jumps it 240*spc ahead, :237). Everything else is a function of
 * the samples. So a long recording can be cut into spans, one per context:
 *   span k is given the samples [first_sample_k, end_k) and decides the reported indices
 *   [first_decision_k, first_decision_{k+1});  first_decision_k >= first_sample_k + shard_back (the filter
 *   windows and the block history must be warm), end_k = first_decision_{k+1} + shard_fwd for every span but
 *   the last (flush = 0), the last span ends with the recording (flush = 1). Reported index = sample index +
 *   history()-1. Halos come from amb_query_geometry.
 * amb_seek resets the stream and positions it; `entry` is the loop state at first_decision (NULL: a fresh
 * general_work call starts there). With option "defer_resolve" = 1 amb_process stops after the dense stages
 * (scan, candidate compaction, exact preamble tests - none of which depends on the loop state), so all spans
 * run concurrently; amb_resolve(entry) then walks the candidates with the state handed over by the previous
 * span and slices the accepted packets, and amb_get_walk_state returns the state to hand to the next span.
 * In deferred mode exactly one amb_process call is allowed between amb_seek and amb_resolve, and its input
 * buffer must stay valid until amb_resolve has completed. Frames carry stream-global sample indices. */
typedef struct amb_walk_state { int64_t pos, p; } amb_walk_state;
AMB_API int amb_seek(amb_ctx* ctx, uint64_t first_sample, uint64_t first_decision, const amb_walk_state* entry);
AMB_API int amb_resolve(amb_ctx* ctx, const amb_walk_state* entry);      /* NULL: keep the context's own state */
AMB_API int amb_get_walk_state(amb_ctx* ctx, amb_walk_state* out);       /* synchronises */
/* Speculative resolution, which takes the hand-over chain off the critical path: resolve every span but the last
 * right away with the default entry ("a fresh general_work call starts at first_decision"), exchange the summaries,
 * and keep a span's result if the true entry (pos, p) - the previous span's exit - cannot have changed it:
 *   p <= first_real (or there is none): the walk never looks at p again once it is behind the first candidate that
 *       passes the pulse tests (preamble_impl.cc:174-179), and
 *   first_packet - pos < exact_span (or there is none): the float arithmetic of :237 is then exact for the true and
 *       for the assumed pos alike (later packets only depend on the one before them).
 * The span's exit state is then (first_packet >= 0 ? pos : the true entry pos, p) as reported here. Otherwise call
 * amb_resolve again with the true entry: the earlier resolution (verdicts, frames) is discarded - allowed until the
 * span's frames have been polled. The last span (flush) is not speculated on: the end-of-stream rules (:150,
 * :212-216) depend on pos directly. first_real / first_packet are -1 when absent. */
typedef struct amb_walk_summary {
    int64_t pos, p;                  /* exit state of this resolution */
    int64_t first_real, first_packet;
    int64_t exact_span;
    int64_t frames_passed;           /* messages this span would queue (slicer_impl.cc:193-194) */
} amb_walk_summary;
AMB_API int amb_get_walk_summary(amb_ctx* ctx, amb_walk_summary* out);   /* synchronises */
/* The same exchange WITHOUT the host in the loop (one NCCL all-gather of 48 bytes per span between two tiny kernels):
 *   amb_walk_summary_async     the six int64 of amb_walk_summary {pos, p, first_real, first_packet, exact_span,
 *                              frames_passed}, written to device memory by a kernel on the context's second stream;
 *   amb_join + all-gather      (the caller's collective, ordered on the caller-visible stream);
 *   amb_compose_entries_async  every rank composes all spans' true entries from the gathered n_spans x 6 table:
 *                              out[0] = first span whose speculation fails (n_spans - 1: none), out[1 + 2k], out[2 + 2k] =
 *                              entry (pos, p) of span k, out[1 + 2 n_spans + k] = messages queued before span k;
 *   amb_resolve_device         the last span (never speculated on) takes its entry from that output on the device.
 * A pass is then a fixed sequence of enqueues; the host only reads out[0] afterwards, and re-resolves the rare pass whose
 * speculation failed with amb_resolve as before. */
AMB_API int amb_walk_summary_async(amb_ctx* ctx, int64_t* dev_out6);
AMB_API int amb_compose_entries_async(amb_ctx* ctx, const int64_t* gathered_dev, int n_spans, int64_t* out_dev, void* cuda_stream);
AMB_API int amb_resolve_device(amb_ctx* ctx, const int64_t* entry_dev, void* after_stream);
/* cuda_stream / after_stream: the caller's stream the exchange runs on (NULL: the caller-visible stream). Running the
 * collective on a side stream (amb_join_stream) keeps the scan stream free for the next pass. */
AMB_API int amb_join_stream(amb_ctx* ctx, void* cuda_stream);

/* ---- Mode A/C replies (option "modeac", no reference equivalent) ---------------------------------------------
 * Secondary-radar replies: a framing pulse F1, 13 code pulses 1.45 us apart, F2 at 20.3 us and an optional SPI pulse
 * at 24.65 us. With amb_set_option(ctx, "modeac", 1) every call also finds them in the same canonical front end the
 * preamble block reads. Notation, on the stream since amb_create / amb_reset / amb_set_rate (not on its cut into calls):
 *   in[n]   the canonical bb (PMF output, or |x|^2 without the PMF; after the DC blocker when that is on), zeros
 *           before sample 0 and after the end at flush
 *   avg[n]  the canonical 48*spc noise floor; thr = the preamble threshold (amb_geometry.threshold)
 *   o(t)    (int)floor(t * rate_int / 1e6 + 0.5), the sample offset of t us, evaluated in double
 *   slot k  o(1.45 k), k = 0..14: F1, C1 A1 C2 A2 C4 A4 X B1 D1 B2 D2 B4 D4, F2; gap g = o(1.45 g + 0.725), g = 0..13;
 *           SPI = o(24.65)
 * A start i is a reply when
 *   1  in[i] > avg[i]*thr, in[i-1] < in[i] and !(in[i+1] > in[i])     (rising-edge peak, preamble_impl.cc:173-175)
 *   2  !(in[i+o(20.3)] < avg[i]*thr)                                  (F2)
 *   3  avgpeak = (in[i] + in[i+o(20.3)]) / 2.0f, space = avg[i] + (avgpeak - avg[i]) / thr   (float, as :198-203)
 *   4  in[i] and in[i+o(20.3)] both > space and > (avg[i]*thr)*thr, and !(in[i+o(10.15)] > space)
 *                                                                     (framing pulses clear of the floor, X quiet)
 *   5  !(in[i+gap g] > space) for all 14 gaps                         (what keeps Mode S data blocks out)
 *   6  code bit 12-(k-1) = in[i+slot k] > space (k = 1..13; bit 6 = X = 0); spi = in[i+o(24.65)] > space
 *   7  no j with i - o(25.1) <= j < i satisfies 1-5, whether or not j was dropped itself (a reply's own code pulses)
 * and becomes a record: sample_index = the reported index frames use (sample + history()-1), stamped as a frame at that
 * index (tag_to_timestamp), code and spi, peak = avgpeak and floor = avg[i] (raw floats, no dB), squawk =
 * decode_id(code) (parse.py:233-254), altitude = decode_alt(code, True) (altitude.py) when D1 = 0 and C1 C2 C4 is one of
 * 001, 011, 010, 110, 100, else AMB_NO_ALTITUDE. Records come in ascending sample_index, whatever the cut into calls.
 * The option needs the PMF and at least 4 Msps (2 samples per 0.5 us chip; amb_process returns AMB_ERR_UNSUPPORTED
 * otherwise): without them a 0.45 us pulse is sampled too coarsely for the fixed offsets. It is accepted only before
 * the first amb_process after amb_create / amb_reset / amb_set_rate (AMB_ERR_STATE otherwise) and persists across them. It is not available in time-sharded operation or with the split-form
 * amb_preamble_process (AMB_ERR_STATE). With it off nothing is launched and nothing changes. */
typedef struct amb_modeac {
    uint64_t sample_index;   /* reported index of F1 (the same numbering as amb_frame.sample_index) */
    uint64_t secs;           /* tag_to_timestamp, as a frame at sample_index */
    double frac;
    float peak;              /* avgpeak of rule 3 */
    float floor;             /* avg[i] */
    int32_t altitude;        /* feet, or AMB_NO_ALTITUDE */
    uint16_t code;           /* 13 bits C1 A1 C2 A2 C4 A4 X B1 D1 B2 D2 B4 D4, MSB first (the Mode S ID13 / AC13 layout) */
    uint16_t squawk;         /* decode_id(code): four octal digits read as a decimal number (7700 = 0x1E14) */
    uint8_t spi;             /* 1 when the SPI pulse is present */
    uint8_t pad_[7];
} amb_modeac;                /* 48 bytes */
#ifdef __cplusplus
static_assert(sizeof(amb_modeac) == 48, "amb_modeac is 48 bytes");
#else
_Static_assert(sizeof(amb_modeac) == 48, "amb_modeac is 48 bytes");
#endif
/* Counts since amb_create / amb_reset / amb_set_rate: starts passing rules 1-2, replies, starts that pass 1-6 but are
 * dropped by rule 7, and replies with an altitude. */
typedef struct amb_modeac_stats { uint64_t candidates, replies, overlap_drops, with_altitude; } amb_modeac_stats;
/* Wait for enqueued work and copy out up to `max` replies in stream order, stamped; returns the count. */
AMB_API int amb_poll_modeac(amb_ctx* ctx, amb_modeac* out, int max);
AMB_API int amb_pending_modeac(amb_ctx* ctx);
/* The device-side amb_poll_modeac: every reply not handed out yet, in stream order and stamped, written to DEVICE
 * memory. out_dev == NULL: report the count, consume nothing. AMB_ERR_OVERFLOW (nothing consumed) if cap is too small.
 * Replies already moved to the host by amb_poll_modeac / amb_pending_modeac stay there. */
AMB_API int amb_drain_modeac_device(amb_ctx* ctx, amb_modeac* out_dev, int cap);
AMB_API int amb_get_modeac_stats(amb_ctx* ctx, amb_modeac_stats* out);   /* synchronises */

/* ---- batch field decode of queued frames (SURVEY.md 8 row f4) ---------------------------------------
 * What the reference does per message in Python after the slicer: modes_reply field extraction
 * (python/parse.py:27-231), decode_alt (python/altitude.py:28-108), decode_id (parse.py:233-254), the BDS0,5 / 0,6 /
 * 0,8 / 0,9 / 6,1 and MB/TCAS sub-decodes (parse.py:256-420) and the stateful CPR position decoder
 * (python/cpr.py:183-240: latest even/odd report per aircraft, 10 s / 25 s expiry, global decode, range/bearing) -
 * here as one GPU pass over a batch of frames in stream order. A decoder owns the per-aircraft report table in device
 * memory (direct-mapped by (ICAO, surface, even/odd): 2^26 entries, 1 GiB) and carries it from batch to batch, like
 * one cpr_decoder instance. One difference, by necessity: cpr.py stamps reports with time.time() when the message
 * is parsed (cpr.py:219-221); a batch has no wall clock, so "now" is the frame's own timestamp secs + frac. Frames
 * must come in non-decreasing time order. No CPU path: without a device amb_decoder_create fails. */
#define AMB_FS_NO_HANDLER 0x01   /* the parser raised NoHandlerError (unknown DF / FTC / BDS0,9 subtype / MB register,
                                    parse.py:52-68): the reference drops the message; only df, ecc (and icao) are set */
#define AMB_FS_METRIC_ALT 0x02   /* decode_alt(ac) raised MetricAltError (altitude.py:32-43): altitude not set */
#define AMB_FS_CPR_NO_POS 0x04   /* CPRNoPositionError: no live even/odd pair (cpr.py:231), or a surface report
                                    without a receiver location (cpr.py:97-99) */
#define AMB_FS_CPR_STRADDLE 0x08 /* CPRBoundaryStraddleError (cpr.py:120-121); AMB_FS_CPR_NO_POS is set as well */
#define AMB_FS_HAS_POS 0x10      /* lat / lon valid */
#define AMB_FS_HAS_RANGE 0x20    /* range / bearing valid (receiver location known, cpr.py:233-237) */
#define AMB_FS_METRIC_THREAT 0x40 /* decode_alt(tida) raised MetricAltError in the TCAS threat sub-decode (parse.py:407): threat_alt not set */
#define AMB_FS_NOT_QUEUED 0x80   /* frame.passed == 0: the slicer never queued it, nothing was decoded */
#define AMB_NO_ALTITUDE INT32_MIN

typedef struct amb_fields {
    uint32_t icao;        /* "aa" where the DF carries one (11, 17), else ecc = AP ^ parity, what msprint.py prints */
    uint32_t ecc;         /* the frame's crc field = message token 2 (parse.py:425) */
    uint8_t df;           /* modes_reply.get_type() (parse.py:228-229) */
    uint8_t status;       /* AMB_FS_* */
    uint8_t bds;          /* DF17: me_reply.get_type() 0x05 / 0x06 / 0x08 / 0x09 / 0x61 (parse.py:140-152); DF20/21: bds1 */
    uint8_t subtype;      /* DF17 BDS0,9: bds09_reply.get_type() 0 / 1 / 3 (parse.py:110-117); 0xff otherwise */
    uint8_t ca, fs, vs, ri;               /* whichever the DF has (parse.py:210-219), else 0 */
    uint8_t sl, cc, dr, um;
    uint8_t ftc, cat, cpr_format, surface;/* DF17 "ftc", BDS0,8 "cat", BDS0,5/0,6 "cpr"; surface = 1 for BDS0,6 */
    uint8_t eps, ast, bds2, tti;          /* BDS6,1 "eps"; BDS0,9-3 "ast" (1 = TAS); MB "bds2"; TCAS "tti" */
    int32_t altitude;     /* decode_alt(ac, True) for DF0/4/16/20, decode_alt(alt, False) for BDS0,5; AMB_NO_ALTITUDE if absent */
    int32_t squawk;       /* decode_id(id) for DF5/21, else -1 */
    int32_t threat_alt;   /* TCAS threat altitude decode_alt(tida, True) (parse.py:407) */
    uint32_t cpr_lat, cpr_lon;            /* encoded 17-bit position */
    uint32_t aux[4];      /* MB bds1 = 1: acs, bcs, ecs, cfs; bds1 = 3: ara, rac, rat | mte << 1, tid (tti 1) or tidr | tidb << 8 (tti 2) */
    char ident[8];        /* BDS0,8 / MB bds1 = 2 callsign (parse.py:257-279, 374-378), no terminator */
    double lat, lon;      /* global CPR decode (cpr.py:89-153), or the local one (AMB_LOCAL_DECODED), degrees; NaN unless AMB_FS_HAS_POS */
    double range, bearing;/* range_bearing(my_location, position) (cpr.py:158-181): statute miles, degrees */
    double val[4];        /* BDS0,9-0: velocity, heading, vert_spd, turn_rate (parse.py:288-313)
                             BDS0,9-1: velocity, heading, vert_spd, alt_geo_diff (parse.py:315-348)
                             BDS0,9-3: mag_hdg, vel, vert_spd, geo_diff (parse.py:350-364)
                             BDS0,6  : ground_track (parse.py:283) */
    uint64_t pad_;        /* [byte 0] local CPR (AMB_FIELDS_LOCAL), [1..4] Comm-B (AMB_FIELDS_COMMB*), [5..7] AMB_FIELDS_ES* */
} amb_fields;             /* 144 bytes */

/* Locally referenced CPR decode (amb_decoder_set_option(d, "local_cpr", S), S in 1..600 seconds). After the global
 * decode, every queued BDS0,5 / BDS0,6 message without AMB_FS_HAS_POS is decoded relative to its aircraft's reference
 * position - the last position (global or local) of the same 24-bit ICAO, airborne and surface alike - when that
 * position's message lies at most S seconds back (0 <= t - ref.t <= S, t = secs + frac): cpr_resolve_local
 * (cpr.py:61-82), longitude brought into (-180, 180] with one +/-360, rejected when |lat| > 90 or when it lies more
 * than half a latitude zone (dlat / 2) from the reference. An accepted fix sets lat / lon and AMB_FS_HAS_POS (with a
 * receiver location also range / bearing and AMB_FS_HAS_RANGE) and becomes the new reference; AMB_FS_CPR_NO_POS and
 * AMB_FS_CPR_STRADDLE keep the global verdict. A global fix leaves the record as it is and becomes the reference.
 * The outcome lives in the first byte of amb_fields.pad_ (byte 136 of the record): */
#define AMB_FIELDS_LOCAL(r) (((uint8_t*)&(r)->pad_)[0])
#define AMB_LOCAL_NOT_TRIED 0    /* option off, not a position message, or the global decode gave a position */
#define AMB_LOCAL_DECODED 1      /* position from the local decode */
#define AMB_LOCAL_NO_REF 2       /* the aircraft has no reference position */
#define AMB_LOCAL_STALE 3        /* its reference position is more than S seconds old (or stamped later than the message) */
#define AMB_LOCAL_REJECTED 4     /* the local decode failed the plausibility check; the reference is kept */
#define AMB_LOCAL_CPR_MAX 600

/* Comm-B register inference (amb_decoder_set_option(d, "commb", S), S in 1..600 seconds). The parser accepts an MB word
 * only when its first byte names register 0,0 / 1,0 / 2,0 / 3,0 (parse.py:180-190); the Enhanced Surveillance replies
 * (BDS 4,0 / 5,0 / 6,0) say nothing of their register and stay AMB_FS_NO_HANDLER. With the option on, a queued 112-bit
 * DF20/21 record whose status is exactly AMB_FS_NO_HANDLER and whose MB first byte is not one of the parser's registers
 * is tried. MB bits are numbered 1..56 (MB bit k = message bit 32 + k); a signed field is a sign bit and n magnitude
 * bits read as two's complement. Fields 0..4 (status bit, value bits, LSB):
 *   4,0  0 MCP/FCU selected altitude 1, 2-13, 16 ft   1 FMS selected altitude 14, 15-26, 16 ft
 *        2 baro setting - 800 mb 27, 28-39, 0.1 mb   3 VNAV/ALT/APP mode bits 48, 49-51   4 target altitude source 54, 55-56
 *        reserved (must be 0) 40-47, 52-53
 *   5,0  0 roll 1, s2 3-11, 45/256 deg   1 true track 12, s13 14-23, 90/512 deg   2 ground speed 24, 25-34, 2 kt
 *        3 track angle rate 35, s36 37-45, 8/256 deg/s   4 true airspeed 46, 47-56, 2 kt
 *   6,0  0 magnetic heading 1, s2 3-12, 90/512 deg   1 IAS 13, 14-23, 1 kt   2 Mach 24, 25-34, 2.048/512
 *        3 baro altitude rate 35, s36 37-45, 32 ft/min   4 inertial vertical rate 46, s47 48-56, 32 ft/min
 * A register is a candidate when every field whose status bit is 0 has all its value bits 0, at least one status bit
 * is 1, the reserved bits are 0, and every present field is plausible (raw units): 4,0 selected altitudes <= 3125, baro
 * 700..3000; 5,0 |roll| <= 284, GS <= 400, TAS <= 300, |GS - TAS| <= 125 when both are present; 6,0 IAS <= 500,
 * Mach <= 250, |baro rate| and |inertial rate| <= 187. One candidate: AMB_COMMB_DECODED. Several: when 5,0 is among them
 * with GS and track present and the address (icao) has a reference - the latest earlier queued DF17 BDS0,9 subtype 0/1
 * record of that icao with val[0], val[1] not NaN, taken when 0 <= t - t_ref <= S (t = secs + frac) - 5,0 is kept alone
 * when |2 gs - val[0]| <= 20 kt and the track difference (fmod(|track - val[1]|, 360), folded to 0..180) is <= 10 deg,
 * else dropped; one register left: AMB_COMMB_RESOLVED. Otherwise AMB_COMMB_AMBIGUOUS. The status and every other field
 * of the record stay as they are; the option writes only aux and bytes 1..4 of pad_: */
#define AMB_FIELDS_COMMB(r) (((uint8_t*)&(r)->pad_)[1])        /* outcome, AMB_COMMB_* */
#define AMB_FIELDS_COMMB_REG(r) (((uint8_t*)&(r)->pad_)[2])    /* 0x40 / 0x50 / 0x60 when DECODED or RESOLVED, else 0 */
#define AMB_FIELDS_COMMB_MASK(r) (((uint8_t*)&(r)->pad_)[3])   /* bit i = status bit of field i of that register */
#define AMB_FIELDS_COMMB_CAND(r) (((uint8_t*)&(r)->pad_)[4])   /* candidates: bit 0 = 4,0, bit 1 = 5,0, bit 2 = 6,0 */
#define AMB_FIELDS_COMMB_RAW(r, i) (((int16_t*)(r)->aux)[i])   /* raw value of field i (0 when absent); 5..7 are 0 */
#define AMB_COMMB_NOT_TRIED 0    /* option off, or not an eligible record */
#define AMB_COMMB_DECODED 1      /* exactly one candidate register */
#define AMB_COMMB_RESOLVED 2     /* several, one left after the test against the aircraft's ADS-B velocity */
#define AMB_COMMB_AMBIGUOUS 3    /* several, and the velocity test could not apply or left more than one */
#define AMB_COMMB_NONE 4         /* no candidate */
#define AMB_COMMB_MAX 600

/* ADS-B operational status, target state and position integrity (amb_decoder_set_option(d, "opstatus", S), S in
 * 1..600 seconds). The parser has no handler for DF17 type codes 29 and 31; with the option on, the queued DF17 records
 * below are decoded. ME bits are numbered 1..56 (ME bit k = message bit 32 + k); t = secs + frac. DF18 is not touched.
 *   TC 31, ME 6-8 subtype 0 (airborne) or 1 (surface), version ME 41-43 in 0..2: AMB_ES_OPSTATUS (aircraft operational
 *         status, BDS6,5); any other subtype or version: AMB_ES_UNSUPPORTED.
 *   TC 29, ME 6-7 = 1: AMB_ES_TARGET_STATE (target state and status, BDS6,2, version 2); subtypes 0, 2, 3:
 *         AMB_ES_UNSUPPORTED.
 *   BDS0,5 (TC 9-18 but 15) and BDS0,6 (TC 5-8), with or without a fix: A = the latest earlier AMB_ES_OPSTATUS record of
 *         the same icao (either subtype, in stream order, since amb_decoder_reset), counted when 0 <= t - t_A <= S;
 *         C = the same over surface ones. Version (of A) 1 or 2: AMB_ES_NIC with NIC and Rc from DESIGN.md §8's tables
 *         by type code and supplements: NIC-A from A; NIC-B = ME 8 of an airborne position for version 2, NIC-A for
 *         version 1; NIC-C from C for version 2 (0 when C does not count), 0 for version 1, where surface TC 8 is NIC 0
 *         with Rc unknown. A combination the tables do not list is NIC 0, Rc unknown. Version 0 or no A: AMB_ES_NUC,
 *         NUCp by type code (airborne 18 - TC, surface 14 - TC), Rc unknown.
 * Status stays AMB_FS_NO_HANDLER for TC 29 / 31. The option writes only aux and bytes 5..7 of pad_ of these records
 * (every other DF17 record keeps aux = 0 and pad_ bytes 5..7 = 0): */
#define AMB_FIELDS_ES(r) (((uint8_t*)&(r)->pad_)[5])          /* outcome, AMB_ES_* */
#define AMB_FIELDS_ES_VERSION(r) (((uint8_t*)&(r)->pad_)[6])  /* TC 31: its version (ME 41-43); TC 29 subtype 1: 2;
                                                                 position: A's version; else AMB_ES_NO_VERSION */
#define AMB_FIELDS_ES_NIC(r) (((uint8_t*)&(r)->pad_)[7])      /* position: NIC (AMB_ES_NIC) or NUCp (AMB_ES_NUC); else 0 */
#define AMB_ES_NOT_TRIED 0       /* option off, or not one of the records above */
#define AMB_ES_OPSTATUS 1        /* TC 31 decoded into aux */
#define AMB_ES_TARGET_STATE 2    /* TC 29 subtype 1 decoded into aux */
#define AMB_ES_NIC 3             /* position with NIC and Rc */
#define AMB_ES_NUC 4             /* position with NUCp only (version 0, or no op status within S) */
#define AMB_ES_UNSUPPORTED 5     /* TC 31 of another subtype or version, TC 29 of another subtype: aux is 0 */
#define AMB_ES_NO_VERSION 0xff
#define AMB_OPSTATUS_MAX 600
/* aux of AMB_ES_OPSTATUS (raw fields; version 0 has another layout: only SUBTYPE, CC and OM are written, the rest is 0) */
#define AMB_FIELDS_OPS_CC(r) (((uint16_t*)(r)->aux)[0])        /* capability class, ME 9-24 */
#define AMB_FIELDS_OPS_OM(r) (((uint16_t*)(r)->aux)[1])        /* operational mode, ME 25-40 */
#define AMB_FIELDS_OPS_SUBTYPE(r) (((uint8_t*)(r)->aux)[4])    /* 0 airborne, 1 surface */
#define AMB_FIELDS_OPS_NIC_A(r) (((uint8_t*)(r)->aux)[5])      /* ME 44 */
#define AMB_FIELDS_OPS_NACP(r) (((uint8_t*)(r)->aux)[6])       /* ME 45-48 */
#define AMB_FIELDS_OPS_GVA(r) (((uint8_t*)(r)->aux)[7])        /* ME 49-50 */
#define AMB_FIELDS_OPS_SIL(r) (((uint8_t*)(r)->aux)[8])        /* ME 51-52 */
#define AMB_FIELDS_OPS_NIC_BARO(r) (((uint8_t*)(r)->aux)[9])   /* ME 53: NICbaro (airborne), TRK/HDG (surface) */
#define AMB_FIELDS_OPS_HRD(r) (((uint8_t*)(r)->aux)[10])       /* ME 54 */
#define AMB_FIELDS_OPS_SIL_SUPP(r) (((uint8_t*)(r)->aux)[11])  /* ME 55 */
#define AMB_FIELDS_OPS_NIC_C(r) (((uint8_t*)(r)->aux)[12])     /* surface: ME 20 (last capability-class bit); else 0 */
#define AMB_FIELDS_OPS_LW(r) (((uint8_t*)(r)->aux)[13])        /* surface: length/width code ME 21-24; else 0 */
/* aux of AMB_ES_TARGET_STATE (raw fields) */
#define AMB_FIELDS_TS_ALT(r) (((uint16_t*)(r)->aux)[0])        /* selected altitude ME 10-20: 0 no data, else (n-1) * 32 ft */
#define AMB_FIELDS_TS_BARO(r) (((uint16_t*)(r)->aux)[1])       /* baro setting ME 21-29: 0 no data, else 800 + (n-1) * 0.8 mb */
#define AMB_FIELDS_TS_HDG(r) (((uint16_t*)(r)->aux)[2])        /* selected heading ME 31-39 (sign included): n * 180/256 deg */
#define AMB_FIELDS_TS_SIL_SUPP(r) (((uint8_t*)(r)->aux)[6])    /* ME 8 */
#define AMB_FIELDS_TS_ALT_TYPE(r) (((uint8_t*)(r)->aux)[7])    /* ME 9: 0 MCP/FCU, 1 FMS */
#define AMB_FIELDS_TS_HDG_STATUS(r) (((uint8_t*)(r)->aux)[8])  /* ME 30: 1 = the heading is valid */
#define AMB_FIELDS_TS_NACP(r) (((uint8_t*)(r)->aux)[9])        /* ME 40-43 */
#define AMB_FIELDS_TS_NIC_BARO(r) (((uint8_t*)(r)->aux)[10])   /* ME 44 */
#define AMB_FIELDS_TS_SIL(r) (((uint8_t*)(r)->aux)[11])        /* ME 45-46 */
#define AMB_FIELDS_TS_MODES(r) (((uint8_t*)(r)->aux)[12])      /* ME 47 (bit 7) .. ME 54 (bit 0): AMB_TS_* */
#define AMB_TS_MODE_STATUS 0x80  /* ME 47: the mode bits below (but TCAS) are valid */
#define AMB_TS_AUTOPILOT 0x40
#define AMB_TS_VNAV 0x20
#define AMB_TS_ALT_HOLD 0x10
#define AMB_TS_APPROACH 0x04     /* 0x08 is ME 51, reserved */
#define AMB_TS_TCAS 0x02         /* TCAS/ACAS operational */
#define AMB_TS_LNAV 0x01
/* aux of AMB_ES_NIC / AMB_ES_NUC (a position): the supplements used (0 where unused, all 0 for NUC) and Rc */
#define AMB_FIELDS_POS_NIC_A(r) (((uint8_t*)(r)->aux)[0])
#define AMB_FIELDS_POS_NIC_B(r) (((uint8_t*)(r)->aux)[1])      /* airborne only */
#define AMB_FIELDS_POS_NIC_C(r) (((uint8_t*)(r)->aux)[2])      /* surface, version 2 only */
#define AMB_FIELDS_POS_RC(r) (((float*)(r)->aux)[1])           /* containment radius, metres; NaN = unknown */

/* Per-aircraft state table (amb_decoder_set_option(d, "track", S), S in 1..3600 seconds): every decode also folds its
 * records, in stream order, into one row per 24-bit address, kept on the device. A record counts when its status has
 * neither AMB_FS_NOT_QUEUED nor AMB_FS_NO_HANDLER; a = its icao field, t = secs + frac of its frame.
 *   expiry    a row whose seen lies more than S before t (t - seen > S) counts as absent;
 *   creation  without a live row, a DF17 record creates one (every column blank, first_seen = t, messages = 0); any
 *             other record is ignored;
 *   apply     messages += 1, seen = t, ref_level = the frame's; altitude from DF0/4/16/20 and BDS0,5 when it is not
 *             AMB_NO_ALTITUDE; BDS0,5 clears AMB_AC_ON_GROUND (with or without an altitude), BDS0,6 sets altitude 0
 *             and AMB_AC_ON_GROUND; squawk from DF5/21; ident,
 *             ftc, cat from BDS0,8; lat, lon, pos_t = t from a record with AMB_FS_HAS_POS (range / bearing with
 *             AMB_FS_HAS_RANGE, else NaN); speed, heading, vertical = val[0..2] of BDS0,9 subtypes 0 and 1; heading =
 *             val[0] of BDS0,6; eps from BDS6,1. Nothing else changes a row.
 * A column whose flag is clear holds NaN, AMB_NO_ALTITUDE or -1 (ident: 8 zero bytes). Every column is a copy of a
 * record or frame value, so a row does not depend on how the stream is cut into calls. */
#define AMB_AC_HAS_ALT 0x001
#define AMB_AC_HAS_SQUAWK 0x002
#define AMB_AC_HAS_IDENT 0x004       /* ident, ftc, cat */
#define AMB_AC_HAS_POS 0x008         /* lat, lon, pos_t */
#define AMB_AC_HAS_RANGE 0x010       /* range, bearing of that position (receiver location known) */
#define AMB_AC_HAS_VELOCITY 0x020    /* speed, vertical */
#define AMB_AC_HAS_HEADING 0x040
#define AMB_AC_HAS_EPS 0x080
#define AMB_AC_ON_GROUND 0x100       /* the last BDS0,5 / BDS0,6 was a surface report */
#define AMB_TRACK_MAX 3600

typedef struct amb_aircraft {
    uint32_t icao;        /* the 24-bit address */
    uint32_t messages;    /* records applied since the row was created */
    double first_seen;    /* t of the DF17 record that created the row */
    double seen;          /* t of the last record applied */
    float ref_level;      /* that record's frame ref_level; rssi = 10 log10(max(1e-8, ref_level)) (parse.py:430) */
    uint16_t flags;       /* AMB_AC_* */
    int8_t ftc, cat;      /* BDS0,8 type code 1..4 and category */
    char ident[8];        /* BDS0,8 callsign, no terminator */
    int32_t altitude;     /* feet */
    int32_t squawk;
    double lat, lon;      /* degrees */
    double range, bearing;/* statute miles, degrees, from the receiver location */
    double pos_t;         /* t of the record that gave the position */
    double speed, heading, vertical;   /* knots, degrees, feet per minute */
    int8_t eps;           /* BDS6,1 emergency/priority status */
    uint8_t pad_[15];     /* 0 */
} amb_aircraft;           /* 128 bytes */

/* Extension of the per-aircraft table (amb_decoder_set_option(d, "track_ext", S2), S2 in 1..3600 seconds; it has an
 * effect only while "track" is on too): what the "opstatus" and "commb" options write into the records, kept per
 * address in six groups. A group holds a copy of the latest record, in stream order, that writes it; its time is that
 * record's t = secs + frac. Every record writes at most one group; a = its icao field:
 *   OPS    a queued record with AMB_FIELDS_ES == AMB_ES_OPSTATUS (needs "opstatus"): aux and its version byte;
 *   TS     AMB_FIELDS_ES == AMB_ES_TARGET_STATE (needs "opstatus"): aux;
 *   INTEG  AMB_FIELDS_ES == AMB_ES_NIC or AMB_ES_NUC, and AMB_FS_HAS_POS (needs "opstatus"): aux[0..1], the outcome,
 *          version and NIC bytes. With "opstatus" on from the start, every position the base row takes is rated, so a
 *          shown INTEG group comes from the record that gave the row its position: t[INTEG] == pos_t;
 *   B40 / B50 / B60  AMB_FIELDS_COMMB == AMB_COMMB_DECODED or AMB_COMMB_RESOLVED with register 0x40 / 0x50 / 0x60
 *          (needs "commb"): the five raw fields, the status mask and the outcome.
 * A snapshot (amb_decoder_aircraft_ext) returns exactly the rows amb_decoder_aircraft would, and beside each row its
 * extension, in which a group is shown when t >= the row's first_seen (it arrived while this row existed), t <= now and
 * now - t <= S2. A group that is not shown has t = NaN and every byte of its fields 0, so snapshots compare byte for
 * byte. amb_decoder_reset forgets every group. */
#define AMB_AXG_OPS 0x01
#define AMB_AXG_TS 0x02
#define AMB_AXG_INTEG 0x04
#define AMB_AXG_B40 0x08
#define AMB_AXG_B50 0x10
#define AMB_AXG_B60 0x20
#define AMB_AXG_N 6              /* group i has bit 1 << i and time t[i] */
#define AMB_TRACK_EXT_MAX 3600

typedef struct amb_aircraft_ext {
    uint32_t icao;        /* the row's address */
    uint8_t shown;        /* AMB_AXG_* of the groups shown */
    uint8_t ops_version;  /* OPS: AMB_FIELDS_ES_VERSION of its record */
    uint8_t integ_es;     /* INTEG: AMB_FIELDS_ES of its record (AMB_ES_NIC / AMB_ES_NUC) */
    uint8_t integ_version;/* INTEG: AMB_FIELDS_ES_VERSION of its record */
    double t[6];          /* t of each group's record, by group index; NaN when not shown */
    uint32_t ops[4];      /* OPS: the record's aux, byte for byte (AMB_AXG_OPS_BYTE) */
    uint32_t ts[4];       /* TS: the record's aux, byte for byte (AMB_AXG_TS_BYTE) */
    uint32_t integ[2];    /* INTEG: aux[0..1] of the record (AMB_AXG_INTEG_BYTE, AMB_AXG_INTEG_RC) */
    uint8_t integ_nic;    /* INTEG: AMB_FIELDS_ES_NIC of its record */
    uint8_t commb_mask[3];/* B40 / B50 / B60: AMB_FIELDS_COMMB_MASK of its record */
    uint8_t commb_outcome[3]; /* B40 / B50 / B60: AMB_FIELDS_COMMB of its record */
    uint8_t pad0_;        /* 0 */
    int16_t commb[3][5];  /* B40 / B50 / B60: AMB_FIELDS_COMMB_RAW(0..4) of its record */
    uint8_t pad_[10];     /* 0 */
} amb_aircraft_ext;       /* 144 bytes */
/* The groups' payloads at the byte offsets the record macros use (x is an amb_aircraft_ext*): byte i of OPS is
 * ((uint8_t*)aux)[i] of its record, so AMB_FIELDS_OPS_NACP reads AMB_AXG_OPS_BYTE(x, 6), AMB_FIELDS_TS_MODES
 * AMB_AXG_TS_BYTE(x, 12), AMB_FIELDS_POS_NIC_B AMB_AXG_INTEG_BYTE(x, 1); the 16-bit words likewise. */
#define AMB_AXG_OPS_BYTE(x, i) (((const uint8_t*)(x)->ops)[i])
#define AMB_AXG_OPS_WORD(x, i) (((const uint16_t*)(x)->ops)[i])      /* 0: capability class, 1: operational mode */
#define AMB_AXG_TS_BYTE(x, i) (((const uint8_t*)(x)->ts)[i])
#define AMB_AXG_TS_WORD(x, i) (((const uint16_t*)(x)->ts)[i])        /* 0: selected altitude, 1: baro, 2: heading */
#define AMB_AXG_INTEG_BYTE(x, i) (((const uint8_t*)(x)->integ)[i])   /* 0: NIC-A, 1: NIC-B, 2: NIC-C */
#define AMB_AXG_INTEG_RC(x) (((const float*)(x)->integ)[1])          /* containment radius, metres; NaN = unknown */
#define AMB_AXG_COMMB_RAW(x, g, i) ((x)->commb[g][i])   /* g = 0 (4,0), 1 (5,0), 2 (6,0); raw field i = 0..4 */

/* SBS-1 (BaseStation) feed (amb_decoder_set_option(d, "sbs1", 1)): every decode also writes the lines that the
 * reference's output_sbs1 (python/sbs1.py, modes_rx -P) would send for its records, in record order, continuing across
 * calls since the last amb_decoder_reset. t = secs + frac of the record's frame.
 *   published  a record counts when its frame was queued, its status lacks AMB_FS_NO_HANDLER, its df is 0, 4, 5, 11 or
 *              17 and its icao fits in 24 bits; icao is the address (the AP syndrome for DF0/4/5, AA for DF11/17).
 *   ids        every published record takes an aircraft id before anything else, as get_aircraft_id (sbs1.py:73-90):
 *              with n ids handed out since the reset, the address's id is live when it was assigned since the reset and
 *              id > n - 10000; a live id is reused, otherwise the record gets n + 1 (the first id after a reset is 1).
 *   lines      MSG,7 (DF0), MSG,5 (DF4), MSG,6 (DF5), MSG,8 (DF11), MSG,1 (BDS0,8), MSG,2 (BDS0,6), MSG,3 (BDS0,5),
 *              MSG,4 (BDS0,9 subtype 1), each ending in "\r\n", field for field as pp0 .. pp17 format them (%.5f / %.1f
 *              round the exact binary value half to even, %i of a float truncates). No line, but an id is taken, for
 *              DF0/4 with AMB_FS_METRIC_ALT, BDS0,5 / 0,6 without AMB_FS_HAS_POS (a local fix counts), BDS0,9 subtypes 0
 *              and 3, BDS6,1 and BDS0,8 whose cat is out of range for its ftc.
 *   date/time  from the frame's stamp, not a wall clock: secs += int(frac), frac -= int(frac); milliseconds
 *              max(0, min(999, floor(frac * 1000))) (a negative frac counts as 0); the proleptic Gregorian date of
 *              secs + 60 * sbs1_tz. Outside 1970-01-01 .. 9999-12-31 23:59:59, or for a frac that is not finite, the four
 *              date/time fields are empty.
 * The ids live in a direct-mapped table in device memory (2^24 x 8 B = 128 MiB), allocated at the first decode with the
 * option on; a reset only records where the ids of the new stream begin. A decode with the option on launches ten
 * kernels more; with it off nothing changes. */
#define AMB_SBS1_TZ_MIN (-720)
#define AMB_SBS1_TZ_MAX 840

/* Receiver coverage map (amb_decoder_set_option(d, "coverage", 1)): the model behind the reference's azimuth map
 * (az_map_model, python/az_map.py:35-82, fed by az_map_output.output, az_map.py:187-202): the greatest range heard in
 * each 5-degree bearing sector, separately for nine altitude bands. It folds in the records of this decoder in stream
 * order, continuing across calls, since the last amb_decoder_reset or amb_decoder_coverage_reset:
 *   1 counted   a record counts when its frame was queued, its status lacks AMB_FS_NO_HANDLER, df == 17, bds is 0x05 or
 *               0x06 and it has AMB_FS_HAS_RANGE (the type17_dl messages az_map_output gets a range for). Without a
 *               receiver location nothing counts. A local fix (option "local_cpr") counts like a global one.
 *   2 altitude  BDS0,6 counts as 0 ft; BDS0,5 uses the record's altitude (decode_alt(alt, False); may be negative).
 *   3 cell      row = ((int64)(bearing + 2.5)) / 5 % 72: the sum in IEEE double, truncated, then divided as an integer
 *               (az_map.py:66 with npoints = 72), so the double just below 2.5 lands in row 1, and 357.5 and 360.0 in
 *               row 0. col = the index of the first of AMB_COVERAGE_ALTITUDES >= altitude, or 8 when altitude >= 30000.
 *   4 update    for every band j in col..8: if range > cell[row][j] then cell[row][j] = range. Cells start at +0.0, so
 *               a range of 0 (or a NaN) changes nothing.
 *   5 units     the records' range: statute miles (cpr.py:162). amb_decoder_set_location changes the ranges of later
 *               records and leaves the grid as it is.
 * The grid is AMB_COVERAGE_ROWS x AMB_COVERAGE_BANDS doubles (5184 bytes of device memory, allocated zeroed at the first
 * decode with the option on); row i covers the bearings [5i - 2.5, 5i + 2.5) up to the rounding of rule 3. It is a
 * maximum over a fixed grid, so it does not depend on how the stream is cut into calls. A decode with the option on
 * launches one kernel more; with it off nothing changes. */
#define AMB_COVERAGE_ROWS 72     /* 5-degree bearing sectors, row i centred on 5 i degrees */
#define AMB_COVERAGE_BANDS 9     /* altitude bands, by their upper edge: */
#define AMB_COVERAGE_ALTITUDES {0, 1000, 2000, 5000, 10000, 15000, 20000, 25000, 30000}   /* feet (az_map.py:42) */

/* Text reports (amb_decoder_set_option(d, "reports", 1)): every decode also writes the lines that the reference's stdout
 * printer (air_modes.output_print, python/msprint.py; what apps/modes_rx prints by default) would print for its records.
 * For every frame, in stream order, the line is exactly report.format_report(text, record) + "\n" of
 * gr_air_modes_b200/report.py, where text = amb_format_message(frame, first); where format_report returns None nothing
 * is written. The lines of one call are concatenated in record order. Consequences:
 *   1 printed   frames that were not queued print nothing; AMB_FS_NO_HANDLER prints nothing unless option "commb" gave a
 *               DF20/21 record a register (DECODED / RESOLVED) or option "opstatus" decoded a TC 31 / TC 29 squitter,
 *               which print their own lines; DF0 with AMB_FS_METRIC_ALT or ri in {1, 5, 6, 7, 8}, DF4 with
 *               AMB_FS_METRIC_ALT, DF4/5 with fs 0, 6 or 7, DF16, BDS0,8 whose cat is out of its ftc's row, BDS0,5 / 0,6
 *               without AMB_FS_HAS_POS (a local fix of option "local_cpr" counts), TCAS tti 2 without a threat
 *               altitude and DF20 without an altitude print nothing. The stage runs after every other stage.
 *   2 prefix    "(%i %.8f) " from the message text, not the raw frame: level' = the double nearest to "%.*g" of the
 *               frame's float32 ref_level (precision 6 for the first message, 10 after), rssi = 10 * log10(max(1e-8,
 *               level')) truncated; frac' = the double nearest to "%.10g" of frac, secs' = secs + int(frac'),
 *               frac' -= int(frac'), and "%.8f" of float(secs') + frac'. So the lines are the same whether the frames
 *               came from rx_path or were parsed back from its messages.
 *   3 first     the first queued frame the stage formats after amb_decoder_create or the last amb_decoder_reset takes
 *               precision 6: the stream's first message when the decoder sees the stream from its start. Turning the
 *               option on mid-stream counts from there; turning it off and on again does not restart the count.
 *   4 numbers   as Python's % writes them: %.Nf (N = 0, 1, 2, 3, 6, 8) the exact binary value rounded half to even (the
 *               stamp exact up to secs = 2^64 - 1), %i of a float truncated, %x / %.6x / %04x lower-case hex. The
 *               derived values are report.py / decode.py's fp64 expressions in the same order, without contraction. A
 *               NaN level prints -80; a +inf level, a frac that is not finite or |frac| >= 2^64, and a body number
 *               %.Nf / %i cannot hold below 2^63 write no line (Python raises, or prints what the receiver never
 *               writes).
 *   5 log10     where level' is a power of ten the rssi is 10 times its exponent; elsewhere 10 * log10(level') lies far
 *               from an integer for every float32 level, so the device's log10 truncates as CPython's does.
 * One flag word (the first message) and, per frame of capacity, 4 + 478 bytes plus 12 bytes per 128 frames, allocated
 * at the first decode with the option on. A decode with the option on launches three kernels more; with it off
 * nothing changes. */

/* Beast binary and AVR raw feeds (amb_decoder_set_option(d, "beast", 1), amb_decoder_set_option(d, "avr", 1 or 2)):
 * every decode also writes its frames in the two wire formats dump1090 and readsb exchange raw frames in (Beast on TCP
 * port 30005, AVR on 30002), what mlat-client and the other consumers of a receiver's raw frames read.
 *   1 frames     a frame is written when its record lacks AMB_FS_NOT_QUEUED (frame.passed != 0), whatever its df and
 *                status, AMB_FS_NO_HANDLER and DF20/21 Comm-B included; a frame fixed by option "ec" or "ec_any" with
 *                its corrected data. The payload is data[0 .. nbits / 8): 14 bytes when nbits is 112, else 7 (nbits is
 *                56 or 112 for every frame the slicer passes). The messages of one call are concatenated in record
 *                order; nothing carries from call to call, so any cut of a stream into calls gives the same bytes.
 *   2 timestamp  T = (secs * 12000000 + (uint64)(int64)rint(frac * 12e6)) mod 2^48: a 48-bit count at 12 MHz from the
 *                frame's stamp, not a wall clock, in uint64 wraparound arithmetic (exact mod 2^48). frac * 12e6 is one
 *                fp64 multiply without contraction, rint rounds half to even. T = 0 when frac is not finite or
 *                |frac * 12e6| >= 2^62. With no start time rx_path stamps a frame sample_index / rate, so T is a
 *                free-running sample clock; with a shared rx_time start, synchronized receivers give the same T for the
 *                same instant, as multilateration needs.
 *   3 signal     S from v = (double)ref_level, a power (the mean of four preamble samples of the PMF'd |x|^2): 0 when v
 *                is NaN or v <= 0, 255 when v >= 1, else max(1, (int)rint(255.0 * sqrt(v))); (S / 255)^2 is the power.
 *   4 Beast      0x1a, the type byte '2' (0x32) for 7 payload bytes or '3' (0x33) for 14, T in 6 bytes big-endian, S,
 *                the payload; every 0x1a after the type byte is written twice. At most 2 + 2 * 21 = 44 bytes.
 *   5 AVR        avr = 1: "*", the payload in upper-case hex, ";\n". avr = 2: "@", T in 12 upper-case hex digits, the
 *                payload's hex, ";\n". Fixed length for a payload length: 17 / 31 bytes (avr 1), 29 / 43 (avr 2).
 * Per frame of capacity, 4 + 44 bytes (Beast) and 4 + 43 bytes (AVR) plus 12 bytes per 128 frames each, allocated at
 * the first decode with the option on. A decode launches three kernels more per option that is on; with both off
 * nothing changes. */

/* FlightGear multiplayer feed (amb_decoder_set_option(d, "flightgear", 1)): every decode also writes the position
 * packets that the reference's output_flightgear (python/flightgear.py, modes_rx -m HOST:PORT) would send by UDP for
 * its records, in record order, continuing across calls since the last amb_decoder_reset. t = secs + frac of the
 * record's frame.
 *   1 published  a record counts when its frame was queued, its status lacks AMB_FS_NO_HANDLER, its df is 17 and its
 *                bds is 0x05, 0x06, 0x08 or 0x09 (the type17_dl messages, flightgear.py:28); icao is the address.
 *   2 callsign   BDS0,8 sets the address's (ident, model): ident = the record's 8 characters; model = modelmap
 *                (flightgear.py:116-132) of categories[ftc - 1][cat] (parse.py:270-275), the santa model where modelmap
 *                has no entry (RESERVED, PARACHUTE, the OBSTRUCTIONs). A cat beyond its ftc row (ftc 2, cat 7: the
 *                reference raises IndexError) changes nothing.
 *   3 velocity   BDS0,9 subtype 0 sets (heading, velocity, turn rate) = (val[1], val[0], val[3]); subtype 1 sets
 *                (val[1], val[0], 0); subtype 3 changes nothing.
 *   4 packet     BDS0,5 with AMB_FS_HAS_POS gives (lat, lon, altitude), BDS0,6 with it (lat, lon, 0); a local fix
 *                (option "local_cpr") counts. When the address has had a callsign and a velocity since the reset (in
 *                this call or an earlier one), the record writes one packet with the latest of each. Callsign and
 *                velocity records write none. No packet either where the reference raises TypeError: the half angle
 *                of the orientation has sin < 1e-12 (e.g. lat -90, lon 0, heading 0 or 360).
 *   5 bytes      232, big-endian: "FGFS", 0x00010001, msgid 7, msglen 232, 0, 0, ident (8 bytes); the model path
 *                NUL-padded to 96 bytes; t and 0.0 as doubles (the reference's time.time() replaced by the frame's
 *                stamp); llh2ecef(lat, lon, alt * 0.3048) (mlat.py:75-86) as three doubles; the orientation as three
 *                floats; (float)(velocity * 0.514444444), 0, 0; 0, 0, (float)(turn rate * (pi / 180.)); six zero
 *                floats and a zero uint32.
 *   orientation  angle * axis of Quat([lat, lon]) * Quat([heading, 0, 0]) (Quaternion.py), each IEEE double operation
 *                in the reference's order, then rounded to float. With P = pi / 180.:
 *                  a = (-S zd * S yd, C zd * S yd, S zd * C yd, C zd * C yd), zd = 0.5 * (lon * P),
 *                      yd = -0.25 * pi - 0.5 * (lat * P), S = sin, C = cos (_latlontoquat);
 *                  ra = heading * (pi / 180.0), dec = roll = 0.0 * (pi / 180.0); T = the matrix of
 *                      _equatorial2transform with its products as written (T00 = ca * cd, T10 = -ca * sd * sr - sa * cr,
 *                      ...); den = (1 + T00 - T11 - T22, 1 - T00 + T11 - T22, 1 - T00 - T11 + T22, 1 + T00 + T11 + T22);
 *                      m = the first index of the largest den; b[m] = 0.5 * sqrt(den[m]), the other three from the
 *                      off-diagonal sums over 4 b[m] (_transform2quat);
 *                  q = a * b (the product of Quaternion.py:393-415, left to right), then q = -q unless q[3] > 0;
 *                  norm = sqrt(((q0^2 + q1^2) + q2^2) + q3^2), rnorm = 1 / norm, angle = acos(clamp(rnorm * q3, -1, 1)),
 *                      s = sin(angle); orientation_i = (float)((2 * angle) * ((rnorm / s) * q_i)).
 * The latest callsign and velocity of every address live in a direct-mapped table in device memory (2^24 x 32 B =
 * 512 MiB), allocated at the first decode with the option on and cleared by amb_decoder_reset; per frame of capacity
 * 32 + 4 + 232 bytes plus 12 bytes per 128 frames. A decode with the option on launches nine kernels more; with it off
 * nothing changes. */
typedef struct amb_decoder amb_decoder;
/* cpr_decoder(my_location) (cpr.py:184-190) + the parser; have_location = 0 is my_location = None. */
AMB_API int amb_decoder_create(int device, int have_location, double lat, double lon, amb_decoder** out);
/* "local_cpr": S = 0 (default, off) .. 600 seconds, locally referenced CPR decode (see AMB_FIELDS_LOCAL); applies from
 * the next call. The table of reference positions (2^24 x 24 B = 384 MiB of device memory) is allocated at the first
 * decode with the option on, written only by such decodes and cleared by amb_decoder_reset. Off changes nothing.
 * "track": S = 0 (default, off) .. 3600 seconds, the per-aircraft table (see amb_aircraft); applies from the next call.
 * Rows are direct-mapped by address: 2^24 x 128 B = 2 GiB of device memory plus a 2 MiB occupancy bitmap, allocated at
 * the first decode with the option on; only the bitmap is cleared (by amb_decoder_reset). A decode with the option on
 * launches six kernels more (13, or 19 with "local_cpr"); with it off nothing changes.
 * "commb": S = 0 (default, off) .. 600 seconds, Comm-B register inference (see AMB_FIELDS_COMMB); applies from the next
 * call. The ADS-B velocity per address (2^24 x 24 B = 384 MiB of device memory) is allocated at the first decode with
 * the option on and cleared by amb_decoder_reset. A decode with the option on launches six kernels more; off changes
 * nothing.
 * "opstatus": S = 0 (default, off) .. 600 seconds, ADS-B op status, target state and position integrity (see
 * AMB_FIELDS_ES); applies from the next call. The latest op status per address (2^24 x 24 B = 384 MiB of device memory)
 * is allocated at the first decode with the option on and cleared by amb_decoder_reset. A decode with the option on
 * launches six kernels more; off changes nothing.
 * "track_ext": S2 = 0 (default, off) .. 3600 seconds, the extension of the per-aircraft table (see amb_aircraft_ext);
 * applies from the next call, and only while "track" is on too. Rows are direct-mapped by address: 2^24 x 144 B =
 * 2.25 GiB of device memory plus a 2 MiB bitmap, allocated at the first decode with both options on; only the bitmap is
 * cleared (by amb_decoder_reset). A decode with both on launches six kernels more; off changes nothing.
 * "sbs1": 0 (default, off) or 1, the SBS-1 feed (see AMB_SBS1_TZ_MIN); applies from the next call.
 * "sbs1_tz": AMB_SBS1_TZ_MIN .. AMB_SBS1_TZ_MAX minutes (default 0, UTC) added to the stamp in the SBS-1 date and time.
 * "coverage": 0 (default, off) or 1, the receiver coverage map (see AMB_COVERAGE_ROWS); applies from the next call.
 * "reports": 0 (default, off) or 1, the text reports (see amb_decoder_reports); applies from the next call.
 * "beast": 0 (default, off) or 1, the Beast binary feed (see amb_decoder_beast); applies from the next call.
 * "avr": 0 (default, off), 1 ("*" lines) or 2 ("@" lines with the timestamp), the AVR raw feed (see amb_decoder_avr);
 * applies from the next call.
 * "flightgear": 0 (default, off) or 1, the FlightGear multiplayer feed (see amb_decoder_flightgear); applies from the
 * next call.
 * Unknown names and out-of-range values return AMB_ERR_INVALID. */
AMB_API int amb_decoder_set_option(amb_decoder* d, const char* name, int value);
/* Snapshot of the per-aircraft table at time `now`: every row with seen <= now and now - seen <= S, in ascending
 * address. now = NaN stands for the t of the latest queued record decoded since the last reset (kept on the device).
 * out == NULL returns the number of rows; a buffer of fewer than that many rows returns AMB_ERR_OVERFLOW and writes
 * nothing. Otherwise returns the number of rows written. AMB_ERR_STATE when the option "track" is off. Three kernel
 * launches (two when nothing is written) and one 4-byte copy to the host; _device writes to device memory. */
AMB_API int amb_decoder_aircraft(amb_decoder* d, double now, amb_aircraft* out, int max);
AMB_API int amb_decoder_aircraft_device(amb_decoder* d, double now, amb_aircraft* out_dev, int cap);
/* The same snapshot with the extension beside it: out[] is byte for byte what amb_decoder_aircraft writes, ext[i] the
 * groups of out[i] shown at `now` (see amb_aircraft_ext). out == NULL returns the number of rows; too small a buffer
 * returns AMB_ERR_OVERFLOW and writes nothing. AMB_ERR_STATE unless both "track" and "track_ext" are on. Three kernel
 * launches (two when nothing is written) and one 4-byte copy to the host; _device writes both arrays to device memory. */
AMB_API int amb_decoder_aircraft_ext(amb_decoder* d, double now, amb_aircraft* out, amb_aircraft_ext* ext, int max);
AMB_API int amb_decoder_aircraft_ext_device(amb_decoder* d, double now, amb_aircraft* out_dev, amb_aircraft_ext* ext_dev,
                                            int cap);
/* The SBS-1 lines of the last decode, concatenated, into out (cap bytes; no terminator); *n_bytes = their length.
 * AMB_ERR_STATE when the option "sbs1" is off; a buffer of fewer than *n_bytes bytes returns AMB_ERR_OVERFLOW with
 * nothing written (out may then be NULL with cap 0). One 8-byte copy to the host, then the text; _device copies the text
 * to device memory instead, so only the byte count crosses PCIe. */
AMB_API int amb_decoder_sbs1(amb_decoder* d, char* out, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_sbs1_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes);
/* The text reports of the last decode, concatenated ("\n" after each line), into out (cap bytes; no terminator);
 * *n_bytes = their length. AMB_ERR_STATE when the option "reports" is off; a buffer of fewer than *n_bytes bytes returns
 * AMB_ERR_OVERFLOW with nothing written (out may then be NULL with cap 0). One 8-byte copy to the host, then the text;
 * _device copies the text to device memory instead, so only the byte count crosses PCIe. */
AMB_API int amb_decoder_reports(amb_decoder* d, char* out, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_reports_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes);
/* The Beast messages (amb_decoder_beast) or AVR lines (amb_decoder_avr) of the last decode, concatenated, into out (cap
 * bytes; no terminator); *n_bytes = their length. AMB_ERR_STATE when the option "beast" / "avr" is off; a buffer of
 * fewer than *n_bytes bytes returns AMB_ERR_OVERFLOW with nothing written (out may then be NULL with cap 0). One 8-byte
 * copy to the host, then the bytes; _device copies them to device memory instead, so only the byte count crosses PCIe. */
AMB_API int amb_decoder_beast(amb_decoder* d, char* out, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_beast_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_avr(amb_decoder* d, char* out, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_avr_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes);
/* The FlightGear position packets of the last decode (232 bytes each, one UDP datagram apiece), concatenated, into out
 * (cap bytes); *n_bytes = their length. AMB_ERR_STATE when the option "flightgear" is off; a buffer of fewer than
 * *n_bytes bytes returns AMB_ERR_OVERFLOW with nothing written (out may then be NULL with cap 0). One 8-byte copy to
 * the host, then the bytes; _device copies them to device memory instead, so only the byte count crosses PCIe. */
AMB_API int amb_decoder_flightgear(amb_decoder* d, char* out, size_t cap, size_t* n_bytes);
AMB_API int amb_decoder_flightgear_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes);
/* The coverage grid, AMB_COVERAGE_ROWS x AMB_COVERAGE_BANDS doubles, row-major (bearing row first, band second), into
 * out (host memory); _device copies it to device memory. All zeros before the first decode with the option on.
 * amb_decoder_coverage_reset clears the grid and nothing else (az_map_model.reset, az_map.py:77-82). All three return
 * AMB_ERR_STATE when the option "coverage" is off. */
AMB_API int amb_decoder_coverage(amb_decoder* d, double* out);
AMB_API int amb_decoder_coverage_device(amb_decoder* d, double* out_dev);
AMB_API int amb_decoder_coverage_reset(amb_decoder* d);
AMB_API void amb_decoder_destroy(amb_decoder* d);
AMB_API int amb_decoder_set_location(amb_decoder* d, int have_location, double lat, double lon);   /* cpr.py:192-193 */
AMB_API int amb_decoder_reset(amb_decoder* d);                      /* forget every stored report, reference position,
                                                                       velocity, op status, aircraft and extension
                                                                       group, SBS-1 id and FlightGear callsign and
                                                                       velocity, and clear the coverage grid */
/* Decode n frames (host or device array, stream order = non-decreasing time). out: n records in host memory.
 * Frames with passed == 0 get AMB_FS_NOT_QUEUED and do not touch the CPR state. */
AMB_API int amb_decode_frames(amb_decoder* d, const amb_frame* frames, int n, int mem_kind, amb_fields* out);
/* The same with frames AND records in device memory: no host copies. */
AMB_API int amb_decode_frames_device(amb_decoder* d, const amb_frame* frames_dev, int n, amb_fields* out_dev);
/* Kernels launched so far / device time in ms of the last amb_decode_frames call (H2D, kernels, D2H). */
AMB_API int amb_decoder_stats(amb_decoder* d, uint64_t* kernel_launches, float* ms_last);
AMB_API const char* amb_decoder_last_error(const amb_decoder* d);   /* d == NULL: why the last amb_decoder_create of this thread failed */
/* data_field.get_bits(start, num) on a frame's payload (parse.py:71-87): host helper for the raw sub-fields that
 * amb_fields does not carry. */
AMB_API uint64_t amb_frame_bits(const amb_frame* f, int start, int num);

/* ---- multilateration (amb_mlat): K synchronized receivers' frames grouped by transmission, each group solved --------
 * The model behind the reference's mlat.py / mlat_client.py, with a formulation that solves physical stamps (the
 * reference's mlat_iter leaves out the reference station's own range, DESIGN.md 8 "Multilateration"). The rules:
 *   stations   K = AMB_MLAT_MIN_STATIONS .. AMB_MLAT_MAX_STATIONS, each at lat, lon (degrees) and height (m above the
 *              WGS84 ellipsoid; no geoid correction). Station k's ECEF s_k is llh2ecef of mlat.py:77-86.
 *   offset     per station, seconds (default 0), subtracted from frac: t = (secs, frac - off_k). It absorbs cable and
 *              front-end delays and the index bias of stations at different rates.
 *   eligible   passed != 0 and either DF 0, 4, 16 or 20 whose AC13 field (message bits 20..32, decode_alt with
 *              bit13 = 1) decodes to feet - not metric, not code 0 - with the address amb_frame.crc; or DF17 TC 9..18
 *              whose 12-bit ME altitude (bit13 = 0) decodes the same way, with the address AA. Nothing else (the solve
 *              needs the altitude). h = feet * 0.3048 m, used as height above the ellipsoid as mlat.py does.
 *   time diff  d(a, b) = (double)(int64)(secs_a - secs_b) + (frac_a - frac_b), never a difference of secs + frac sums.
 *              t orders by the sign of d, ties by station index.
 *   run        the eligible frames of all stations (the carried ones included) sorted by (payload, t, station); a run
 *              is a maximal sequence of identical payloads (nbits and bytes) whose consecutive frames are at most W
 *              apart (d <= W). W = option "window_us" / 1e6 s; default: the largest station-to-station distance / c
 *              plus 2 us.
 *   complete   the call's end stamp promises that every station has delivered every frame with t <= end. A run is
 *              complete when d(end, t_last) >= W or the call has flush set. The frames of incomplete runs are carried
 *              on the device into the next call; the others are dropped after the call. amb_mlat_reset clears the carry.
 *   accepted   a complete run with no station twice (else DUPLICATE), at least 3 frames (else TOO_FEW) and
 *              d(t_last, t_first) <= W (else SPAN) is a group; the others are only counted.
 *   solve      per group, fp64 without contraction. c = 299792458 / 1.0003, a = 6378137, b = 6356752.314245,
 *              e2 = 0.0066943799901975848. Reference station r = the earliest t (ties: lower index); rows follow
 *              ascending station index. x starts at llh2ecef(lat_r, lon_r, h). Rows: for i != r
 *              |x - s_i| - |x - s_r| - c d(t_i, t_r) with gradient (x - s_i)/|x - s_i| - (x - s_r)/|x - s_r|, and the
 *              altitude row |x| - |llh2ecef(lat(x), lon(x), h)| (Bowring's ecef2llh, mlat.py:58-86) with gradient
 *              x/|x|: n = number of stations rows. Each Gauss-Newton step solves J dx = -f by Householder QR
 *              (DESIGN.md 8 writes out the operations). |dx| <= 1e-3 m: SOLVED; 25 steps without: NO_CONVERGENCE; a
 *              diagonal |R_jj| < 1e-9 max |R_jj| (or all zero): DEGENERATE.
 *   fix        one amb_mlat_fix per group, ordered by the reference station's t (ties: lower reference station). rms
 *              and dop = sqrt(trace((J^T J)^-1)) are evaluated at the last x (dop NaN when that J is degenerate).
 * The grouping does not depend on how the streams are cut into calls, as long as every call's end keeps its promise. */
#define AMB_MLAT_MIN_STATIONS 3
#define AMB_MLAT_MAX_STATIONS 32
#define AMB_MLAT_SOLVED 1
#define AMB_MLAT_NO_CONVERGENCE 2
#define AMB_MLAT_DEGENERATE 3
typedef struct amb_mlat amb_mlat;
/* 112 bytes */
typedef struct amb_mlat_fix {
    uint8_t data[14];      /* the payload (nbits / 8 bytes; the rest zero) */
    uint8_t nbits, df;
    uint32_t addr;         /* AA of DF17, the address/parity overlay (amb_frame.crc) of DF0/4/16/20 */
    uint8_t status;        /* AMB_MLAT_* */
    uint8_t n;             /* stations in the group = rows of the solve */
    uint8_t steps;         /* Gauss-Newton steps taken */
    uint8_t ref;           /* the reference station r */
    uint32_t stations;     /* bit k: station k heard it */
    int32_t altitude;      /* feet */
    uint64_t secs;         /* emission time t_r - |x - s_r| / c: secs, and frac normalised to [0, 1) */
    double frac;
    double lat, lon, height;   /* ecef2llh of x: degrees, degrees, m above the ellipsoid */
    double x, y, z;            /* ECEF, m */
    double rms;                /* sqrt(sum f^2 / n) at x, m */
    double dop;                /* sqrt(trace((J^T J)^-1)) at x */
} amb_mlat_fix;
typedef struct amb_mlat_counts {
    uint64_t eligible;         /* eligible frames taken in */
    uint64_t carried;          /* frames carried into the next call now */
    uint64_t solved, no_convergence, degenerate;     /* groups by outcome */
    uint64_t too_few, duplicate, span;               /* complete runs rejected, by reason */
    uint64_t kernel_launches;
    float ms_last;             /* device time of the last call */
    uint32_t pad_;
} amb_mlat_counts;   /* 80 bytes */
/* K stations; lat[k], lon[k] in degrees, height[k] in m above the ellipsoid. */
AMB_API int amb_mlat_create(int device, int K, const double* lat, const double* lon, const double* height, amb_mlat** out);
AMB_API void amb_mlat_destroy(amb_mlat* m);
/* "window_us": W in microseconds, > 0 (a double: W = value / 1e6 s); applies from the next call. */
AMB_API int amb_mlat_set_option(amb_mlat* m, const char* name, double value);
AMB_API int amb_mlat_get_option(amb_mlat* m, const char* name, double* value);
AMB_API int amb_mlat_set_offset(amb_mlat* m, int k, double seconds);   /* applies to the frames of later calls */
AMB_API int amb_mlat_reset(amb_mlat* m);                             /* drop the carried frames */
/* One call: frames[k] holds counts[k] frames of station k in stream order (non-decreasing t), host memory for
 * amb_mlat_process, device memory for amb_mlat_process_device; out holds cap fixes in the same kind of memory.
 * (end_secs, end_frac): see "complete" above; flush = 1 completes every run (end is then not read).
 * Returns AMB_OK with *n_out fixes written. When more than cap fixes are due, returns AMB_ERR_OVERFLOW with *n_out = the
 * number due and changes nothing - carry, counters and kernel_launches stay as they were: call again with a larger
 * buffer. A station whose frames are out of time order returns AMB_ERR_INVALID and changes nothing either. Synchronises the stage's own stream: device frames must be complete when called. */
AMB_API int amb_mlat_process(amb_mlat* m, const amb_frame* const* frames, const int* counts, uint64_t end_secs,
                             double end_frac, int flush, amb_mlat_fix* out, int cap, int* n_out);
AMB_API int amb_mlat_process_device(amb_mlat* m, const amb_frame* const* frames_dev, const int* counts, uint64_t end_secs,
                                    double end_frac, int flush, amb_mlat_fix* out_dev, int cap, int* n_out);
AMB_API int amb_mlat_stats(amb_mlat* m, amb_mlat_counts* out);
AMB_API const char* amb_mlat_last_error(const amb_mlat* m);          /* m == NULL: the last failed amb_mlat_create */

/* ---- Beast binary input (amb_beast_reader): another receiver's frames, parsed on the device -------------------------
 * The byte stream dump1090 and readsb serve on TCP port 30005 (and amb_decoder_beast writes) turned into amb_frame
 * records for amb_decode_frames_device or amb_mlat_process_device. The rules are defined on the byte stream since
 * amb_beast_reader_create or the last amb_beast_reader_reset, not on how it was cut into calls:
 *   1 tokens     left to right, 0x1a 0x1a is one data token (an escaped 0x1a); 0x1a t with t != 0x1a a sync token of
 *                type t; any other byte a data token. The stream's start counts as preceded by a byte that is not 0x1a:
 *                a byte starts a token exactly when the run of 0x1a bytes right before it has even length.
 *   2 messages   a sync token of type '1' (Mode A/C), '2' (Mode S short) or '3' (Mode S long) takes the next 9, 14 or 21
 *                data tokens as its body: T (6 bytes, big-endian), S, then 2, 7 or 14 payload bytes. When a sync token
 *                comes first the message is truncated: dropped and counted, its data tokens with it. Data tokens after a
 *                complete body and before the next sync token, before the first sync token, and after a sync token of
 *                any other type ('4' included; counted as "other") are skipped and counted. Mode A/C messages are
 *                counted and give no frame.
 *   3 frames     every complete Mode S message gives one amb_frame, in stream order: data = the payload zero-padded to
 *                14 bytes, nbits 56 or 112 from the type, df = data[0] >> 3, crc = the slicer's syndrome
 *                amb_modes_check_crc(data, nbits / 8 - 3) ^ the last 3 payload bytes, secs = T / 12000000,
 *                frac = (double)(T % 12000000) / 12e6 (one IEEE division), ref_level = (float)((double)(S * S) / 65025.0),
 *                sample_index = the stream offset of the message's sync byte; numlowconf, lowconfbits, ec, ec_flips and
 *                pad_ are 0. These invert rules 2 to 4 of amb_decoder_beast: T and S of a frame written by it read back
 *                unchanged.
 *   4 passed     1 unless the payload is all zero, or nbits is not 112 for DF 16, 17, 20, 21 and 56 for the others, or
 *                crc != 0 for DF 11 or 17 (the reference slicer's drop rules that need no samples). Unpassed frames are
 *                still written, as amb_drain_device writes them; the decoder marks them AMB_FS_NOT_QUEUED.
 *   5 calls      any cut of a stream into calls, flush on the last, gives the same frames and counters as one call. What
 *                cannot be decided yet (an incomplete last message, a final lone 0x1a: at most AMB_BEAST_CARRY_MAX bytes)
 *                is carried on the device to the next call. At flush an incomplete message is truncated and a final lone
 *                0x1a is dropped uncounted; later calls return AMB_ERR_STATE until amb_beast_reader_reset. */
#define AMB_BEAST_CARRY_MAX 43
#define AMB_BEAST_PUSH_MAX ((size_t)0x7FFF0000)   /* bytes in one call: every index of the call fits an int */
typedef struct amb_beast_reader amb_beast_reader;
typedef struct amb_beast_counts {
    uint64_t bytes_in;         /* bytes given since create or reset */
    uint64_t modes;            /* complete Mode S messages (= frames) */
    uint64_t modeac;           /* complete Mode A/C messages */
    uint64_t other;            /* sync tokens of any other type */
    uint64_t truncated;        /* Mode S and Mode A/C messages cut by a sync token or by flush */
    uint64_t skipped;          /* data tokens outside every message body */
    uint64_t passed;           /* frames with passed = 1 */
    uint64_t carried;          /* bytes carried into the next call now */
    uint64_t kernel_launches;  /* since create: five per call */
} amb_beast_counts;   /* 72 bytes */
AMB_API int amb_beast_reader_create(int device, amb_beast_reader** out);
AMB_API void amb_beast_reader_destroy(amb_beast_reader* r);
/* Start a new stream: drop the carry, offsets and counters (but kernel_launches) restart at 0, flush is undone. */
AMB_API int amb_beast_reader_reset(amb_beast_reader* r);
/* The next n bytes of the stream: host memory (AMB_MEM_HOST, copied once to the device) or device memory
 * (AMB_MEM_DEVICE, read in place; it must be complete when called). flush != 0 ends the stream. Returns this call's frame
 * count; they stay readable until the next call or reset. n > AMB_BEAST_PUSH_MAX or another memory kind:
 * AMB_ERR_INVALID. Five kernel launches whatever n is; only the frame count crosses PCIe. Synchronises the reader's
 * own stream. */
AMB_API int amb_beast_reader_push(amb_beast_reader* r, const void* bytes, size_t n, int mem_kind, int flush);
/* The frames of the last push into out (host memory; _device: device memory), as amb_drain_device writes them:
 * out == NULL returns their count; cap below it returns AMB_ERR_OVERFLOW and writes nothing; else returns the count. */
AMB_API int amb_beast_reader_frames(amb_beast_reader* r, amb_frame* out, int cap);
AMB_API int amb_beast_reader_frames_device(amb_beast_reader* r, amb_frame* out_dev, int cap);
AMB_API int amb_beast_reader_stats(amb_beast_reader* r, amb_beast_counts* out);
AMB_API const char* amb_beast_reader_last_error(const amb_beast_reader* r);   /* r == NULL: the last failed create */

AMB_API const char* amb_strerror(int code);
AMB_API const char* amb_last_error(const amb_ctx* ctx);
AMB_API const char* amb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* AIRMODES_B200_H */
