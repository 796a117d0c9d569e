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
    uint8_t pad_[6];
} amb_frame;                 /* 80 bytes */

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
    int reserved_;
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
AMB_API int amb_set_option(amb_ctx* ctx, const char* name, int value); /* "resolver": 0 auto, 1 sequential, 2 parallel */
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
    double lat, lon;      /* global CPR decode (cpr.py:89-153), degrees; NaN unless AMB_FS_HAS_POS */
    double range, bearing;/* range_bearing(my_location, position) (cpr.py:158-181): statute miles, degrees */
    double val[4];        /* BDS0,9-0: velocity, heading, vert_spd, turn_rate (parse.py:288-313)
                             BDS0,9-1: velocity, heading, vert_spd, alt_geo_diff (parse.py:315-348)
                             BDS0,9-3: mag_hdg, vel, vert_spd, geo_diff (parse.py:350-364)
                             BDS0,6  : ground_track (parse.py:283) */
    uint64_t pad_;
} amb_fields;             /* 144 bytes */

typedef struct amb_decoder amb_decoder;
/* cpr_decoder(my_location) (cpr.py:184-190) + the parser; have_location = 0 is my_location = None. */
AMB_API int amb_decoder_create(int device, int have_location, double lat, double lon, amb_decoder** out);
AMB_API void amb_decoder_destroy(amb_decoder* d);
AMB_API int amb_decoder_set_location(amb_decoder* d, int have_location, double lat, double lon);   /* cpr.py:192-193 */
AMB_API int amb_decoder_reset(amb_decoder* d);                      /* forget every stored report */
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

AMB_API const char* amb_strerror(int code);
AMB_API const char* amb_last_error(const amb_ctx* ctx);
AMB_API const char* amb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* AIRMODES_B200_H */
