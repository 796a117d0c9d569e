// TEST HARNESS (not a product path): runs the decoder's kernel source - gr_air_modes_b200/csrc/amb_decode_kernels.cuh
// and the stage headers it includes - on the host under tests/simt/simt_emul.h, with the decoder's own state, options,
// launch sequence and read-outs: amb_decode_set_option / amb_decode_set_location set what amb_decoder_set_option /
// amb_decoder_set_location set, amb_decode_prepare allocates what the stages that are on need (host memory here),
// amb_decode_launch enqueues fields, pairing, resolve and every stage that is on, amb_decode_text, amb_decode_snapshot_*
// and amb_decode_coverage read the results out, and amb_decode_reset / amb_decode_free are what amb_decoder_reset /
// amb_decoder_destroy run. The tests/test_*_simt.py modules build it with plain g++ and bind it through
// tests/emul_build.py.
#include "simt_emul.h"

#include "../../gr_air_modes_b200/csrc/amb_decode_kernels.cuh"

#include <algorithm>

struct Emul {
    AmbDecodeState st;                                  // kept across calls, like the decoder's
};

// The pairing table and the local stage's table hold 2^log2_slots entries (the tests keep the position squitters'
// addresses small); every other table spans all 2^24 addresses like the decoder's.
extern "C" void* emul_new(int log2_slots)
{
    Emul* e = new Emul();
    e->st.table_slots = e->st.local_slots = (size_t)1 << log2_slots;
    cudaError_t err = cudaSuccess;
    if (amb_decode_prepare(&e->st, 0, nullptr, &err) < 0) { amb_decode_free(&e->st); delete e; return nullptr; }
    return e;
}

extern "C" void emul_free(void* h)
{
    Emul* e = static_cast<Emul*>(h);
    amb_decode_free(&e->st);
    delete e;
}

extern "C" void emul_reset(void* h)
{
    cudaError_t err = cudaSuccess;
    amb_decode_reset(&static_cast<Emul*>(h)->st, nullptr, &err);
}

// amb_decoder_set_option, from the next emul_decode on: returns 0, or -1 when the setting is refused
extern "C" int emul_set_option(void* h, const char* name, int value)
{
    return amb_decode_set_option(&static_cast<Emul*>(h)->st, name, value) ? -1 : 0;
}

extern "C" void emul_set_location(void* h, int have_location, double lat, double lon)
{
    amb_decode_set_location(&static_cast<Emul*>(h)->st, have_location, lat, lon);
}

// amb_decode_frames: returns 0, -1 when a position squitter's address does not fit the test's tables, -2 when a stage
// fails to launch, -3 when the stages' memory cannot be had
extern "C" int emul_decode(void* h, const amb_frame* frames, int n, amb_fields* out)
{
    AmbDecodeState& st = static_cast<Emul*>(h)->st;
    if (n <= 0) return 0;
    for (int k = 0; k < n; k++) {
        amb_fields r; AmbPosRec p;
        amb_decode_fields(frames[k], &r, &p);
        if (p.key != AMB_NO_KEY && (((size_t)p.key << 1) | 1u) >= st.table_slots) return -1;   // test table too small
    }
    const bool had_rows = st.trows, had_xrows = st.xrows;
    cudaError_t err = cudaSuccess;
    if (amb_decode_prepare(&st, n, nullptr, &err) < 0) return -3;
    // rows are never cleared: the first ones start as garbage
    if (!had_rows && st.trows) memset(st.trows, 0xA5, 4096 * 4);
    if (!had_xrows && st.xrows) memset(st.xrows, 0xA5, 4096 * 4);
    if (st.sbs1 > 0) {                                  // the SBS-1 scratch poisoned before every call: no kernel may
        AmbSbs1Bufs& b = st.sb;                         // read what an earlier call left there
        const size_t c = (size_t)st.scap, nb = (c + 127) / 128, chunks = (c + AMB_SBS1_CHUNK - 1) / AMB_SBS1_CHUNK;
        std::fill_n(b.src, c, 0xDEADBEEFull); std::fill_n(b.gid, c, 0xDEADBEEFull);
        std::fill_n(b.flag, chunks, 0xDEADBEEFull);
        memset(b.slots, '?', c * AMB_SBS1_STRIDE); memset(b.text, '?', c * AMB_SBS1_STRIDE);
        std::fill_n(b.len, c, 7u); std::fill_n(b.bsum, nb, 7u); std::fill_n(b.boff, nb + 1, 7ull);
    }
    return amb_decode_launch(&st, frames, n, out, nullptr, &err) < 0 ? -2 : 0;
}

// amb_decoder_aircraft (ext == NULL) or amb_decoder_aircraft_ext over the first `words` bitmap words (a multiple of
// AMB_SNAP_WORDS): out == NULL returns the count, too small a `max` -5.
extern "C" int emul_snapshot(void* h, double now, unsigned words, amb_aircraft* out, amb_aircraft_ext* ext, int max)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    if (!st.tocc) return 0;                             // nothing decoded with the track stage on yet
    cudaError_t err = cudaSuccess;
    const int total = amb_decode_snapshot_count(&st, now, words, nullptr, &err);
    if (total < 0) return -1;
    if (!out) return total;
    if (total > max) return -5;
    if (total == 0) return 0;
    return amb_decode_snapshot_gather(&st, now, words, out, ext, nullptr, &err) < 0 ? -1 : total;
}

// amb_decoder_reports (reports = 1) or amb_decoder_sbs1 (0): the last decode's packed lines into text; returns 0, or -5
// when they do not fit `cap` (*n_bytes = their length either way)
extern "C" int emul_text(void* h, int reports, char* text, size_t cap, size_t* n_bytes)
{
    const char* src = nullptr;
    unsigned long long total = 0;
    amb_decode_text(&static_cast<Emul*>(h)->st, reports != 0, nullptr, &src, &total);
    *n_bytes = (size_t)total;
    if (total > cap) return -5;
    if (total) memcpy(text, src, total);
    return 0;
}

// the ids of the last call's published records, in stream order (count returned)
extern "C" int emul_sbs1_ids(void* h, const amb_fields* recs, int n, unsigned long long* ids)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    int m = 0;
    for (int k = 0; k < n; k++)
        if (amb_sbs1_published(&recs[k])) ids[m++] = st.sb.gid[k] - st.sctr->base;
    return m;
}

// amb_decoder_coverage: the grid into out (AMB_COVERAGE_CELLS doubles); returns whether the grid is allocated
extern "C" int emul_coverage(void* h, double* out)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    amb_decode_coverage(&st, out, false, nullptr);
    return st.cgrid != nullptr;
}

// the coverage stage alone (amb_coverage_launch) over n given records, into the decoder's grid (allocated by
// amb_decode_prepare with the option on): for records whose range and bearing a test chooses; returns 0, or -2 / -3
extern "C" int emul_coverage_records(void* h, const amb_fields* recs, int n)
{
    AmbDecodeState& st = static_cast<Emul*>(h)->st;
    st.coverage = 1;
    cudaError_t err = cudaSuccess;
    if (amb_decode_prepare(&st, 0, nullptr, &err) < 0) return -3;
    return amb_coverage_launch(recs, n, st.cgrid, nullptr, &err) < 0 ? -2 : 0;
}

// what the text-report stage holds: bit 0 its buffers, bit 1 its first-message flag, bit 2 the flag's value
extern "C" int emul_reports_state(void* h)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    return (st.rb.text ? 1 : 0) | (st.rfirst ? 2 : 0) | (st.rfirst && *st.rfirst ? 4 : 0);
}
