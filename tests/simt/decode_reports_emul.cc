// TEST HARNESS (not a product path): the decoder harness tests/simt/decode_emul.cc plus what tests/test_reports_simt.py
// needs of the text-report stage (amb_decode_reports.cuh). The option lives in the decoder's own AmbDecodeState; the
// harness's emul_decode sets every other option from its EmulOpts and leaves this one as emul_set_reports put it, so
// amb_decode_prepare, amb_decode_launch, amb_decode_reset and amb_decode_free treat the stage as the library does.
#include "decode_emul.cc"

// amb_decoder_set_option(d, "reports", on): applies from the next emul_decode
extern "C" void emul_set_reports(void* h, int on)
{
    static_cast<Emul*>(h)->st.reports = on;
}

// amb_decoder_reports after a decode of n frames with the option on: the packed lines into text; returns 0, or -5 when
// they do not fit `cap` (*n_bytes = their length either way)
extern "C" int emul_report_text(void* h, int n, char* text, size_t cap, size_t* n_bytes)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    *n_bytes = 0;
    if (n <= 0) return 0;
    const size_t total = (size_t)st.rb.boff[(n + 127) / 128];
    *n_bytes = total;
    if (total > cap) return -5;
    memcpy(text, st.rb.text, total);
    return 0;
}

// what the stage holds: bit 0 its buffers, bit 1 its first-message flag, bit 2 the flag's value
extern "C" int emul_reports_state(void* h)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    return (st.rb.text ? 1 : 0) | (st.rfirst ? 2 : 0) | (st.rfirst && *st.rfirst ? 4 : 0);
}

// amb_decoder_set_option(d, "coverage", on), which emul_decode's options do not carry: applies from the next emul_decode
extern "C" void emul_set_coverage(void* h, int on)
{
    static_cast<Emul*>(h)->st.coverage = on;
}
