// TEST HARNESS (not a product path): the decoder harness tests/simt/decode_emul.cc plus what the tests of the Beast and
// AVR feeds need beside it: any kind of amb_decode_text (amb_decoder_beast / amb_decoder_avr included), the poisoning
// of the feeds' scratch between calls and whether their buffers are allocated.
#include "decode_emul.cc"

// amb_decode_text of `kind` (AMB_TEXT_*): the last decode's bytes into out; returns 0, or -5 when they do not fit `cap`
// (*n_bytes = their length either way)
extern "C" int emul_feed(void* h, int kind, char* out, size_t cap, size_t* n_bytes)
{
    const char* src = nullptr;
    unsigned long long total = 0;
    amb_decode_text(&static_cast<Emul*>(h)->st, kind, nullptr, &src, &total);
    *n_bytes = (size_t)total;
    if (total > cap) return -5;
    if (total) memcpy(out, src, total);
    return 0;
}

// every byte of the feeds' allocated scratch set to garbage: no kernel may read what an earlier call left there
extern "C" void emul_feed_poison(void* h)
{
    AmbDecodeState& st = static_cast<Emul*>(h)->st;
    const struct { AmbReportBufs* b; int cap; size_t bytes; } sets[] = {{&st.bb, st.bcap, AMB_BEAST_MAX_MSG},
                                                                     {&st.ab, st.acap, AMB_AVR_MAX_LINE}};
    for (const auto& x : sets) {
        if (!x.b->text) continue;
        const size_t c = (size_t)x.cap, nb = (c + 127) / 128;
        std::fill_n(x.b->len, c, 0xA5A5A5A5u); std::fill_n(x.b->bsum, nb, 0xA5A5A5A5u);
        std::fill_n(x.b->boff, nb + 1, 0xA5A5A5A5A5ull); memset(x.b->text, 0x1a, c * x.bytes);
    }
}

// bit 0: the Beast feed's buffers are allocated, bit 1: the AVR feed's
extern "C" int emul_feed_state(void* h)
{
    const AmbDecodeState& st = static_cast<Emul*>(h)->st;
    return (st.bb.text ? 1 : 0) | (st.ab.text ? 2 : 0);
}
