// TEST HARNESS (not a product path): the shared decoder harness tests/simt/decode_emul.cc, unchanged, plus the option
// "opstatus". emul_decode leaves AmbDecodeState::opstatus as it finds it, so emul_decode_all sets the op-status stage's
// S and table on the state and then decodes through emul_decode - the decoder's own amb_decode_launch, with every stage
// whose S is > 0. The op-status table spans all 2^24 addresses like the decoder's; it is allocated at the first decode
// with the stage on and kept per harness handle. tests/test_opstatus_simt.py builds it with plain g++
// (tests/emul_build.py).
#include "decode_emul.cc"

#include <map>

static std::map<void*, std::vector<AmbOpsSlot>> g_otables;   // the op-status table of each handle

// amb_decode_frames with every option; returns what emul_decode returns
extern "C" int emul_decode_all(void* h, const amb_frame* frames, int n, int have_loc, double lat, double lon, int local_S,
                               int commb_S, int opstatus_S, int track_S, amb_fields* out)
{
    Emul* e = static_cast<Emul*>(h);
    if (opstatus_S > 0 && !e->st.otable) {
        std::vector<AmbOpsSlot>& t = g_otables[h];
        t.resize((size_t)AMB_OPS_SLOTS);
        memset(t.data(), 0xFF, t.size() * sizeof(AmbOpsSlot));
        e->st.otable = t.data();
    }
    e->st.opstatus = opstatus_S;
    return emul_decode(h, frames, n, have_loc, lat, lon, local_S, commb_S, track_S, out);
}

extern "C" void emul_free_all(void* h)
{
    g_otables.erase(h);
    emul_free(h);
}
