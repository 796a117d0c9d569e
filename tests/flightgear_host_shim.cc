// TEST HARNESS, not a product path: compiles the FlightGear packet math of the decoder (gr_air_modes_b200/csrc/
// amb_fg_format.h - the __host__ __device__ code amb_fg_count / amb_fg_write call on the device) for the host, so that
// tests/test_flightgear_cpu.py can check it byte for byte against tests/flightgear_oracle.py without a GPU. Built by the
// test into a temporary directory with plain g++ (-ffp-contract=off, as the device code is built with -fmad=false).
#include "../gr_air_modes_b200/csrc/amb_fg_format.h"

// the packets of n inputs into out + i * AMB_FG_PACKET; ok[i] = bytes written (0: the reference raises TypeError)
extern "C" void shim_fg_packets(const char* ident, const int* model, const double* lat, const double* lon,
                                const double* alt, const double* t, const double* hdg, const float* vel, const float* turn,
                                long n, char* out, int* ok)
{
    for (long i = 0; i < n; i++)
        ok[i] = (int)amb_fg_packet(ident + 8 * i, model[i], lat[i], lon[i], alt[i], t[i], hdg[i], vel[i], turn[i],
                                   out + i * AMB_FG_PACKET);
}

// amb_fg_model(ftc, cat)
extern "C" int shim_fg_model(int ftc, int cat) { return amb_fg_model(ftc, cat); }
