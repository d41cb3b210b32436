// Host build of the smoothing kernel's 9x9 part (nyx_b200/csrc/nyxb_smooth.h), for the CPU test
// tests/test_oracle_smooth.py::test_host_build_of_the_9x9_core_matches_the_restatement: same source as the CUDA kernel compiles.
// Test infrastructure only — not linked into libnyxb.so.
#include "../../nyx_b200/csrc/nyxb_smooth.h"

// one smoothed estimate from row-major phi, P, x: returns 0, or 1 on a singular phi
extern "C" int shim_smooth_core(const double* phi, const double* P, const double* x, double* Ps, double* xs, double* Pi) {
    double T[81], ph[81];
    for (int e = 0; e < 81; ++e) ph[e] = phi[e];
    if (!nyxb_smooth_core(ph, P, x, Pi, T, ph, xs)) return 1;
    for (int e = 0; e < 81; ++e) Ps[e] = ph[e];
    return 0;
}
