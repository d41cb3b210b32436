// Host build of the targeter's per-problem arithmetic (nyx_b200/csrc/nyxb_target.h), for the CPU test
// tests/test_oracle_target.py::test_host_build_of_the_header_matches_the_restatement: same source as the update kernels compile.
// Test infrastructure only — not linked into libnyxb.so.
#include "../../nyx_b200/csrc/nyxb_target.h"

extern "C" double shim_tgt_eval(int param, const double* rv, double mu) { return nyxb_tgt_eval(param, rv, mu); }

extern "C" void shim_tgt_perturbed(const nyxb_target_config* cfg, int j, const double* xi, double* out) { nyxb_tgt_perturbed(*cfg, j, xi, out); }

// xf [(V + 1)][6] row-major; xi[6], total[6], err[6], prev_norm[1] in / out
extern "C" int shim_tgt_step(const nyxb_target_config* cfg, double mu, int it, const double* xf, double* xi, double* total, double* err,
                             double* prev_norm) {
    return nyxb_tgt_step(*cfg, mu, it, xf, xi, total, err, prev_norm);
}
