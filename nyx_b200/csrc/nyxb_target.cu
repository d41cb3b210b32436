// nyxb_target.cu — the update kernels of nyxb_target_batch (host loop in nyxb_api.cu).  Built once, without FMA contraction, for
// both modes: this is negligible work next to the propagations, and the host restatement then matches it up to libm ulps.
//
// Per-problem arrays have stride n (problem p); the propagation slab has stride M = A (V + 1) for the A active problems, slot
// j A + a holding problem idx[a]'s nominal (j = 0) or perturbation j - 1.
#include <cub/cub.cuh>

#include "nyxb_target.h"
#include "nyxb_target_dev.h"

namespace {

__global__ void __launch_bounds__(128) nyxb_tgt_init(TgtDev t, nyxb_target_config cfg, const double* __restrict__ pre_state,
                                                     const long long* __restrict__ pre_epoch, const int* __restrict__ pre_status) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= t.n) return;
    const size_t n = t.n;
    double rv[6];
    for (int i = 0; i < 9; ++i) t.start[i * n + p] = pre_state[i * n + p];
    for (int i = 0; i < 6; ++i) rv[i] = pre_state[i * n + p];
    t.epoch_c[p] = pre_epoch[p];
    const int s = pre_status[p];
    for (int j = 0; j < cfg.n_vars; ++j) t.total[j * n + p] = cfg.vars[j].init_guess;
    for (int i = 0; i < cfg.n_objs; ++i) t.err[i * n + p] = NAN;
    for (int i = 0; i < 6; ++i) t.achieved[i * n + p] = rv[i];
    t.iters[p] = 0;
    t.prev_norm[p] = INFINITY;
    t.idx[p] = (int)p;
    if (s & 0xFF) {
        t.status[p] = s;
        t.flag[p] = 0;
        return;
    }
    double g[6];
    for (int j = 0; j < cfg.n_vars; ++j) g[j] = cfg.vars[j].init_guess;
    nyxb_tgt_apply_vars(cfg, g, rv);
    for (int i = 0; i < 6; ++i) t.xi[i * n + p] = rv[i];
    t.status[p] = s;   // the warn flag so far
    t.flag[p] = 1;
}

// (V + 1) start states of every active problem
__global__ void __launch_bounds__(128) nyxb_tgt_stage(TgtDev t, nyxb_target_config cfg, int A, const int* __restrict__ idx) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    const size_t n = t.n, M = (size_t)A * (cfg.n_vars + 1);
    const size_t p = (size_t)idx[a];
    double xi[6], x[6];
    for (int i = 0; i < 6; ++i) xi[i] = t.xi[i * n + p];
    for (int j = 0; j <= cfg.n_vars; ++j) {
        const size_t k = (size_t)j * A + a;
        if (j == 0) for (int i = 0; i < 6; ++i) x[i] = xi[i];
        else nyxb_tgt_perturbed(cfg, j - 1, xi, x);
        for (int i = 0; i < 6; ++i) t.l_state[i * M + k] = x[i];
        for (int i = 6; i < 9; ++i) t.l_state[i * M + k] = t.start[i * n + p];
        for (int i = 0; i < 4; ++i) t.l_consts[i * M + k] = t.consts[i * n + p];
        t.l_epoch[k] = t.epoch_c[p];
    }
}

// one iteration of every active problem from its (V + 1) final states; flag[a] = 1 while it goes on
__global__ void __launch_bounds__(128) nyxb_tgt_update(TgtDev t, nyxb_target_config cfg, double mu, int A, const int* __restrict__ idx) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    const size_t n = t.n, M = (size_t)A * (cfg.n_vars + 1);
    const size_t p = (size_t)idx[a];
    int warn = t.status[p];
    int fail = 0;
    double xf[42];
    for (int j = 0; j <= cfg.n_vars; ++j) {
        const size_t k = (size_t)j * A + a;
        const int s = t.o_status[k];
        warn |= s & ~0xFF;
        if ((s & 0xFF) && !fail) fail = s & 0xFF;
        for (int i = 0; i < 6; ++i) xf[6 * j + i] = t.o_state[i * M + k];
    }
    const int it = t.iters[p];
    for (int i = 0; i < 6; ++i) t.achieved[i * n + p] = xf[i];
    int rc = fail;
    if (!fail) {
        double xi[6], tot[6], err[6], prev = t.prev_norm[p];
        for (int i = 0; i < 6; ++i) xi[i] = t.xi[i * n + p];
        for (int j = 0; j < cfg.n_vars; ++j) tot[j] = t.total[j * n + p];
        rc = nyxb_tgt_step(cfg, mu, it, xf, xi, tot, err, &prev);
        for (int i = 0; i < 6; ++i) t.xi[i * n + p] = xi[i];
        for (int j = 0; j < cfg.n_vars; ++j) t.total[j * n + p] = tot[j];
        for (int i = 0; i < cfg.n_objs; ++i) t.err[i * n + p] = err[i];
        t.prev_norm[p] = prev;
    }
    if (rc == NYXB_TGT_CONTINUE) {
        t.status[p] = warn;
        t.iters[p] = it + 1;
        t.flag[a] = 1;
    } else {
        t.status[p] = rc | warn;
        t.flag[a] = 0;
    }
}

// corrected = start + total correction, applied once with the DCM of the start state; achieved = final orbit + start's other entries
__global__ void __launch_bounds__(128) nyxb_tgt_finish(TgtDev t, nyxb_target_config cfg) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= t.n) return;
    const size_t n = t.n;
    double rv[6], tot[6];
    for (int i = 0; i < 6; ++i) rv[i] = t.start[i * n + p];
    for (int j = 0; j < cfg.n_vars; ++j) tot[j] = t.total[j * n + p];
    nyxb_tgt_apply_vars(cfg, tot, rv);
    for (int i = 0; i < 6; ++i) t.corrected[i * n + p] = rv[i];
    for (int i = 6; i < 9; ++i) {
        t.corrected[i * n + p] = t.start[i * n + p];
        t.achieved[i * n + p] = t.start[i * n + p];
    }
}

inline unsigned blocks(size_t n) { return (unsigned)((n + 127) / 128); }

}  // namespace

cudaError_t nyxb_tgt_launch_init(const TgtDev& t, const nyxb_target_config& cfg, const double* pre_state, const long long* pre_epoch,
                                 const int* pre_status, cudaStream_t st) {
    nyxb_tgt_init<<<blocks(t.n), 128, 0, st>>>(t, cfg, pre_state, pre_epoch, pre_status);
    return cudaGetLastError();
}

cudaError_t nyxb_tgt_launch_stage(const TgtDev& t, const nyxb_target_config& cfg, int A, const int* idx, cudaStream_t st) {
    nyxb_tgt_stage<<<blocks((size_t)A), 128, 0, st>>>(t, cfg, A, idx);
    return cudaGetLastError();
}

cudaError_t nyxb_tgt_launch_update(const TgtDev& t, const nyxb_target_config& cfg, double mu, int A, const int* idx, cudaStream_t st) {
    nyxb_tgt_update<<<blocks((size_t)A), 128, 0, st>>>(t, cfg, mu, A, idx);
    return cudaGetLastError();
}

cudaError_t nyxb_tgt_launch_finish(const TgtDev& t, const nyxb_target_config& cfg, cudaStream_t st) {
    nyxb_tgt_finish<<<blocks(t.n), 128, 0, st>>>(t, cfg);
    return cudaGetLastError();
}

// Stable compaction: out[0..*count) = the in[a] with flag[a] != 0, in order.  With temp == NULL only *temp_bytes is set.
cudaError_t nyxb_tgt_compact(void* temp, size_t* temp_bytes, const int* in, const int* flag, int* out, int* count, int A, cudaStream_t st) {
    return cub::DeviceSelect::Flagged(temp, *temp_bytes, in, flag, out, count, A, st);
}
