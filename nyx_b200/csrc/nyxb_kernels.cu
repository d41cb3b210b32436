// nyxb_kernels.cu — per-thread propagation kernel: one CUDA thread integrates one
// trajectory from its start epoch to the end epoch without touching HBM in between
// (state, stage derivatives and controller live in registers / L1-resident local memory).
//
// Built twice from this one source:
//   -DNYXB_STRICT=1 -fmad=false : reference operation order, no FMA contraction.  Output is
//                                 bit-identical to the CPU oracle wherever libm is not involved.
//   -DNYXB_STRICT=0 -fmad=true  : same algorithm, FMA contraction allowed (tolerance parity).
//
// Reference behaviour: PropInstance::propagate / single_step / derive
// (propagators/instance.rs:87-262, 343-352, 358-493).
#include "nyxb_device.cuh"

#ifndef NYXB_STRICT
#error "NYXB_STRICT must be defined to 0 or 1"
#endif

#if NYXB_STRICT
#define NYXB_KTHREAD nyxb_k_thread_strict
#define NYXB_LAUNCH_THREAD nyxb_launch_thread_strict
#else
#define NYXB_KTHREAD nyxb_k_thread_fast
#define NYXB_LAUNCH_THREAD nyxb_launch_thread_fast
#endif

struct Inst {
    double y[9];
    long long epoch_ns, step_ns;
    int fixed;
    int status;
    // details
    long long det_step_ns;
    double det_error;
    int det_attempts;
    long long n_steps, n_rejected, n_rhs;
    double dry_mass, extra_mass, srp_area, drag_area;
    // trajectory recording (instance.rs:186-193, 255-259)
    DevSink sink;
    size_t idx, n;
    double ev_prev;
    int ev_count;
};

// instance.rs:358-493
template <bool GRAV>
__device__ static int derive(const DevSetup& S, Inst& in, long long& dt_ns, double next[9]) {
    double k[NYXB_MAX_STAGES][6];
    const int stages = S.tb.stages;
    in.det_attempts = 1;
    double h = dur_to_seconds(in.step_ns);
    for (;;) {
        int rc = eom_full<GRAV>(S, in.epoch_ns, 0.0, in.y, in.dry_mass, in.extra_mass, in.srp_area, in.drag_area, k[0]);
        in.n_rhs++;
        if (rc) return rc;
        for (int i = 0; i < stages - 1; ++i) {
            double wi[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            const double* arow = &S.tb.a[i * NYXB_MAX_STAGES];
            for (int j = 0; j <= i; ++j) {
                double a_ij = arow[j];
#if !NYXB_STRICT
                if (a_ij == 0.0) continue;
#endif
#pragma unroll
                for (int e = 0; e < 6; ++e) wi[e] += a_ij * k[j][e];
            }
            double ys[9];
#pragma unroll
            for (int e = 0; e < 6; ++e) ys[e] = in.y[e] + h * wi[e];
            // components 6..8 have zero derivative: y + h*0 (NaN-propagating like the reference's 90-vector algebra, instance.rs:394)
            const double hz = h * 0.0;
            ys[6] = in.y[6] + hz; ys[7] = in.y[7] + hz; ys[8] = in.y[8] + hz;
            rc = eom_full<GRAV>(S, in.epoch_ns, S.tb.c[i] * h, ys, in.dry_mass, in.extra_mass, in.srp_area, in.drag_area, k[i + 1]);
            in.n_rhs++;
            if (rc) return rc;
        }
        double err_est[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int e = 0; e < 9; ++e) next[e] = in.y[e];
        { const double hz = h * 0.0; next[6] += hz; next[7] += hz; next[8] += hz; }
        for (int i = 0; i < stages; ++i) {
            if (!in.fixed) {
                double cf = h * S.tb.e[i];
#pragma unroll
                for (int e = 0; e < 6; ++e) err_est[e] += cf * k[i][e];
            }
            double cb = h * S.tb.b[i];
#pragma unroll
            for (int e = 0; e < 6; ++e) next[e] += cb * k[i][e];
        }
        if (in.fixed) {
            in.det_step_ns = in.step_ns;
            dt_ns = in.step_ns;
            return 0;
        }
        in.det_error = error_estimate(S.error_ctrl, err_est, next, in.y);
        if (ctl_accept(S, in.det_error, h, in.det_attempts)) {
#pragma unroll
            for (int e = 0; e < 9; ++e)
                if (next[e] != next[e]) return NYXB_ERR_PROP_MATH;
            in.step_ns = ctl_accepted<pow_inv_int>(S, in.det_error, h, in.det_attempts, in.status, in.det_step_ns);
            dt_ns = in.det_step_ns;
            return 0;
        }
        in.det_attempts += 1;
        in.n_rejected += 1;
        h = ctl_retry<pow_inv_int>(S, in.det_error, h);
    }
}

// one record of the trajectory sink: epoch + position/velocity of trajectory `idx` at slot s (step-major SoA)
__device__ __forceinline__ void record_state(const Inst& in, long long s) {
    if (s >= in.sink.cap) return;
    in.sink.epoch[(size_t)s * in.n + in.idx] = in.epoch_ns;
#pragma unroll
    for (int c = 0; c < 6; ++c) in.sink.state[((size_t)c * in.sink.cap + s) * in.n + in.idx] = in.y[c];
}

// instance.rs:343-352 + spacecraft.rs:158-189
template <bool GRAV>
__device__ static int single_step(const DevSetup& S, Inst& in) {
    long long dt;
    double next[9];
    int rc = derive<GRAV>(S, in, dt, next);
    if (rc) return rc;
    in.epoch_ns += dt;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = next[e];
    in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);  // cosmic/spacecraft.rs:494
    in.n_steps += 1;
    record_state(in, in.n_steps);  // the channel send of instance.rs:186-193 / 255-259
    return (in.y[8] < 0.0) ? NYXB_ERR_FUEL_EXHAUSTED : 0;
}

// instance.rs:87-262
template <bool GRAV>
__device__ static int propagate(const DevSetup& S, Inst& in, long long duration_ns) {
    if (duration_ns == 0) return 0;
    long long stop = in.epoch_ns + duration_ns;
    if (in.y[8] < 0.0) return NYXB_ERR_FUEL_EXHAUSTED;
    bool backprop = duration_ns < 0;
    if (backprop) in.step_ns = -in.step_ns;
    for (;;) {
        long long epoch = in.epoch_ns;
        if (ctl_past_stop(epoch, in.step_ns, stop, backprop)) {
            if (stop == epoch) return 0;
            long long prev_step = in.step_ns;
            int prev_fixed = in.fixed;
            in.step_ns = stop - epoch;
            in.fixed = 1;
            int rc = single_step<GRAV>(S, in);
            if (rc) return rc;
            in.step_ns = prev_step;
            in.fixed = prev_fixed;
            if (backprop) in.step_ns = -in.step_ns;
            return 0;
        }
        int rc = single_step<GRAV>(S, in);
        if (rc) return rc;
        if (in.sink.ev_kind) {  // stop condition, evaluated on non-final steps only (instance.rs:243-252, event.rs:120-150)
            const double yn = event_eval(in.sink.ev_kind, in.sink.ev_value, in.y[0], in.y[1], in.y[2], in.y[3], in.y[4], in.y[5]);
            if (in.ev_prev * yn < 0.0) in.ev_count += 1;
            in.ev_prev = yn;
            if (in.ev_count >= in.sink.ev_trigger) return 0;
        }
    }
}

// GRAV = false: the instantiation for dynamics without a gravity field (no Legendre scratch: fewer registers, smaller stack)
template <bool GRAV>
__global__ void __launch_bounds__(128)
NYXB_KTHREAD(const __grid_constant__ DevSetup S, size_t n,
             const double* __restrict__ state, const double* __restrict__ consts,
             const long long* __restrict__ epoch0, long long end_epoch,
             long long* __restrict__ step_io,
             double* __restrict__ out_state, long long* __restrict__ out_epoch,
             nyxb_details* __restrict__ out_details, int* __restrict__ out_status, const DevSink sink) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Inst in;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = state[(size_t)e * n + i];  // coalesced SoA loads
    in.dry_mass = consts[i]; in.extra_mass = consts[n + i]; in.srp_area = consts[2 * n + i]; in.drag_area = consts[3 * n + i];
    in.epoch_ns = epoch0[i];
    in.step_ns = step_io ? step_io[i] : S.init_step_ns;  // propagator.rs:88-108
    in.fixed = S.fixed_step;
    in.status = 0;
    in.det_step_ns = S.init_step_ns; in.det_error = 0.0; in.det_attempts = 1;
    in.n_steps = 0; in.n_rejected = 0; in.n_rhs = 0;
    in.sink = sink; in.idx = i; in.n = n;
    record_state(in, 0);  // start state (instance.rs:307, 321)
    in.ev_count = 0;
    in.ev_prev = sink.ev_kind ? event_eval(sink.ev_kind, sink.ev_value, in.y[0], in.y[1], in.y[2], in.y[3], in.y[4], in.y[5]) : 0.0;
    const int rc = propagate<GRAV>(S, in, end_epoch - in.epoch_ns);
#pragma unroll
    for (int e = 0; e < 9; ++e) out_state[(size_t)e * n + i] = in.y[e];
    out_epoch[i] = in.epoch_ns;
    if (step_io) step_io[i] = in.step_ns;
    if (out_details) {
        nyxb_details d;
        d.step_ns = in.det_step_ns; d.error = in.det_error; d.attempts = in.det_attempts; d._pad = 0;
        d.n_steps = in.n_steps; d.n_rejected = in.n_rejected; d.n_rhs = in.n_rhs;
        out_details[i] = d;
    }
    out_status[i] = ctl_finish(sink, i, in.status, rc, in.ev_count, in.n_steps);
}

extern "C" cudaError_t NYXB_LAUNCH_THREAD(const DevSetup* S, size_t n, const double* state, const double* consts,
                                          const long long* epoch0, long long end_epoch, long long* step_io,
                                          double* out_state, long long* out_epoch, nyxb_details* out_details,
                                          int* out_status, int block, const DevSink* sink, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    unsigned grid = (unsigned)((n + block - 1) / block);
    if (S->has_grav)
        NYXB_KTHREAD<true><<<grid, block, 0, stream>>>(*S, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch,
                                                       out_details, out_status, *sink);
    else
        NYXB_KTHREAD<false><<<grid, block, 0, stream>>>(*S, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch,
                                                        out_details, out_status, *sink);
    return cudaGetLastError();
}

