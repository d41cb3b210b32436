// nyxb_od.cu — state-transition-matrix propagation and the sequential Kalman filter, one CUDA thread per trajectory
// (SURVEY.md §8 (f)-2; BASELINE configs[4]).  The whole arc of a filter — propagation of the nominal state and the STM
// between measurements, time updates, measurement updates, state replacement — runs inside ONE kernel launch; state,
// STM, covariance and stage data stay in registers / L1-resident local memory, HBM sees the inputs once and the
// per-measurement residual records as coalesced [m][..][n] stores.
//
// Built twice like nyxb_kernels.cu: -DNYXB_STRICT=1 -fmad=false (same operation order as oracle/nyx_oracle_od.c for
// the dynamics) and -DNYXB_STRICT=0 -fmad=true.
//
// Reference behaviour (paths relative to /root/reference/nyx-core/src):
//   SpacecraftDynamics::eom `Some(stm)` branch / dual_eom      dynamics/spacecraft.rs:203-227, 312-363
//   OrbitalDynamics::dual_eom, PointMasses::gradient           dynamics/orbital.rs:116-172, 249-307
//   GravityField::gradient                                     dynamics/gravity_field.rs:273-431
//   SolarPressure::gradient                                    dynamics/solarpressure.rs:167-233
//   PropInstance::{propagate, single_step, derive}             propagators/instance.rs:87-262, 343-493
//   KalmanODProcess::process_arc                               od/process/mod.rs:128-497
//   KalmanFilter::{time_update, measurement_update}            od/kalman/filtering.rs:59-316
//   ProcessNoise::propagate                                    od/snc.rs:175-286
//   GroundStation::measure_instantaneous, ScalarSensitivity    od/ground_station/trk_device.rs:154-200, od/msr/sensitivity.rs:118-239
// The reference gets the partials from forward-mode dual numbers (hyperdual 1.5.0); so does this file, with a 3-partial
// dual type (only d/d(position) is ever read).
#include "nyxb_od_device.cuh"

#ifndef NYXB_STRICT
#error "NYXB_STRICT must be defined to 0 or 1"
#endif
#if NYXB_STRICT
#define NYXB_KSTM nyxb_k_stm_strict
#define NYXB_KOD nyxb_k_od_strict
#define NYXB_LAUNCH_STM nyxb_launch_stm_strict
#define NYXB_LAUNCH_OD nyxb_launch_od_strict
#else
#define NYXB_KSTM nyxb_k_stm_fast
#define NYXB_KOD nyxb_k_od_fast
#define NYXB_LAUNCH_STM nyxb_launch_stm_fast
#define NYXB_LAUNCH_OD nyxb_launch_od_fast
#endif

// ------------------------------------------------------------------------- PropInstance over state + STM
struct InstS {
    double y[9];
    double phi[81];  // column-major like the reference's vector tail: (r, c) at c*9 + r
    long long epoch_ns, step_ns;
    int fixed, status;
    long long det_step_ns;
    double det_error;
    int det_attempts;
    long long n_steps, n_rejected, n_rhs;
    double dry_mass, extra_mass, srp_area;
};

__device__ __forceinline__ void phi_identity(double* phi) {
    for (int e = 0; e < 81; ++e) phi[e] = 0.0;
    for (int c = 0; c < 9; ++c) phi[c * 9 + c] = 1.0;
}

// one RHS evaluation: k[6] = (v, a), A-parts G[9], gcr[3]
__device__ static int eom_stm(const DevSetup& S, InstS& in, double delta_t_s, const double ys[9], double k[6], double G[9], double gcr[3]) {
    long long t_ns = in.epoch_ns + dur_from_seconds(delta_t_s);
    double yy[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) yy[e] = ys[e];
    yy[6] = yy[6] < 0.0 ? 0.0 : (yy[6] > 2.0 ? 2.0 : yy[6]);
    double mass = in.dry_mass + yy[8] + in.extra_mass;
    if (S.has_srp && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3];
    int rc = dual_eom_dev<true>(S, t_ns, yy, mass, in.srp_area, acc, G, gcr);
    in.n_rhs++;
    if (rc) return rc;
    k[0] = yy[3]; k[1] = yy[4]; k[2] = yy[5];
    k[3] = acc[0]; k[4] = acc[1]; k[5] = acc[2];
    return 0;
}

// instance.rs:358-493 on the 90-vector; stage STM derivative = ctx.stm * A_i (spacecraft.rs:213) with ctx = step start
__device__ static int derive_stm(const DevSetup& S, InstS& in, long long& dt_ns, double next[9], double next_phi[81]) {
    double k[NYXB_MAX_STAGES][6];
    double Ai[NYXB_MAX_STAGES][12];
    const int stages = S.tb.stages;
    in.det_attempts = 1;
    double h = dur_to_seconds(in.step_ns);
    for (;;) {
        int rc = eom_stm(S, in, 0.0, in.y, k[0], Ai[0], Ai[0] + 9);
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
            const double hz = h * 0.0;
            ys[6] = in.y[6] + hz; ys[7] = in.y[7] + hz; ys[8] = in.y[8] + hz;
            rc = eom_stm(S, in, S.tb.c[i] * h, ys, k[i + 1], Ai[i + 1], Ai[i + 1] + 9);
            if (rc) return rc;
        }
        double err_est[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int e = 0; e < 9; ++e) next[e] = in.y[e];
        { const double hz = h * 0.0; next[6] += hz; next[7] += hz; next[8] += hz; }
        for (int e = 0; e < 81; ++e) next_phi[e] = in.phi[e];
        for (int i = 0; i < stages; ++i) {
            if (!in.fixed) {
                double cf = h * S.tb.e[i];
#pragma unroll
                for (int e = 0; e < 6; ++e) err_est[e] += cf * k[i][e];
            }
            double cb = h * S.tb.b[i];
#pragma unroll
            for (int e = 0; e < 6; ++e) next[e] += cb * k[i][e];
            // (phi * A_i)(r, c): c < 3: sum_q phi(r, 3+q) G(q, c); 3 <= c < 6: phi(r, c-3); c == 6: sum_q phi(r, 3+q) gcr(q)
            const double* Gi = Ai[i];
            for (int r = 0; r < 9; ++r) {
                double p3 = in.phi[27 + r], p4 = in.phi[36 + r], p5 = in.phi[45 + r];
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    next_phi[c * 9 + r] += cb * ((p3 * Gi[c] + p4 * Gi[3 + c]) + p5 * Gi[6 + c]);
#pragma unroll
                for (int c = 3; c < 6; ++c) next_phi[c * 9 + r] += cb * in.phi[(c - 3) * 9 + r];
                next_phi[54 + r] += cb * ((p3 * Gi[9] + p4 * Gi[10]) + p5 * Gi[11]);
            }
        }
        if (in.fixed) {
            in.det_step_ns = in.step_ns;
            dt_ns = in.step_ns;
            return 0;
        }
        in.det_error = error_estimate(S.error_ctrl, err_est, next, in.y);
        if (ctl_accept(S, in.det_error, h, in.det_attempts)) {
            for (int e = 0; e < 9; ++e)
                if (next[e] != next[e]) return NYXB_ERR_PROP_MATH;
            for (int e = 0; e < 81; ++e)
                if (next_phi[e] != next_phi[e]) return NYXB_ERR_PROP_MATH;
            in.step_ns = ctl_accepted<pow_inv_int>(S, in.det_error, h, in.det_attempts, in.status, in.det_step_ns);
            dt_ns = in.det_step_ns;
            return 0;
        }
        in.det_attempts += 1;
        in.n_rejected += 1;
        h = ctl_retry<pow_inv_int>(S, in.det_error, h);
    }
}

__device__ static int single_step_stm(const DevSetup& S, InstS& in) {
    long long dt;
    double next[9], next_phi[81];
    int rc = derive_stm(S, in, dt, next, next_phi);
    if (rc) return rc;
    in.epoch_ns += dt;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = next[e];
    for (int e = 0; e < 81; ++e) in.phi[e] = next_phi[e];
    in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
    in.n_steps += 1;
    return (in.y[8] < 0.0) ? NYXB_ERR_FUEL_EXHAUSTED : 0;
}

__device__ static int propagate_stm(const DevSetup& S, InstS& in, long long duration_ns) {
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
            int rc = single_step_stm(S, in);
            if (rc) return rc;
            in.step_ns = prev_step;
            in.fixed = prev_fixed;
            if (backprop) in.step_ns = -in.step_ns;
            return 0;
        }
        int rc = single_step_stm(S, in);
        if (rc) return rc;
    }
}

__device__ __forceinline__ void inst_load(const DevSetup& S, InstS& in, size_t i, size_t n, const double* state, const double* consts,
                                          const long long* epoch0, const long long* step_io) {
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = state[(size_t)e * n + i];
    in.dry_mass = consts[i]; in.extra_mass = consts[n + i]; in.srp_area = consts[2 * n + i];
    in.epoch_ns = epoch0[i];
    in.step_ns = step_io ? step_io[i] : S.init_step_ns;
    in.fixed = S.fixed_step;
    in.status = 0;
    in.det_step_ns = S.init_step_ns; in.det_error = 0.0; in.det_attempts = 1;
    in.n_steps = 0; in.n_rejected = 0; in.n_rhs = 0;
}

__device__ __forceinline__ void inst_store(const InstS& in, int rc, size_t i, size_t n, double* out_state, long long* out_epoch,
                                           nyxb_details* out_details, int* out_status) {
#pragma unroll
    for (int e = 0; e < 9; ++e) out_state[(size_t)e * n + i] = in.y[e];
    out_epoch[i] = in.epoch_ns;
    if (out_details) {
        nyxb_details d;
        d.step_ns = in.det_step_ns; d.error = in.det_error; d.attempts = in.det_attempts; d._pad = 0;
        d.n_steps = in.n_steps; d.n_rejected = in.n_rejected; d.n_rhs = in.n_rhs;
        out_details[i] = d;
    }
    out_status[i] = (in.status & NYXB_WARN_MAX_ATTEMPTS) | rc;
}

__global__ void __launch_bounds__(64)
NYXB_KSTM(const __grid_constant__ DevSetup S, size_t n, const double* __restrict__ state, const double* __restrict__ consts,
          const long long* __restrict__ epoch0, long long end_epoch, long long* __restrict__ step_io,
          const double* __restrict__ stm_in, double* __restrict__ out_state, long long* __restrict__ out_epoch,
          double* __restrict__ out_stm, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    InstS in;
    inst_load(S, in, i, n, state, consts, epoch0, step_io);
    if (stm_in) { for (int e = 0; e < 81; ++e) in.phi[e] = stm_in[(size_t)e * n + i]; }
    else phi_identity(in.phi);
    int rc = propagate_stm(S, in, end_epoch - in.epoch_ns);
    for (int e = 0; e < 81; ++e) out_stm[(size_t)e * n + i] = in.phi[e];
    if (step_io) step_io[i] = in.step_ns;
    inst_store(in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

// ------------------------------------------------------------------------- 9x9 helpers (row-major)
__device__ static void mat9_mul(const double* A, const double* B, double* Cm) {  // C = A B
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) {
            double s = 0.0;
            for (int k = 0; k < 9; ++k) s += A[r * 9 + k] * B[k * 9 + c];
            Cm[r * 9 + c] = s;
        }
}
__device__ static void mat9_mul_bt(const double* A, const double* B, double* Cm) {  // C = A B^T
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) {
            double s = 0.0;
            for (int k = 0; k < 9; ++k) s += A[r * 9 + k] * B[c * 9 + k];
            Cm[r * 9 + c] = s;
        }
}

struct Filt {
    double P[81];      // covariance, row-major
    double xdev[9];    // state deviation (CKF)
    long long prev_epoch;
};

// ProcessNoise::propagate (snc.rs:211-286) added onto Pbar
__device__ static void add_snc(const DevOd& od, const InstS& in, const Filt& f, double* Pbar) {
    if (!od.snc_enabled) return;
    long long delta = in.epoch_ns - f.prev_epoch;
    if (delta > od.snc_disable_ns) return;
    double s[3] = { od.snc_diag[0], od.snc_diag[1], od.snc_diag[2] };
    if (od.snc_frame == 1) {  // RIC: rotate, keep the diagonal (snc.rs:226-247)
        const double* y = in.y;
        double rn = norm3(y[0], y[1], y[2]);
        double rh[3] = { y[0] / rn, y[1] / rn, y[2] / rn };
        double hx = y[1] * y[5] - y[2] * y[4], hy = y[2] * y[3] - y[0] * y[5], hz = y[0] * y[4] - y[1] * y[3];
        double hn = norm3(hx, hy, hz);
        double ch[3] = { hx / hn, hy / hn, hz / hn };
        double ih[3] = { ch[1] * rh[2] - ch[2] * rh[1], ch[2] * rh[0] - ch[0] * rh[2], ch[0] * rh[1] - ch[1] * rh[0] };
        double d[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) d[i] = ((rh[i] * s[0]) * rh[i] + (ih[i] * s[1]) * ih[i]) + (ch[i] * s[2]) * ch[i];
        s[0] = d[0]; s[1] = d[1]; s[2] = d[2];
    }
    double dt = dur_to_seconds(delta);
    double g1 = (dt * dt) / 2.0, g2 = dt;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        Pbar[i * 9 + i] += (g1 * s[i]) * g1;
        Pbar[i * 9 + 3 + i] += (g1 * s[i]) * g2;
        Pbar[(3 + i) * 9 + i] += (g2 * s[i]) * g1;
        Pbar[(3 + i) * 9 + 3 + i] += (g2 * s[i]) * g2;
    }
}

// covar_bar = stm * P * stm^T (+ SNC); filtering.rs:61-78 / 132-150
__device__ static void covar_bar(const DevOd& od, const InstS& in, const Filt& f, double* Pbar) {
    double Phi[81], T[81];
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) Phi[r * 9 + c] = in.phi[c * 9 + r];
    mat9_mul(Phi, f.P, T);
    mat9_mul_bt(T, Phi, Pbar);
    add_snc(od, in, f, Pbar);
}

// KalmanFilter::time_update, filtering.rs:59-102
__device__ static void time_update(const DevOd& od, const InstS& in, Filt& f) {
    double Pbar[81];
    covar_bar(od, in, f, Pbar);
    if (od.variant == NYXB_KF_DEVIATION_TRACKING) {
        double nx[9];
        for (int r = 0; r < 9; ++r) {
            double s = 0.0;
            for (int k = 0; k < 9; ++k) s += in.phi[k * 9 + r] * f.xdev[k];
            nx[r] = s;
        }
        for (int r = 0; r < 9; ++r) f.xdev[r] = nx[r];
    } else {
        for (int r = 0; r < 9; ++r) f.xdev[r] = 0.0;
    }
    for (int e = 0; e < 81; ++e) f.P[e] = Pbar[e];
    f.prev_epoch = in.epoch_ns;
}

__global__ void __launch_bounds__(64)
NYXB_KOD(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, size_t n, const double* __restrict__ state,
         const double* __restrict__ consts, const long long* __restrict__ epoch0, double* __restrict__ out_state,
         long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    InstS in;
    inst_load(S, in, i, n, state, consts, epoch0, nullptr);
    phi_identity(in.phi);                                    // prop.with(nominal.with_stm()) process/mod.rs:167
    if (!in.fixed) in.step_ns = od.max_step_ns;              // :170-172
    Filt f;
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) f.P[r * 9 + c] = od.covar0[(size_t)(c * 9 + r) * n + i];
    for (int r = 0; r < 9; ++r) f.xdev[r] = 0.0;
    f.prev_epoch = in.epoch_ns;
    long long epoch = in.epoch_ns;
    int rc = 0;
    const bool ekf = od.variant == NYXB_KF_REFERENCE_UPDATE;
    const int M = od.msr_size;
    for (long long k = 0; k < od.n_msr && rc == 0; ++k) {
        const long long t_k = od.msr_epoch[k];
        const double o[2] = { od.obs[((size_t)k * 2 + 0) * n + i], od.obs[((size_t)k * 2 + 1) * n + i] };
        int flags = 0;
        if (o[0] != o[0] && o[1] != o[1]) {
            if (od.flags) od.flags[(size_t)k * n + i] = NYXB_MSRF_ABSENT;
            continue;
        }
        for (;;) {
            long long delta_t = t_k - epoch;
            long long next_step = delta_t;                                      // :218
            if (in.step_ns < next_step) next_step = in.step_ns;
            if (od.max_step_ns < next_step) next_step = od.max_step_ns;
            rc = propagate_stm(S, in, next_step);                               // :232-234
            if (rc) break;
            epoch = in.epoch_ns;
            long long gap = in.epoch_ns - t_k;
            if (gap < 0) gap = -gap;
            if (gap < od.eps_ns) {                                              // :250
                in.epoch_ns = t_k;                                              // :254
                const int trk = od.msr_tracker[k];
                if (trk < 0 || trk >= od.n_stations) break;                     // unknown tracker :400-410
                const DevStation& gs = od.stations[trk];
                const int windows = gs.n_types / M;
                for (int wno = 0; wno <= windows; ++wno) {                      // :270-398
                    OdWindow w;
                    const int wrc = od_window_setup(S, gs, M, wno, o, t_k, in.y, w);
                    if (wrc == OD_WIN_EMPTY) break;
                    if (wrc == OD_WIN_UNAVAILABLE) continue;
                    if (wrc == OD_WIN_EPHEMERIS) { rc = NYXB_ERR_EPHEMERIS; break; }
                    if (wrc == OD_WIN_NOT_VISIBLE) { flags |= NYXB_MSRF_NOT_VISIBLE; continue; }
                    const int ncur = w.ncur;
                    const double (&H)[2][9] = w.H;
                    const double* Rk = w.Rk;
                    const double* real_obs = w.real_obs;
                    const double* comp = w.comp;
                    // ---- measurement_update (filtering.rs:107-316)
                    double Pbar[81];
                    covar_bar(od, in, f, Pbar);
                    double PHt[9][2], Sk[2][2] = { {0.0, 0.0}, {0.0, 0.0} }, pre[2] = { 0.0, 0.0 };
                    for (int r = 0; r < 9; ++r)
                        for (int q = 0; q < M; ++q) {
                            double s = 0.0;
                            for (int c = 0; c < 9; ++c) s += Pbar[r * 9 + c] * H[q][c];
                            PHt[r][q] = s;
                        }
                    for (int a = 0; a < M; ++a)
                        for (int b = 0; b < M; ++b) {
                            double s = 0.0;
                            for (int c = 0; c < 9; ++c) s += H[a][c] * PHt[c][b];
                            Sk[a][b] = s + ((a == b) ? Rk[a] : 0.0);
                        }
                    for (int q = 0; q < M; ++q) pre[q] = real_obs[q] - comp[q];
                    double ratio;
                    if (!od_ratio(M, Sk, Rk, pre, ratio)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularNoiseRk
                    const int rslot = (M == 1) ? wno : 0;
                    if (od.ratio) od.ratio[((size_t)k * 2 + rslot) * n + i] = ratio;
                    if (od.prefit) for (int q = 0; q < ncur; ++q) od.prefit[((size_t)k * 2 + wno * M + q) * n + i] = pre[q];
                    flags |= NYXB_MSRF_PROCESSED;
                    if (od.reject >= 0.0 && ratio > od.reject) {                // :169-184
                        time_update(od, in, f);
                        flags |= NYXB_MSRF_REJECTED;
                    } else {
                        // gain K = PHt S^-1 (Cholesky solve; plain inverse when S is not positive definite)
                        double Si[2][2];
                        if (!od_sinv(M, Sk, Si)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularKalmanGain
                        double K[9][2];
                        for (int r = 0; r < 9; ++r)
                            for (int q = 0; q < M; ++q) {
                                double s = 0.0;
                                for (int b = 0; b < M; ++b) s += PHt[r][b] * Si[b][q];
                                K[r][q] = s;
                            }
                        double xhat[9], post[2] = { 0.0, 0.0 };
                        if (ekf) {
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += K[r][q] * pre[q]; xhat[r] = s; }
                            for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xhat[c]; post[q] = pre[q] - s; }
                        } else {
                            double xbar[9];
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int c = 0; c < 9; ++c) s += in.phi[c * 9 + r] * f.xdev[c]; xbar[r] = s; }
                            for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xbar[c]; post[q] = pre[q] - s; }
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += K[r][q] * post[q]; xhat[r] = xbar[r] + s; }
                        }
                        // Joseph update: (I - K H) Pbar (I - K H)^T + K R K^T, then symmetrise (filtering.rs:290-300)
                        double F[81], T[81], Cv[81];
                        for (int r = 0; r < 9; ++r)
                            for (int c = 0; c < 9; ++c) {
                                double s = 0.0;
                                for (int q = 0; q < M; ++q) s += K[r][q] * H[q][c];
                                F[r * 9 + c] = ((r == c) ? 1.0 : 0.0) - s;
                            }
                        mat9_mul(F, Pbar, T);
                        mat9_mul_bt(T, F, Cv);
                        for (int r = 0; r < 9; ++r)
                            for (int c = 0; c < 9; ++c) {
                                double s = 0.0;
                                for (int q = 0; q < M; ++q) s += (K[r][q] * Rk[q]) * K[c][q];
                                Cv[r * 9 + c] += s;
                            }
                        for (int r = 0; r < 9; ++r)
                            for (int c = 0; c < 9; ++c) f.P[r * 9 + c] = 0.5 * (Cv[r * 9 + c] + Cv[c * 9 + r]);
                        for (int r = 0; r < 9; ++r) f.xdev[r] = xhat[r];
                        f.prev_epoch = in.epoch_ns;
                        if (od.postfit) for (int q = 0; q < ncur; ++q) od.postfit[((size_t)k * 2 + wno * M + q) * n + i] = post[q];
                        if (ekf) {                                               // :364-369 `Spacecraft + OVector<9>`
                            for (int r = 0; r < 9; ++r) in.y[r] = in.y[r] + xhat[r];
                            in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
                        }
                    }
                    phi_identity(in.phi);                                        // reset_stm :371
                }
                if (od.est_state) for (int r = 0; r < 9; ++r) od.est_state[((size_t)k * 9 + r) * n + i] = in.y[r];
                if (od.est_cov) for (int r = 0; r < 9; ++r) od.est_cov[((size_t)k * 9 + r) * n + i] = f.P[r * 9 + r];
                break;
            } else {
                time_update(od, in, f);                                          // :417-421
                phi_identity(in.phi);
            }
        }
        if (od.flags) od.flags[(size_t)k * n + i] = flags;
    }
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) od.covar[(size_t)(c * 9 + r) * n + i] = f.P[r * 9 + c];
    if (od.state_dev) for (int r = 0; r < 9; ++r) od.state_dev[(size_t)r * n + i] = f.xdev[r];
    inst_store(in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

extern "C" cudaError_t NYXB_LAUNCH_STM(const DevSetup* S, size_t n, const double* state, const double* consts, const long long* epoch0,
                                       long long end_epoch, long long* step_io, const double* stm_in, double* out_state,
                                       long long* out_epoch, double* out_stm, nyxb_details* out_details, int* out_status,
                                       cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KSTM<<<grid, block, 0, stream>>>(*S, n, state, consts, epoch0, end_epoch, step_io, stm_in, out_state, out_epoch, out_stm,
                                          out_details, out_status);
    return cudaGetLastError();
}

extern "C" cudaError_t NYXB_LAUNCH_OD(const DevSetup* S, const DevOd* od, size_t n, const double* state, const double* consts,
                                      const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                      int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // few, long-running threads: spread them over as many SMs as possible
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KOD<<<grid, block, 0, stream>>>(*S, *od, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    return cudaGetLastError();
}
