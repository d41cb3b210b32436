// nyxb_od_arc.cuh — the PropInstance over state + STM and the filter loop (KalmanODProcess::process_arc), written once for the
// per-thread (nyxb_od.cu) and the warp-cooperative (nyxb_od_coop.cu) kernels.
//
// Both kernels instantiate these templates with a backend B, a plain struct that says who computes what and where the arrays live:
//   B::stride, first()   an 81-entry loop runs over entries first(), first() + stride, ...: 0 and 1 for one thread per filter, the lane
//                        and 32 for one warp per filter;
//   sync()               makes the entries written by every lane visible to all of them (nothing, or __syncwarp());
//   lead()               the lane that writes the scalar records;
//   any(v)               v on any lane (the NaN check of the candidate);
//   S                    the DevSetup;
//   phi                  the STM, column-major like the ABI;
//   B::Step(b)           one propagation's scratch: candidate STM nphi, stage derivatives k[i][6], stage A-matrix parts Ai[i][12];
//   B::Filt(b)           one filter's storage: covariance P and state deviation xdev, and the update scratch Pb, T, F (9x9,
//                        row-major), PHt and K (9x2);
//   rhs(in, dt, ys, st, i) one right-hand side at in.epoch + dt into stage slot i: st.k[i] = (v, a), st.Ai[i][0..8] = d(a)/d(r)
//                        row-major, st.Ai[i][9..11] = d(a)/d(Cr).
// The scratch types let the per-thread backend keep its temporaries in scoped locals; the warp backend points them into its slab.
// Every scalar below (OdInst, h, the window, the gain inputs) is computed by every lane alike, so all lanes take the same branches.
#pragma once
#include <cfloat>
#include <type_traits>
#include "nyxb_od_device.cuh"

// PropInstance scalars of one trajectory or filter (instance.rs:87-262)
struct OdInst {
    double y[9];
    long long epoch_ns, step_ns;
    int fixed, status;
    long long det_step_ns;
    double det_error;
    int det_attempts;
    long long n_steps, n_rejected, n_rhs;
    double dry_mass, extra_mass, srp_area;
};

__device__ __forceinline__ void od_load(const DevSetup& S, OdInst& in, size_t i, size_t n, const double* state, const double* consts,
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

template <class B>
__device__ __forceinline__ void od_store(const B& b, const OdInst& in, int rc, size_t i, size_t n, double* out_state, long long* out_epoch,
                                         nyxb_details* out_details, int* out_status) {
    for (int r = b.first(); r < 9; r += B::stride) out_state[(size_t)r * n + i] = in.y[r];
    if (!b.lead()) return;
    out_epoch[i] = in.epoch_ns;
    if (out_details) {
        nyxb_details d;
        d.step_ns = in.det_step_ns; d.error = in.det_error; d.attempts = in.det_attempts; d._pad = 0;
        d.n_steps = in.n_steps; d.n_rejected = in.n_rejected; d.n_rhs = in.n_rhs;
        out_details[i] = d;
    }
    out_status[i] = (in.status & NYXB_WARN_MAX_ATTEMPTS) | rc;
}

template <class B>
__device__ __forceinline__ void od_reset_stm(B& b) {
    for (int e = b.first(); e < 81; e += B::stride) b.phi[e] = ((e / 9) == (e % 9)) ? 1.0 : 0.0;
    b.sync();
}

// ------------------------------------------------------------------------- PropInstance over state + STM
// instance.rs:358-493 on the 90-vector; stage STM derivative = ctx.stm * A_i (spacecraft.rs:213) with ctx = step start.  The candidate
// STM goes to st.nphi.  Components 6-8 get h * 0 added (instance.rs:394): NaN-propagating, and -0 becomes +0.
template <class B>
__device__ __forceinline__ int od_derive(B& b, typename B::Step& st, OdInst& in, long long& dt_ns, double next[9]) {
    const DevSetup& S = b.S;
    const int stages = S.tb.stages;
    in.det_attempts = 1;
    double h = dur_to_seconds(in.step_ns);
    for (;;) {
        int rc = b.rhs(in, 0.0, in.y, st, 0);
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
                for (int e = 0; e < 6; ++e) wi[e] += a_ij * st.k[j][e];
            }
            double ys[9];
#pragma unroll
            for (int e = 0; e < 6; ++e) ys[e] = in.y[e] + h * wi[e];
            const double hz = h * 0.0;
            ys[6] = in.y[6] + hz; ys[7] = in.y[7] + hz; ys[8] = in.y[8] + hz;
            rc = b.rhs(in, S.tb.c[i] * h, ys, st, i + 1);
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
                for (int e = 0; e < 6; ++e) err_est[e] += cf * st.k[i][e];
            }
            double cb = h * S.tb.b[i];
#pragma unroll
            for (int e = 0; e < 6; ++e) next[e] += cb * st.k[i][e];
        }
        // candidate STM: entry (r, c) = phi(r, c) + sum_i (h b_i) (phi A_i)(r, c), where (phi A_i)(r, c) is
        // c < 3: sum_q phi(r, 3+q) G(q, c); 3 <= c < 6: phi(r, c-3); c == 6: sum_q phi(r, 3+q) gcr(q); c > 6: 0
        bool bad = false;
        for (int e = b.first(); e < 81; e += B::stride) {
            const int c = e / 9, r = e - 9 * c;
            double v = b.phi[e];
            if (c < 7) {
                const double p3 = b.phi[27 + r], p4 = b.phi[36 + r], p5 = b.phi[45 + r], pc = (c >= 3 && c < 6) ? b.phi[(c - 3) * 9 + r] : 0.0;
                for (int i = 0; i < stages; ++i) {
                    const double cb = h * S.tb.b[i];
                    const double* Gi = st.Ai[i];
                    double d;
                    if (c < 3) d = (p3 * Gi[c] + p4 * Gi[3 + c]) + p5 * Gi[6 + c];
                    else if (c < 6) d = pc;
                    else d = (p3 * Gi[9] + p4 * Gi[10]) + p5 * Gi[11];
                    v += cb * d;
                }
            }
            st.nphi[e] = v;
            bad = bad || (v != v);
        }
        b.sync();
        if (in.fixed) {
            in.det_step_ns = in.step_ns;
            dt_ns = in.step_ns;
            return 0;
        }
        in.det_error = error_estimate(S.error_ctrl, err_est, next, in.y);
        if (ctl_accept(S, in.det_error, h, in.det_attempts)) {
            for (int e = 0; e < 9; ++e) bad = bad || (next[e] != next[e]);
            if (b.any(bad)) return NYXB_ERR_PROP_MATH;
            in.step_ns = ctl_accepted<pow_inv_int>(S, in.det_error, h, in.det_attempts, in.status, in.det_step_ns);
            dt_ns = in.det_step_ns;
            return 0;
        }
        in.det_attempts += 1;
        in.n_rejected += 1;
        h = ctl_retry<pow_inv_int>(S, in.det_error, h);
    }
}

template <class B>
__device__ __forceinline__ int od_single_step(B& b, typename B::Step& st, OdInst& in) {
    long long dt;
    double next[9];
    int rc = od_derive(b, st, in, dt, next);
    if (rc) return rc;
    in.epoch_ns += dt;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = next[e];
    for (int e = b.first(); e < 81; e += B::stride) b.phi[e] = st.nphi[e];
    b.sync();
    in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
    in.n_steps += 1;
    return (in.y[8] < 0.0) ? NYXB_ERR_FUEL_EXHAUSTED : 0;
}

template <class B>
__device__ int od_propagate(B& b, OdInst& in, long long duration_ns) {
    if (duration_ns == 0) return 0;
    long long stop = in.epoch_ns + duration_ns;
    if (in.y[8] < 0.0) return NYXB_ERR_FUEL_EXHAUSTED;
    bool backprop = duration_ns < 0;
    if (backprop) in.step_ns = -in.step_ns;
    typename B::Step st(b);
    for (;;) {
        long long epoch = in.epoch_ns;
        if (ctl_past_stop(epoch, in.step_ns, stop, backprop)) {
            if (stop == epoch) return 0;
            long long prev_step = in.step_ns;
            int prev_fixed = in.fixed;
            in.step_ns = stop - epoch;
            in.fixed = 1;
            int rc = od_single_step(b, st, in);
            if (rc) return rc;
            in.step_ns = prev_step;
            in.fixed = prev_fixed;
            if (backprop) in.step_ns = -in.step_ns;
            return 0;
        }
        int rc = od_single_step(b, st, in);
        if (rc) return rc;
    }
}

// ------------------------------------------------------------------------- time update, measurement update (filtering.rs:59-316)
// f.Pb = Phi P Phi^T (+ SNC: ProcessNoise::propagate, snc.rs:211-286); filtering.rs:61-78 / 132-150
template <class B, class Dev>
__device__ __forceinline__ void od_covar_bar(const DevOdT<Dev>& od, const OdInst& in, long long prev_epoch, B& b, typename B::Filt& f) {
    for (int e = b.first(); e < 81; e += B::stride) {   // T = Phi P
        const int r = e / 9, c = e - 9 * r;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) s += b.phi[k * 9 + r] * f.P[k * 9 + c];
        f.T[e] = s;
    }
    b.sync();
    for (int e = b.first(); e < 81; e += B::stride) {   // Pb = T Phi^T
        const int r = e / 9, c = e - 9 * r;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) s += f.T[r * 9 + k] * b.phi[k * 9 + c];
        f.Pb[e] = s;
    }
    b.sync();
    if (!od.snc_enabled) return;
    const long long delta = in.epoch_ns - prev_epoch;
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
    for (int i = b.first(); i < 3; i += B::stride) {
        f.Pb[i * 9 + i] += (g1 * s[i]) * g1;
        f.Pb[i * 9 + 3 + i] += (g1 * s[i]) * g2;
        f.Pb[(3 + i) * 9 + i] += (g2 * s[i]) * g1;
        f.Pb[(3 + i) * 9 + 3 + i] += (g2 * s[i]) * g2;
    }
    b.sync();
}

// KalmanFilter::time_update, filtering.rs:59-102
template <class B, class Dev>
__device__ __forceinline__ void od_time_update(const DevOdT<Dev>& od, const OdInst& in, long long& prev_epoch, B& b, typename B::Filt& f) {
    od_covar_bar(od, in, prev_epoch, b, f);
    const bool tracking = od.variant == NYXB_KF_DEVIATION_TRACKING;
    for (int r = b.first(); r < 9; r += B::stride) {   // new deviation into T, free once Pb is formed
        double s = 0.0;
        if (tracking)
            for (int k = 0; k < 9; ++k) s += b.phi[k * 9 + r] * f.xdev[k];
        f.T[r] = s;
    }
    b.sync();
    for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] = f.T[r];
    for (int e = b.first(); e < 81; e += B::stride) f.P[e] = f.Pb[e];
    b.sync();
    prev_epoch = in.epoch_ns;
}

// ------------------------------------------------------------------------- KalmanODProcess::process_arc (od/process/mod.rs:128-497)
// One estimate record (OdEstRecords, nyxb_od.cuh) at the reference's push points: the nominal state, deviation and covariance of the
// estimate just formed and the STM since the previous record, before the STM reset.
template <class B>
__device__ __forceinline__ void od_est_push(const OdEstRecords& er, long long& cnt, long long tag, const OdInst& in, B& b,
                                            const typename B::Filt& f, size_t i, size_t n) {
    const long long k = cnt++;
    if (k >= er.cap) return;
    if (b.lead()) { er.epoch[(size_t)k * n + i] = in.epoch_ns; er.tag[(size_t)k * n + i] = tag; }
    for (int r = b.first(); r < 9; r += B::stride) {
        er.nominal[((size_t)k * 9 + r) * n + i] = in.y[r];
        er.dev[((size_t)k * 9 + r) * n + i] = f.xdev[r];
    }
    for (int e = b.first(); e < 81; e += B::stride) {
        const int r = e / 9, c = e - 9 * r;
        er.covar[((size_t)k * 81 + c * 9 + r) * n + i] = f.P[e];
        er.stm[((size_t)k * 81 + e) * n + i] = b.phi[e];        // phi is column-major: e = c*9 + r
    }
}

// Loads filter i, runs the whole arc and stores the final covariance, deviation, state, details and status.  REC: also write one
// estimate record per entry of the reference's ODSolution.estimates into *er (null when REC is false); the filter's arithmetic and
// outputs are the same either way.  TRK: the tracker kind (GroundTrk, PosTrk, AerTrk, LinkTrk in nyxb_od_device.cuh); B::Filt's PHt and K hold
// 9 x TRK::NS entries.
template <class B, bool REC = false, class TRK = GroundTrk>
__device__ void od_process_arc(const DevOdT<typename TRK::Dev>& od, B& b, size_t i, size_t n, const double* state, const double* consts, const long long* epoch0,
                               double* out_state, long long* out_epoch, nyxb_details* out_details, int* out_status,
                               const OdEstRecords* er = nullptr) {
    constexpr int NS = TRK::NS;
    const DevSetup& S = b.S;
    OdInst in;
    od_load(S, in, i, n, state, consts, epoch0, nullptr);
    if (!in.fixed) in.step_ns = od.max_step_ns;              // :170-172
    typename B::Filt f(b);
    static_assert(sizeof(f.PHt) == sizeof(double) * 9 * NS && sizeof(f.K) == sizeof(double) * 9 * NS, "B::Filt of another tracker kind");
    for (int e = b.first(); e < 81; e += B::stride) {
        const int r = e / 9, c = e - 9 * r;
        f.P[e] = od.covar0[(size_t)(c * 9 + r) * n + i];
    }
    for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] = 0.0;
    od_reset_stm(b);                                         // prop.with(nominal.with_stm()) :167
    long long prev_epoch = in.epoch_ns;
    long long epoch = in.epoch_ns;
    int rc = 0;
    const bool ekf = od.variant == NYXB_KF_REFERENCE_UPDATE;
    const int M = od.msr_size;
    long long nrec = 0;
    for (long long k = 0; k < od.n_msr && rc == 0; ++k) {
        const long long t_k = od.msr_epoch[k];
        double o[NS];
#pragma unroll
        for (int s = 0; s < NS; ++s) o[s] = od.obs[((size_t)k * NS + s) * n + i];
        int flags = 0;
        if (TRK::absent(o)) {
            if (od.flags && b.lead()) od.flags[(size_t)k * n + i] = NYXB_MSRF_ABSENT;
            continue;
        }
        for (;;) {
            long long delta_t = t_k - epoch;
            long long next_step = delta_t;                                      // :218
            if (in.step_ns < next_step) next_step = in.step_ns;
            if (od.max_step_ns < next_step) next_step = od.max_step_ns;
            rc = od_propagate(b, in, next_step);                                // :232-234
            if (rc) break;
            epoch = in.epoch_ns;
            long long gap = in.epoch_ns - t_k;
            if (gap < 0) gap = -gap;
            if (!(gap < od.eps_ns)) {                                           // :250
                od_time_update(od, in, prev_epoch, b, f);                       // :417-421
                if (REC) od_est_push(*er, nrec, -1, in, b, f, i, n);            // push_time_update
                od_reset_stm(b);
                continue;
            }
            in.epoch_ns = t_k;                                                  // :254
            const int trk = od.msr_tracker[k];
            if (trk < 0 || trk >= od.n_stations) break;                         // unknown tracker :400-410
            const typename TRK::Dev& gs = od.stations[trk];
            const int windows = gs.n_types / M;
            for (int wno = 0; wno <= windows; ++wno) {                          // :270-398
                typename TRK::Win w;
                const int wrc = TRK::setup(S, gs, M, wno, o, t_k, epoch, in.y, w);
                if (wrc == OD_WIN_EMPTY) break;
                if (wrc == OD_WIN_UNAVAILABLE) continue;
                if (wrc == OD_WIN_EPHEMERIS) { rc = NYXB_ERR_EPHEMERIS; break; }
                if constexpr (std::is_same<TRK, LinkTrk>::value) {              // the failures only an interlink window has
                    if (wrc == OD_WIN_TX_NO_DATA) { rc = NYXB_ERR_TX_NO_DATA; break; }
                    if (wrc == OD_WIN_NO_RANGE) { rc = NYXB_ERR_NO_RANGE; break; }
                }
                if (wrc == OD_WIN_NOT_VISIBLE) { flags |= NYXB_MSRF_NOT_VISIBLE; continue; }
                const double (&H)[NS][9] = w.H;
                const double* Rk = w.Rk;
                // ---- measurement_update (filtering.rs:107-316)
                od_covar_bar(od, in, prev_epoch, b, f);
                for (int e = b.first(); e < 9 * NS; e += B::stride) {           // PHt[r][q], r = e / NS, q = e % NS
                    const int r = (NS == 2) ? (e >> 1) : e / NS, q = (NS == 2) ? (e & 1) : e % NS;
                    double s = 0.0;
                    if (q < M)
                        for (int c = 0; c < 9; ++c) s += f.Pb[r * 9 + c] * H[q][c];
                    f.PHt[e] = s;
                }
                b.sync();
                double Sk[NS][NS], pre[NS];
#pragma unroll
                for (int a = 0; a < NS; ++a) {
                    pre[a] = 0.0;
#pragma unroll
                    for (int bb = 0; bb < NS; ++bb) Sk[a][bb] = 0.0;
                }
                for (int a = 0; a < M; ++a)
                    for (int bb = 0; bb < M; ++bb) {
                        double s = 0.0;
                        for (int c = 0; c < 9; ++c) s += H[a][c] * f.PHt[c * NS + bb];
                        Sk[a][bb] = s + ((a == bb) ? Rk[a] : 0.0);
                    }
                for (int q = 0; q < M; ++q) pre[q] = w.real_obs[q] - w.comp[q];
                double ratio;
                if (!TRK::ratio(M, Sk, Rk, pre, ratio)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularNoiseRk
                const int rslot = TRK::ratio_slot(M, wno);
                if (b.lead()) {
                    if (od.ratio) od.ratio[((size_t)k * NS + rslot) * n + i] = ratio;
                    if (od.prefit) for (int q = 0; q < w.ncur; ++q) od.prefit[((size_t)k * NS + wno * M + q) * n + i] = pre[q];
                }
                flags |= NYXB_MSRF_PROCESSED;
                if (od.reject >= 0.0 && ratio > od.reject) {                    // :169-184
                    od_time_update(od, in, prev_epoch, b, f);
                    flags |= NYXB_MSRF_REJECTED;
                    if (REC) od_est_push(*er, nrec, TRK::tag(k, wno, 1, M), in, b, f, i, n);   // push_measurement_update
                } else {
                    // gain K = PHt S^-1 (Cholesky solve; plain inverse when S is not positive definite)
                    typename TRK::Gain g;
                    if (!TRK::gain_setup(M, Sk, g)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularKalmanGain
                    for (int e = b.first(); e < 9 * NS; e += B::stride) {       // K[r][q]
                        const int r = (NS == 2) ? (e >> 1) : e / NS, q = (NS == 2) ? (e & 1) : e % NS;
                        f.K[e] = TRK::gain_entry(M, g, &f.PHt[r * NS], q);
                    }
                    b.sync();
                    // xhat and postfit in every lane, so that the state replacement stays in registers
                    double xhat[9], post[NS];
#pragma unroll
                    for (int q = 0; q < NS; ++q) post[q] = 0.0;
                    if (ekf) {
                        for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += f.K[r * NS + q] * pre[q]; xhat[r] = s; }
                        for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xhat[c]; post[q] = pre[q] - s; }
                    } else {
                        double xbar[9];
                        for (int r = 0; r < 9; ++r) { double s = 0.0; for (int c = 0; c < 9; ++c) s += b.phi[c * 9 + r] * f.xdev[c]; xbar[r] = s; }
                        for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xbar[c]; post[q] = pre[q] - s; }
                        for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += f.K[r * NS + q] * post[q]; xhat[r] = xbar[r] + s; }
                    }
                    // Joseph update: (I - K H) Pbar (I - K H)^T + K R K^T, then symmetrise (filtering.rs:290-300)
                    for (int e = b.first(); e < 81; e += B::stride) {           // F = I - K H
                        const int r = e / 9, c = e - 9 * r;
                        double s = 0.0;
                        for (int q = 0; q < M; ++q) s += f.K[r * NS + q] * H[q][c];
                        f.F[e] = ((r == c) ? 1.0 : 0.0) - s;
                    }
                    b.sync();
                    for (int e = b.first(); e < 81; e += B::stride) {           // T = F Pb
                        const int r = e / 9, c = e - 9 * r;
                        double s = 0.0;
#pragma unroll
                        for (int kk = 0; kk < 9; ++kk) s += f.F[r * 9 + kk] * f.Pb[kk * 9 + c];
                        f.T[e] = s;
                    }
                    b.sync();
                    for (int e = b.first(); e < 81; e += B::stride) {           // Pb <- T F^T + K R K^T (Pb is dead after T)
                        const int r = e / 9, c = e - 9 * r;
                        double s = 0.0;
#pragma unroll
                        for (int kk = 0; kk < 9; ++kk) s += f.T[r * 9 + kk] * f.F[c * 9 + kk];
                        double s2 = 0.0;
                        for (int q = 0; q < M; ++q) s2 += (f.K[r * NS + q] * Rk[q]) * f.K[c * NS + q];
                        f.Pb[e] = s + s2;
                    }
                    b.sync();
                    for (int e = b.first(); e < 81; e += B::stride) {
                        const int r = e / 9, c = e - 9 * r;
                        f.P[e] = 0.5 * (f.Pb[e] + f.Pb[c * 9 + r]);
                    }
                    for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] = xhat[r];
                    b.sync();
                    prev_epoch = in.epoch_ns;
                    if (od.postfit && b.lead()) for (int q = 0; q < w.ncur; ++q) od.postfit[((size_t)k * NS + wno * M + q) * n + i] = post[q];
                    if (REC) od_est_push(*er, nrec, TRK::tag(k, wno, 0, M), in, b, f, i, n);   // pre-update nominal, x-hat
                    if (ekf) {                                                  // :364-369 `Spacecraft + OVector<9>`
                        for (int r = 0; r < 9; ++r) in.y[r] = in.y[r] + xhat[r];
                        in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
                    }
                }
                od_reset_stm(b);                                                // reset_stm :371
            }
            for (int r = b.first(); r < 9; r += B::stride) {
                if (od.est_state) od.est_state[((size_t)k * 9 + r) * n + i] = in.y[r];
                if (od.est_cov) od.est_cov[((size_t)k * 9 + r) * n + i] = f.P[r * 9 + r];
            }
            break;
        }
        if (od.flags && b.lead()) od.flags[(size_t)k * n + i] = flags;
    }
    b.sync();
    for (int e = b.first(); e < 81; e += B::stride) {
        const int r = e / 9, c = e - 9 * r;
        od.covar[(size_t)(c * 9 + r) * n + i] = f.P[e];
    }
    if (od.state_dev) for (int r = b.first(); r < 9; r += B::stride) od.state_dev[(size_t)r * n + i] = f.xdev[r];
    if (REC && b.lead()) er->count[i] = nrec;
    od_store(b, in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

// ------------------------------------------------------------------------- KalmanODProcess::predict_until (od/process/mod.rs:440-486)
// record k of run i (layout: OdRecords, nyxb_od.cuh)
template <class B>
__device__ __forceinline__ void od_record(const OdRecords& rec, long long k, const OdInst& in, B& b, const typename B::Filt& f, size_t i,
                                          size_t n) {
    if (k >= rec.cap) return;
    if (rec.state)
        for (int r = b.first(); r < 9; r += B::stride) {
            double v = in.y[r] + f.xdev[r];
            if (r == 6) v = v < 0.0 ? 0.0 : (v > 2.0 ? 2.0 : v);
            rec.state[((size_t)k * 9 + r) * n + i] = v;
        }
    if (rec.covar)
        for (int e = b.first(); e < 81; e += B::stride) {
            const int r = e / 9, c = e - 9 * r;
            rec.covar[((size_t)k * 81 + c * 9 + r) * n + i] = f.P[e];
        }
}

// Maps the covariance of estimate i from epoch0[i] until end_epoch[i]: the initial estimate is record 0, then chunks of max_step, each
// closed by a time update.  Unlike process_arc there is no set_step(max_step) (:452): the first chunk starts from the initial step, and
// the adaptive step carries over from chunk to chunk.  The loop stops at the first chunk end at or after end_epoch, so an end at or
// before the start still gives one chunk.  `kf.initialize_process_noises()` is not called here in the reference: it only resets the SNC
// decay, which DevOd does not carry, so there is nothing to skip.  A propagation error ends run i with that status; the records written
// up to then stay valid and rec_count[i] counts them.  dev0: [9][n] initial state deviation or null (zero).
template <class B>
__device__ void od_predict(const DevOd& od, B& b, size_t i, size_t n, const double* state, const double* consts, const long long* epoch0,
                           const long long* end_epoch, const double* dev0, const OdRecords& rec, long long* rec_count, double* out_state,
                           long long* out_epoch, nyxb_details* out_details, int* out_status) {
    const DevSetup& S = b.S;
    OdInst in;
    od_load(S, in, i, n, state, consts, epoch0, nullptr);
    typename B::Filt f(b);
    for (int e = b.first(); e < 81; e += B::stride) {
        const int r = e / 9, c = e - 9 * r;
        f.P[e] = od.covar0[(size_t)(c * 9 + r) * n + i];
    }
    for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] = dev0 ? __ldg(dev0 + (size_t)r * n + i) : 0.0;
    od_reset_stm(b);                                          // prop.with(nominal.with_stm()) :452
    const long long end = __ldg(end_epoch + i);
    long long prev_epoch = in.epoch_ns;
    long long k = 0;
    od_record(rec, k++, in, b, f, i, n);                      // push_time_update(initial_estimate) :448
    int rc = 0;
    for (;;) {                                                // :466-483
        rc = od_propagate(b, in, od.max_step_ns);             // for_duration(max_step)
        if (rc) break;
        od_time_update(od, in, prev_epoch, b, f);
        od_record(rec, k++, in, b, f, i, n);
        od_reset_stm(b);
        if (in.epoch_ns >= end) break;
    }
    b.sync();
    for (int e = b.first(); e < 81; e += B::stride) {
        const int r = e / 9, c = e - 9 * r;
        od.covar[(size_t)(c * 9 + r) * n + i] = f.P[e];
    }
    if (od.state_dev) for (int r = b.first(); r < 9; r += B::stride) od.state_dev[(size_t)r * n + i] = f.xdev[r];
    if (rec_count && b.lead()) rec_count[i] = k;
    od_store(b, in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

// ------------------------------------------------------------------------- BatchLeastSquares::estimate / evaluate (od/blse/mod.rs:146-541)
// The 9x9 algebra below is scalar code that every lane runs alike, so the decisions it feeds are uniform.  It reads the backend's arrays
// and writes each entry of its result exactly once, with a value that is the same on every lane, from sums kept in registers: a lane
// that runs ahead never changes an entry a slower lane has still to read.  Row-major 9x9 throughout.

// Cholesky factor L (lower triangle of L) of A + diag(add): the column-oriented ("gaxpy") algorithm of Golub & Van Loan, Matrix
// Computations, 4th ed., Alg. 4.2.2.  False when a pivot is not positive (nalgebra's `cholesky()` returning None).
__device__ __forceinline__ bool bls_chol(const double* A, const double add[9], double* L) {
    for (int j = 0; j < 9; ++j) {
        double d = A[j * 9 + j] + add[j];
        for (int k = 0; k < j; ++k) d -= L[j * 9 + k] * L[j * 9 + k];
        if (!(d > 0.0)) return false;
        d = sqrt(d);
        L[j * 9 + j] = d;
        for (int r = j + 1; r < 9; ++r) {
            double s = A[r * 9 + j];
            for (int k = 0; k < j; ++k) s -= L[r * 9 + k] * L[j * 9 + k];
            L[r * 9 + j] = s / d;
        }
    }
    return true;
}

// x = (L L^T)^-1 b: forward then back substitution
__device__ __forceinline__ void bls_chol_solve(const double* L, const double* b, double x[9]) {
    double y[9];
    for (int r = 0; r < 9; ++r) {
        double s = b[r];
        for (int k = 0; k < r; ++k) s -= L[r * 9 + k] * y[k];
        y[r] = s / L[r * 9 + r];
    }
    for (int r = 8; r >= 0; --r) {
        double s = y[r];
        for (int k = r + 1; k < 9; ++k) s -= L[k * 9 + r] * x[k];
        x[r] = s / L[r * 9 + r];
    }
}

// A = U D U^T with U unit upper triangular (Bierman, Factorization Methods for Discrete Sequential Estimation, 1977, the UDU^T
// factorisation, columns from the last to the first; the order nalgebra's `udu()` uses).  U goes to U (entries on and above the
// diagonal), D to d.  False when a d_j is zero.
__device__ __forceinline__ bool bls_udu(const double* A, double* U, double d[9]) {
    d[8] = A[80];
    if (d[8] == 0.0) return false;
    for (int i = 0; i < 9; ++i) U[i * 9 + 8] = (1.0 / d[8]) * A[i * 9 + 8];
    for (int j = 7; j >= 0; --j) {
        double dj = 0.0;
        for (int k = j + 1; k < 9; ++k) dj += d[k] * (U[j * 9 + k] * U[j * 9 + k]);
        d[j] = A[j * 9 + j] - dj;
        if (d[j] == 0.0) return false;
        for (int i = j - 1; i >= 0; --i) {
            double u = 0.0;
            for (int k = j + 1; k < 9; ++k) u += (d[k] * U[j * 9 + k]) * U[i * 9 + k];
            U[i * 9 + j] = (A[i * 9 + j] - u) / d[j];
        }
        U[j * 9 + j] = 1.0;
    }
    return true;
}

// V = U^-1 of a unit upper-triangular U (back substitution, column by column; entries above and on the diagonal)
__device__ __forceinline__ void bls_unit_upper_inv(const double* U, double* V) {
    for (int c = 0; c < 9; ++c) {
        V[c * 9 + c] = 1.0;
        for (int r = c - 1; r >= 0; --r) {
            double s = 0.0;
            for (int k = r + 1; k <= c; ++k) s += U[r * 9 + k] * V[k * 9 + c];
            V[r * 9 + c] = -s;
        }
    }
}

// Problem i of a batch: estimate() from the guess (state, epoch0) or, with bl.evaluate, the RMS of that state.  Storage: the
// information matrix in f.P, the accumulated STM product in f.Pb, the product scratch and U^-1 in f.T, the Cholesky / UDU factor in
// f.F, the normal vector in f.xdev.  The STM is set to the identity at the start of each iteration (`with_stm()`) and never reset
// inside it, so after each chunk phi = Phi(t, t0) and `stm_acc = phi * stm_acc` is the product of cumulative STMs, as coded (:219-222).
// A failed problem stores its status and the estimate it had reached.
template <class B>
__device__ void od_bls(const DevOd& od, const DevBls& bl, B& b, size_t i, size_t n, const double* state, const double* consts,
                       const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details, int* out_status) {
    const DevSetup& S = b.S;
    OdInst in;
    od_load(S, in, i, n, state, consts, epoch0, nullptr);
    const long long t0 = in.epoch_ns;
    double x[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) x[r] = in.y[r];
    typename B::Filt f(b);
    long long n_msr = 0;                                     // :152 the non-rejected (present) measurements of problem i
    for (long long k = 0; k < od.n_msr; ++k) {
        const double o0 = od.obs[((size_t)k * 2 + 0) * n + i], o1 = od.obs[((size_t)k * 2 + 1) * n + i];
        if (!(o0 != o0 && o1 != o1)) ++n_msr;
    }
    const bool lm = bl.solver == NYXB_BLS_LEVENBERG_MARQUARDT;
    double lambda = bl.lm_init, cur_rms = DBL_MAX, corr = DBL_MAX, rms = 0.0;
    int iter = 0, rc = 0;
    bool converged = false;
    if (!bl.evaluate && bl.covar)                            // :170 zeros until an iteration is accepted
        for (int e = b.first(); e < 81; e += B::stride) bl.covar[(size_t)e * n + i] = 0.0;
    if (n_msr < (bl.evaluate ? 1 : 2)) rc = NYXB_ERR_TOO_FEW_MEASUREMENTS;   // :155-161, :459-465
    const int passes = bl.evaluate ? 1 : bl.max_iter;
    while (rc == 0 && iter < passes) {
        ++iter;
        // prop.with(current_estimate.with_stm()): a new instance at the initial step (no set_step(max_step)); the counters carry on
#pragma unroll
        for (int r = 0; r < 9; ++r) in.y[r] = x[r];
        in.epoch_ns = t0;
        in.step_ns = S.init_step_ns;
        in.fixed = S.fixed_step;
        in.det_step_ns = S.init_step_ns; in.det_error = 0.0; in.det_attempts = 1;
        for (int e = b.first(); e < 81; e += B::stride) {    // info = I, stm_acc = I, STM = I (:186-197)
            const double v = ((e / 9) == (e % 9)) ? 1.0 : 0.0;
            f.P[e] = v; f.Pb[e] = v; b.phi[e] = v;
        }
        for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] = 0.0;
        b.sync();
        double ssq = 0.0;
        long long epoch = t0;
        for (long long k = 0; k < od.n_msr && rc == 0; ++k) {
            const long long t_k = od.msr_epoch[k];
            const double o[2] = { od.obs[((size_t)k * 2 + 0) * n + i], od.obs[((size_t)k * 2 + 1) * n + i] };
            if (o[0] != o[0] && o[1] != o[1]) continue;      // absent from problem i: `rejected`
            for (;;) {
                const long long delta_t = t_k - epoch;
                if (delta_t <= 0) break;                     // :207-210
                long long next_step = delta_t;               // :213
                if (in.step_ns < next_step) next_step = in.step_ns;
                if (od.max_step_ns < next_step) next_step = od.max_step_ns;
                rc = od_propagate(b, in, next_step);
                if (rc) break;
                epoch = in.epoch_ns;
                if (!bl.evaluate) {                          // stm_acc = phi * stm_acc (:220-222)
                    for (int e = b.first(); e < 81; e += B::stride) {
                        const int r = e / 9, c = e - 9 * r;
                        double s = 0.0;
#pragma unroll
                        for (int q = 0; q < 9; ++q) s += b.phi[q * 9 + r] * f.Pb[q * 9 + c];
                        f.T[e] = s;
                    }
                    b.sync();
                    for (int e = b.first(); e < 81; e += B::stride) f.Pb[e] = f.T[e];
                    b.sync();
                }
                long long gap = epoch - t_k;
                if (gap < 0) gap = -gap;
                if (!(gap < od.eps_ns)) continue;            // :224
                const int trk = od.msr_tracker[k];
                if (trk < 0 || trk >= od.n_stations) continue;   // unknown tracker :226-237
                const DevStation& gs = od.stations[trk];
                for (int wno = 0; wno < gs.n_types; ++wno) {     // each type of msr.data on its own, as U1 (:240-297)
                    OdWindow w;
                    const int wrc = od_window_setup<false>(S, gs, 1, wno, o, epoch, in.y, w);
                    if (wrc == OD_WIN_UNAVAILABLE || wrc == OD_WIN_NOT_VISIBLE) continue;   // type not in msr.data / not visible
                    if (wrc == OD_WIN_EPHEMERIS) { rc = NYXB_ERR_EPHEMERIS; break; }
                    const double real_obs = w.real_obs[0];
                    if (!isfinite(real_obs)) { rc = NYXB_ERR_INVALID_MEASUREMENT; break; }   // :266-272
                    const double resid = real_obs - w.comp[0];
                    const double weight = 1.0 / w.Rk[0];     // Rk > 0: checked by the host (:282)
                    if (!bl.evaluate) {
                        double h[9];                         // h = h_tilde * stm_acc (:286)
#pragma unroll
                        for (int c = 0; c < 9; ++c) {
                            double s = 0.0;
#pragma unroll
                            for (int q = 0; q < 9; ++q) s += w.H[0][q] * f.Pb[q * 9 + c];
                            h[c] = s;
                        }
                        for (int e = b.first(); e < 81; e += B::stride) {   // info += h^T h W (:290)
                            const int r = e / 9, c = e - 9 * r;
                            f.P[e] += (h[r] * h[c]) * weight;
                        }
                        for (int r = b.first(); r < 9; r += B::stride) f.xdev[r] += (h[r] * resid) * weight;   // :293
                        b.sync();
                    }
                    ssq += (weight * resid) * resid;         // :296
                }
            }
        }
        if (rc) break;
        rms = sqrt(ssq / (double)n_msr);                     // :307
        if (bl.evaluate) break;
        // ---- solve (:309-379)
        double add[9], dx[9];
        if (lm) {
            for (int q = 0; q < 9; ++q) {
                double d = 1.0;
                if (bl.lm_diag && q < 6) { d = f.P[q * 9 + q]; if (d <= 0.0) d = 1e-6; }
                add[q] = d * lambda;
            }
        } else {
            for (int q = 0; q < 9; ++q) add[q] = 0.0;
        }
        const bool ok = bls_chol(f.P, add, f.F);
        if (ok) bls_chol_solve(f.F, f.xdev, dx);
        b.sync();
        bool accept;
        if (!lm) {
            if (!ok) { rc = NYXB_ERR_SINGULAR_INFORMATION; break; }
            accept = true;
            cur_rms = rms;
        } else if (!ok) {                                    // :369-377 singular: raise lambda, the iteration is spent
            lambda *= bl.lm_inc * 10.0;
            lambda = fmin(lambda, bl.lm_max);
            continue;
        } else if (rms < cur_rms) {
            accept = true;
            lambda /= bl.lm_dec;
            lambda = fmax(lambda, bl.lm_min);
            cur_rms = rms;
        } else {
            accept = false;
            lambda *= bl.lm_inc;
            lambda = fmin(lambda, bl.lm_max);
        }
        if (!accept) { corr = DBL_MAX; continue; }           // :424-430
        // ---- `Spacecraft + OVector<9>`, correction size, covariance (:384-423)
#pragma unroll
        for (int r = 0; r < 9; ++r) x[r] = x[r] + dx[r];
        x[6] = x[6] < 0.0 ? 0.0 : (x[6] > 2.0 ? 2.0 : x[6]);
        corr = sqrt((dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2]);
        if (bl.covar) {
            double d[9];
            const bool udu = bls_udu(f.P, f.F, d);
            if (udu) bls_unit_upper_inv(f.F, f.T);
            b.sync();
            for (int e = b.first(); e < 81; e += B::stride) { // U^-T (D^-1 U^-1), or I when the factorisation fails
                const int r = e / 9, c = e - 9 * r;
                double s = (r == c) ? 1.0 : 0.0;
                if (udu) {
                    s = 0.0;
                    for (int k = 0; k <= (r < c ? r : c); ++k) s += f.T[k * 9 + r] * ((1.0 / d[k]) * f.T[k * 9 + c]);
                }
                bl.covar[(size_t)(c * 9 + r) * n + i] = s;
            }
            b.sync();
        }
        if (corr < bl.tol_pos_km) { converged = true; break; }
    }
#pragma unroll
    for (int r = 0; r < 9; ++r) in.y[r] = x[r];
    in.epoch_ns = t0;
    if (b.lead()) {
        if (bl.iters) bl.iters[i] = iter;
        if (bl.rms) bl.rms[i] = bl.evaluate ? rms : cur_rms;
        if (bl.corr_pos_km) bl.corr_pos_km[i] = corr;
        if (bl.converged) bl.converged[i] = converged ? 1 : 0;
    }
    od_store(b, in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

// ------------------------------------------------------------------------- one entry per OD job (nyxb_od.cuh), for either backend
// The job's input arrays are read through __ldg: unlike __restrict__ kernel arguments, pointers inside a descriptor do not tell the
// compiler that nothing the kernel writes aliases them, so the read-only path has to be asked for.
template <class B>
__device__ __forceinline__ void od_run(const OdStmJob& job, B& b, size_t i, size_t n, const double* state, const double* consts,
                                       const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                       int* out_status) {
    OdInst in;
    od_load(b.S, in, i, n, state, consts, epoch0, job.step_io);
    if (job.stm_in) { for (int e = 0; e < 81; ++e) b.phi[e] = __ldg(job.stm_in + (size_t)e * n + i); }
    else od_reset_stm(b);
    int rc = od_propagate(b, in, job.end_epoch - in.epoch_ns);
    for (int e = 0; e < 81; ++e) job.out_stm[(size_t)e * n + i] = b.phi[e];
    if (job.step_io) job.step_io[i] = in.step_ns;
    od_store(b, in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

template <class B, class Dev, bool REC>
__device__ __forceinline__ void od_run(const OdFilterJob<Dev, REC>& job, B& b, size_t i, size_t n, const double* state, const double* consts,
                                       const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                       int* out_status) {
    if constexpr (REC) {
        const OdEstRecords er = job.er;
        od_process_arc<B, true, typename Dev::Trk>(job.od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status, &er);
    } else {
        od_process_arc<B, false, typename Dev::Trk>(job.od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    }
}

template <class B>
__device__ __forceinline__ void od_run(const OdPredictJob& job, B& b, size_t i, size_t n, const double* state, const double* consts,
                                       const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                       int* out_status) {
    od_predict(job.od, b, i, n, state, consts, epoch0, job.end_epoch, job.dev0, job.rec, job.rec_count, out_state, out_epoch, out_details,
               out_status);
}

template <class B>
__device__ __forceinline__ void od_run(const OdBlsJob& job, B& b, size_t i, size_t n, const double* state, const double* consts,
                                       const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                       int* out_status) {
    od_bls(job.od, job.bl, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}
