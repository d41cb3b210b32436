// nyxb_coop_strict.cu — lane-cooperative propagation kernel, STRICT mode: bit-identical to the CPU oracle.
//
// Built with -fmad=false -DNYXB_STRICT=1.  G lanes of one warp integrate ONE trajectory and reproduce the reference's
// floating-point operation order exactly (gravity_field.rs:148-268, instance.rs:358-493), so the result equals the
// per-thread STRICT kernel and the oracle bit for bit, while the harmonic sum is still shared by the lanes:
//
//   phase 1  columns: lane walks whole columns m of the derived-Legendre triangle with the reference recursion
//            a[n][m] = u*b[n][m]*a[n-1][m] - c[n][m]*a[n-2][m]  (every value depends on its own column only, so
//            any column->lane assignment yields the reference's values) and stores them in the trajectory's
//            shared-memory triangle;  all lanes run the (inherently sequential) r_m/i_m recurrence redundantly.
//   phase 2  rows: lane evaluates whole degrees n: the four partial sums over m = 0..min(n,M) in the reference's
//            order (sequential in m), then rr_n * sum_n, written to rowres[n].
//   phase 3  every lane adds rowres[1..N] in ascending n (the reference's `accel4 += rr * sum` order) and finishes.
//
// No FMA, no regrouping, no approximations: sin/cos via the shared deterministic routine, controller power via
// pow_inv_int.  RK stage algebra, error norm and controller as in the per-thread STRICT kernel.
#include <algorithm>
#include <numeric>
#include <vector>

#include "nyxb_coop.h"

#if !NYXB_STRICT
#error "nyxb_coop_strict.cu must be built with -DNYXB_STRICT=1 -fmad=false"
#endif

#define SCOOP_CTA 128
#define SCOOP_FIXED 120  // kst[96] + ys[6] + ycur[6] + nxt[6] + er[6]

__host__ __device__ inline int scoop_traj_stride(int N) {
    // + rm[N+2] + im[N+2] + rowres[(N+1)*4] + A[(N+2)(N+3)/2]
    int s = SCOOP_FIXED + 2 * (N + 2) + 4 * (N + 1) + (N + 2) * (N + 3) / 2;
    return s + ((8 - (s & 15)) & 15);
}

size_t nyxb_coop_strict_smem(int N, int G) { return (size_t)(SCOOP_CTA / G) * (size_t)scoop_traj_stride(N) * sizeof(double); }

void nyxb_coop_strict_build_host(int N, int M, int G, CoopStrictHost& out) {
    auto lpt = [&](const std::vector<std::pair<int, int>>& items /* (id, weight), any order */, std::vector<std::vector<int>>& lists) {
        std::vector<std::pair<int, int>> it = items;
        std::sort(it.begin(), it.end(), [](auto& a, auto& b) { return a.second > b.second; });
        std::vector<int> load(G, 0);
        lists.assign(G, {});
        for (auto& p : it) {
            int best = (int)(std::min_element(load.begin(), load.end()) - load.begin());
            lists[best].push_back(p.first);
            load[best] += p.second;
        }
        for (auto& l : lists) std::sort(l.begin(), l.end());  // ascending: rows must be walked in increasing n
    };
    const int mcols = std::min(M + 1, N + 1);
    std::vector<std::pair<int, int>> cols, rows;
    for (int m = 1; m <= mcols; ++m) cols.push_back({m, N + 2 - m});
    for (int n = 1; n <= N; ++n) rows.push_back({n, std::min(n, M) + 1});
    std::vector<std::vector<int>> cl, rl;
    lpt(cols, cl);
    lpt(rows, rl);
    out.G = G;
    out.kc = 1; out.kr = 1;
    for (auto& l : cl) out.kc = std::max(out.kc, (int)l.size());
    for (auto& l : rl) out.kr = std::max(out.kr, (int)l.size());
    out.cols.assign((size_t)G * (out.kc + 1), -1);
    out.rows.assign((size_t)G * (out.kr + 1), -1);
    for (int l = 0; l < G; ++l) {
        for (size_t k = 0; k < cl[l].size(); ++k) out.cols[(size_t)l * (out.kc + 1) + k] = cl[l][k];
        for (size_t k = 0; k < rl[l].size(); ++k) out.rows[(size_t)l * (out.kr + 1) + k] = rl[l][k];
    }
}

struct SCtx {
    double* kst; double* ys; double* ycur; double* nxt; double* er;
    double* rm; double* im; double* rowres; double* A;
    double dry_mass, extra_mass, srp_area, drag_area;
    double cr, cd, pm, hz;
};

static __device__ __noinline__ int scoop_pre(const DevSetup& S, long long t_ns, const double y[9], double bpos[NYXB_MAX_BODIES][3], double acc[3]) {
    return accel_pre(S, t_ns, y, bpos, acc);
}
static __device__ __noinline__ void scoop_xfields(const DevSetup& S, long long t_ns, const double y[9], const double bpos[NYXB_MAX_BODIES][3], double acc[3]) {
    accel_extra_fields(S, t_ns, y, bpos, acc);
}
static __device__ __noinline__ void scoop_post(const DevSetup& S, const SCtx& g, long long t_ns, const double y[9],
                                               const double bpos[NYXB_MAX_BODIES][3], double mass, double acc[3]) {
    accel_post(S, t_ns, y, bpos, mass, g.srp_area, g.drag_area, acc);
}

// SpacecraftDynamics::eom (spacecraft.rs:191-310), cooperative, reference operation order; lane c < 6 receives dy[c].
template <int G>
__device__ __forceinline__ int scoop_rhs(const DevSetup& S, const DevCoopStrict& Cs, const SCtx& g, int lane, unsigned gmask,
                                         long long t_ns, double& dyc) {
    const DevGrav& gv = S.grav;
    const int N = gv.N, M = gv.M;
    double y[9];
#pragma unroll
    for (int e = 0; e < 6; ++e) y[e] = g.ys[e];
    y[6] = g.cr + g.hz; y[7] = g.cd + g.hz; y[8] = g.pm + g.hz;
    const double mass = g.dry_mass + y[8] + g.extra_mass;
    const bool has_force = S.has_srp || S.has_drag;
    if (has_force && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3];
    double bpos[NYXB_MAX_BODIES][3];
    int rc = scoop_pre(S, t_ns, y, bpos, acc);  // two-body + point masses, reference order
    if (rc) return rc;

    // ---- DCM: lanes 0..2 evaluate one deterministic sin/cos pair each (same routine as rotation_dcm)
    double R[9];
    if (gv.rot.kind == 0) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    } else {
        const double t_s = dur_to_seconds(t_ns);
        const double d = t_s / 86400.0;
        const double T = d / 36525.0;
        double ang;
        if (lane == 0) ang = (gv.rot.ra0 + gv.rot.ra1 * T) * NYXB_DEG2RAD;
        else if (lane == 1) ang = (gv.rot.dec0 + gv.rot.dec1 * T) * NYXB_DEG2RAD;
        else ang = fmod(gv.rot.w0 + gv.rot.w1 * d, 360.0) * NYXB_DEG2RAD;
        double sv, cv;
        det_sincos(ang, sv, cv);
        const double sa = __shfl_sync(gmask, sv, 0, G), ca = __shfl_sync(gmask, cv, 0, G);
        const double sd = __shfl_sync(gmask, sv, 1, G), cd = __shfl_sync(gmask, cv, 1, G);
        const double sw = __shfl_sync(gmask, sv, 2, G), cw = __shfl_sync(gmask, cv, 2, G);
        const double b00 = -sa, b01 = ca, b02 = 0.0;
        const double b10 = -(sd * ca), b11 = -(sd * sa), b12 = cd;
        const double b20 = cd * ca, b21 = cd * sa, b22 = sd;
        R[0] = cw * b00 + sw * b10; R[1] = cw * b01 + sw * b11; R[2] = cw * b02 + sw * b12;
        R[3] = cw * b10 - sw * b00; R[4] = cw * b11 - sw * b01; R[5] = cw * b12 - sw * b02;
        R[6] = b20; R[7] = b21; R[8] = b22;
    }
    double rb[3], rel[3];
    grav_rel(S.grav_body, y, bpos, rel);   // field of another body: the state is translated to it first (gravity_field.rs:149-154)
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = (R[3 * i] * rel[0] + R[3 * i + 1] * rel[1]) + R[3 * i + 2] * rel[2];
    const double r_ = norm3(rb[0], rb[1], rb[2]);
    const double s_ = rb[0] / r_, t_ = rb[1] / r_, u_ = rb[2] / r_;

    // ---- phase 1: columns of the derived-Legendre triangle (gravity_field.rs:61-66, 168-181)
    {
        const int* myc = Cs.cols + lane * (Cs.kc + 1);
        for (int k = 0;; ++k) {
            const int m = __ldg(myc + k);
            if (m < 0) break;
            double a2 = __ldg(gv.a_diag + m);  // a[m][m]
            g.A[tri(m, m)] = a2;
            if (m + 1 <= N + 1) {
                double a1 = __ldg(gv.offdiag + m) * u_ * a2;  // a[m+1][m] = sqrt(2m+3) * u * a[m][m]
                g.A[tri(m + 1, m)] = a1;
                // (b, c) of the next degree are fetched one iteration ahead: the recursion is a dependent chain
                const double2* bc = reinterpret_cast<const double2*>(gv.tab);  // DevHarm = {b,c | vr01,vr11 | cbar,sbar}
                double2 nbc = (m + 2 <= N + 1) ? __ldg(bc + 3 * tri(m + 2, m)) : make_double2(0.0, 0.0);
                for (int n = m + 2; n <= N + 1; ++n) {
                    const double2 cur = nbc;
                    if (n + 1 <= N + 1) nbc = __ldg(bc + 3 * tri(n + 1, m));
                    const double an = u_ * cur.x * a1 - cur.y * a2;
                    g.A[tri(n, m)] = an;
                    a2 = a1; a1 = an;
                }
            }
        }
        // r_m / i_m recurrence (gravity_field.rs:184-193): sequential by nature, evaluated redundantly, stored once
        const int mm = N < M ? N : M;
        double rr = 1.0, ii = 0.0;
        if (lane == 0) { g.rm[0] = rr; g.im[0] = ii; }
        for (int m = 1; m <= mm; ++m) {
            const double nr = s_ * rr - t_ * ii;
            const double ni = s_ * ii + t_ * rr;
            rr = nr; ii = ni;
            if (lane == 0) { g.rm[m] = rr; g.im[m] = ii; }
        }
    }
    __syncwarp(gmask);

    // ---- phase 2: degrees n assigned to this lane, ascending (gravity_field.rs:209-249)
    {
        const double rho = gv.r_eq / r_;
        double rho_np1 = gv.mu / r_ * rho;
        int nprev = 0;
        const double sqrt2 = sqrt(2.0);
        const int* myr = Cs.rows + lane * (Cs.kr + 1);
        for (int k = 0;; ++k) {
            const int n = __ldg(myr + k);
            if (n < 0) break;
            while (nprev < n) { rho_np1 *= rho; ++nprev; }  // the reference multiplies once per degree, n = 1, 2, ...
            double sx = 0.0, sy = 0.0, sz = 0.0, sw = 0.0;
            const DevHarm* trow = gv.tab + tri(n, 0);
            const double* An = g.A + tri(n, 0);
            const double* An1 = g.A + tri(n + 1, 0);
            const int mtop = n < M ? n : M;
            double rm_prev = 0.0, im_prev = 0.0;
            // software pipeline: coefficients of term m+1 are in flight while term m is summed
            const double2* t2 = reinterpret_cast<const double2*>(trow);
            double2 nvr = __ldg(t2 + 1), ncs = __ldg(t2 + 2);
            for (int m = 0; m <= mtop; ++m) {
                const double2 vr = nvr, csv = ncs;
                if (m < mtop) { nvr = __ldg(t2 + 3 * (m + 1) + 1); ncs = __ldg(t2 + 3 * (m + 1) + 2); }
                const double cv = csv.x, sv = csv.y;
                const double rmm = g.rm[m], imm = g.im[m];
                const double d_ = (cv * rmm + sv * imm) * sqrt2;
                if (m != 0) {
                    const double e_ = (cv * rm_prev + sv * im_prev) * sqrt2;
                    const double f_ = (sv * rm_prev - cv * im_prev) * sqrt2;
                    const double anm = An[m];
                    sx += (double)m * anm * e_;
                    sy += (double)m * anm * f_;
                }  // m == 0: the reference adds (0*a)*0 = +-0, which leaves the sums unchanged
                const double a_n_m1 = (m + 1 <= n) ? An[m + 1] : 0.0;  // above the diagonal the matrix is zero
                sz += vr.x * a_n_m1 * d_;
                sw -= vr.y * An1[m + 1] * d_;
                rm_prev = rmm; im_prev = imm;
            }
            const double rr = rho_np1 / gv.r_eq;
            double* o = g.rowres + 4 * n;
            o[0] = rr * sx; o[1] = rr * sy; o[2] = rr * sz; o[3] = rr * sw;
        }
    }
    __syncwarp(gmask);

    // ---- phase 3: accel4 += rr * sum in ascending degree (gravity_field.rs:247-248), then :250-267
    double a4x = 0.0, a4y = 0.0, a4z = 0.0, a4w = 0.0;
    for (int n = 1; n <= N; ++n) {
        const double* o = g.rowres + 4 * n;
        a4x += o[0]; a4y += o[1]; a4z += o[2]; a4w += o[3];
    }
    const double ab0 = a4x + a4w * s_, ab1 = a4y + a4w * t_, ab2 = a4z + a4w * u_;
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[i] += (R[i] * ab0 + R[3 + i] * ab1) + R[6 + i] * ab2;
    if (S.n_xgrav > 0) scoop_xfields(S, t_ns, y, bpos, acc);
    if (has_force) scoop_post(S, g, t_ns, y, bpos, mass, acc);
    double out = y[3];
    if (lane == 1) out = y[4];
    else if (lane == 2) out = y[5];
    else if (lane == 3) out = acc[0];
    else if (lane == 4) out = acc[1];
    else if (lane == 5) out = acc[2];
    dyc = out;
    return 0;
}

template <int G>
__global__ void __launch_bounds__(SCOOP_CTA, 3)
nyxb_k_coop_strict(const __grid_constant__ DevSetup S, const __grid_constant__ DevCoopStrict Cs, size_t n,
                   const double* __restrict__ state, const double* __restrict__ consts,
                   const long long* __restrict__ epoch0, long long end_epoch, long long* __restrict__ step_io,
                   double* __restrict__ out_state, long long* __restrict__ out_epoch,
                   nyxb_details* __restrict__ out_details, int* __restrict__ out_status, const DevSink sink) {
    extern __shared__ __align__(16) double ssm[];
    const int tid = threadIdx.x;
    const int lane = tid % G, grp = tid / G;
    const int N = S.grav.N;
    const size_t traj = (size_t)blockIdx.x + (size_t)gridDim.x * grp;  // strided: every SM gets the same share
    if (traj >= n) return;
    double* sm = ssm + (size_t)grp * scoop_traj_stride(N);
    SCtx g;
    g.kst = sm; g.ys = sm + 96; g.ycur = sm + 102; g.nxt = sm + 108; g.er = sm + 114;
    g.rm = sm + SCOOP_FIXED; g.im = g.rm + (N + 2); g.rowres = g.im + (N + 2); g.A = g.rowres + 4 * (N + 1);
    g.hz = 0.0;
    const unsigned lw = tid & 31;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lw - lane));

    const int cidx = lane < 6 ? lane : 0;
    double yc = state[(size_t)cidx * n + traj];
    g.cr = state[6 * n + traj]; g.cd = state[7 * n + traj]; g.pm = state[8 * n + traj];
    g.dry_mass = consts[traj]; g.extra_mass = consts[n + traj]; g.srp_area = consts[2 * n + traj]; g.drag_area = consts[3 * n + traj];
    long long epoch = epoch0[traj];
    long long step_ns = step_io ? step_io[traj] : S.init_step_ns;
    int fixed = S.fixed_step;
    int status = 0, rc = 0;
    long long det_step = S.init_step_ns, n_steps = 0, n_rej = 0, n_rhs = 0;
    double det_error = 0.0;
    int det_attempts = 1;
    // the whole triangle starts at zero: entries never written (column 0, columns beyond M+1) read as the reference's zeros
    for (int k = lane; k < (N + 2) * (N + 3) / 2; k += G) g.A[k] = 0.0;
    if (lane < 6) g.ycur[lane] = yc;
    int ev_count = 0;
    double ev_prev = sink.ev_kind ? event_eval(sink.ev_kind, sink.ev_value, state[traj], state[n + traj], state[2 * n + traj],
                                               state[3 * n + traj], state[4 * n + traj], state[5 * n + traj]) : 0.0;
    if (sink.cap > 0) {  // start state (instance.rs:307, 321)
        if (lane < 6) sink.state[((size_t)lane * sink.cap) * n + traj] = yc;
        if (lane == 6) sink.epoch[traj] = epoch;
    }
    __syncwarp(gmask);

    const int stages = S.tb.stages;
    const long long duration = end_epoch - epoch;
    const long long stop = end_epoch;
    const bool backprop = duration < 0;
    bool done = (duration == 0);
    if (!done && g.pm < 0.0) { rc = NYXB_ERR_FUEL_EXHAUSTED; done = true; }
    if (!done && backprop) step_ns = -step_ns;

    while (!done) {
        // ---- instance.rs:149-196
        bool last = false;
        const long long prev_step = step_ns;
        const int prev_fixed = fixed;
        if (ctl_past_stop(epoch, step_ns, stop, backprop)) {
            if (stop == epoch) break;
            step_ns = stop - epoch;
            fixed = 1;
            last = true;
        }
        // ---- derive(): instance.rs:358-493
        det_attempts = 1;
        double h = dur_to_seconds(step_ns);
        long long dt_ns = 0;
        double nx = 0.0;
        for (;;) {
            double dyc;
            for (int i = 0; i < stages; ++i) {
                if (lane < 6) {
                    double ysv = yc;
                    if (i > 0) {
                        const double* arow = &S.tb.a[(i - 1) * NYXB_MAX_STAGES];
                        double w = 0.0;
                        for (int j = 0; j < i; ++j) w += arow[j] * g.kst[j * 6 + lane];  // zeros included (instance.rs:381-387)
                        ysv = yc + h * w;                                                // instance.rs:394
                    }
                    g.ys[lane] = ysv;
                }
                __syncwarp(gmask);
                g.hz = (i > 0) ? h * 0.0 : 0.0;
                const long long t_ns = (i > 0) ? epoch + dur_from_seconds(S.tb.c[i - 1] * h) : epoch;
                rc = scoop_rhs<G>(S, Cs, g, lane, gmask, t_ns, dyc);
                ++n_rhs;
                if (rc) break;
                if (lane < 6) g.kst[i * 6 + lane] = dyc;
            }
            if (rc) break;
            double er = 0.0;
            nx = yc;
            __syncwarp(gmask);
            if (lane < 6) {
                for (int i = 0; i < stages; ++i) {   // instance.rs:407-414
                    const double ki = g.kst[i * 6 + lane];
                    if (!fixed) er += (h * S.tb.e[i]) * ki;
                    nx += (h * S.tb.b[i]) * ki;
                }
                g.nxt[lane] = nx;
                g.er[lane] = er;
            }
            __syncwarp(gmask);
            if (fixed) { det_step = step_ns; dt_ns = step_ns; break; }
            double e9[9], c9[9], y9[9];
#pragma unroll
            for (int e = 0; e < 6; ++e) { e9[e] = g.er[e]; c9[e] = g.nxt[e]; y9[e] = g.ycur[e]; }
            e9[6] = e9[7] = e9[8] = 0.0;
            y9[6] = g.cr; y9[7] = g.cd; y9[8] = g.pm;
            c9[6] = g.cr + g.hz; c9[7] = g.cd + g.hz; c9[8] = g.pm + g.hz;
            det_error = error_estimate(S.error_ctrl, e9, c9, y9);
            if (ctl_accept(S, det_error, h, det_attempts)) {
                bool bad = false;
#pragma unroll
                for (int e = 0; e < 9; ++e) bad |= (c9[e] != c9[e]);
                if (bad) { rc = NYXB_ERR_PROP_MATH; break; }
                step_ns = ctl_accepted<pow_inv_int>(S, det_error, h, det_attempts, status, det_step);
                dt_ns = det_step;
                break;
            }
            det_attempts += 1;
            n_rej += 1;
            h = ctl_retry<pow_inv_int>(S, det_error, h);
            __syncwarp(gmask);
        }
        if (rc) break;
        epoch += dt_ns;
        __syncwarp(gmask);
        if (lane < 6) { yc = nx; g.ycur[lane] = nx; }
        g.cr = g.cr < 0.0 ? 0.0 : (g.cr > 2.0 ? 2.0 : g.cr);
        n_steps += 1;
        if (n_steps < sink.cap) {  // the channel send of instance.rs:186-193 / 255-259
            if (lane < 6) sink.state[((size_t)lane * sink.cap + (size_t)n_steps) * n + traj] = nx;
            if (lane == 6) sink.epoch[(size_t)n_steps * n + traj] = epoch;
        }
        if (g.pm < 0.0) { rc = NYXB_ERR_FUEL_EXHAUSTED; break; }
        if (sink.ev_kind && !last) {  // stop condition on non-final steps (instance.rs:243-252, event.rs:120-150)
            const double yn = event_eval(sink.ev_kind, sink.ev_value, g.nxt[0], g.nxt[1], g.nxt[2], g.nxt[3], g.nxt[4], g.nxt[5]);
            if (ev_prev * yn < 0.0) ev_count += 1;
            ev_prev = yn;
            if (ev_count >= sink.ev_trigger) break;
        }
        if (last) {
            step_ns = prev_step;
            fixed = prev_fixed;
            if (backprop) step_ns = -step_ns;
            break;
        }
    }
    __syncwarp(gmask);
    if (lane < 6) out_state[(size_t)lane * n + traj] = g.ycur[lane];
    if (lane == 6) {
        out_state[6 * n + traj] = g.cr; out_state[7 * n + traj] = g.cd; out_state[8 * n + traj] = g.pm;
        out_epoch[traj] = epoch;
        if (step_io) step_io[traj] = step_ns;
        out_status[traj] = ctl_finish(sink, traj, status, rc, ev_count, n_steps);
    }
    if (lane == 7 && out_details) {
        nyxb_details d;
        d.step_ns = det_step; d.error = det_error; d.attempts = det_attempts; d._pad = 0;
        d.n_steps = n_steps; d.n_rejected = n_rej; d.n_rhs = n_rhs;
        out_details[traj] = d;
    }
}

template <int G>
static cudaError_t launch_strict_g(const DevSetup* S, const DevCoopStrict* Cs, size_t n, const double* state, const double* consts,
                                   const long long* epoch0, long long end_epoch, long long* step_io, double* out_state,
                                   long long* out_epoch, nyxb_details* out_details, int* out_status, const DevSink* sink,
                                   cudaStream_t stream) {
    const size_t groups = SCOOP_CTA / G;
    const size_t smem = nyxb_coop_strict_smem(S->grav.N, G);
    if (smem > NYXB_COOP_STRICT_SMEM_MAX) return cudaErrorInvalidConfiguration;   // nyxb_engine_set_lanes refuses these first
    cudaError_t e = cudaFuncSetAttribute(nyxb_k_coop_strict<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int dev = 0, sms = 0, occ = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, nyxb_k_coop_strict<G>, SCOOP_CTA, smem);
    if (e != cudaSuccess) return e;
    if (occ < 1) occ = 1;
    size_t grid = (n + groups - 1) / groups;
    if (grid <= (size_t)sms * occ) {
        grid = ((grid + sms - 1) / sms) * sms;
        if (grid * groups < n) grid = (n + groups - 1) / groups;
    }
    nyxb_k_coop_strict<G><<<(unsigned)grid, SCOOP_CTA, smem, stream>>>(*S, *Cs, n, state, consts, epoch0, end_epoch, step_io,
                                                                       out_state, out_epoch, out_details, out_status, *sink);
    return cudaGetLastError();
}

extern "C" cudaError_t nyxb_launch_coop_strict(const DevSetup* S, const DevCoopStrict* Cs, size_t n, const double* state,
                                               const double* consts, const long long* epoch0, long long end_epoch,
                                               long long* step_io, double* out_state, long long* out_epoch,
                                               nyxb_details* out_details, int* out_status, const DevSink* sink,
                                               cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    switch (Cs->G) {
    case 8: return launch_strict_g<8>(S, Cs, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    case 16: return launch_strict_g<16>(S, Cs, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    case 32: return launch_strict_g<32>(S, Cs, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    default: return cudaErrorInvalidValue;
    }
}
