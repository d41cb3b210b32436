// nyxb_od_coop.cu — warp-cooperative sequential Kalman filter (FAST mode): the 32 lanes of a warp run ONE filter.
//
// Why: an orbit-determination ensemble is small (BASELINE configs[4]: 1 000 filters) and every right-hand side carries
// the dual-number spherical-harmonic gradient (GravityField::gradient, gravity_field.rs:273-431: ~2 600 (n, m) entries for
// 70x70, each ~100 FP64 instructions).  One thread per filter leaves the GPU at 32 warps; one WARP per filter gives 1 000
// warps and splits the double sum by COLUMNS of the Legendre triangle:
//   * a lane owns a few columns m (longest-processing-time assignment from the host) and runs the column recursion of
//     A[n][m] and A[n+1][m+1] in dual numbers in registers;
//   * the four partial sums of the reference are regrouped so that everything that depends on n is accumulated first
//     (X_C = sum_n rr_n A[n][m] C_nm, ...) and the per-column constants (cos/sin(m lambda) duals) are applied once per
//     column; one xor-butterfly over the warp adds the lanes (every lane ends with bit-identical sums, so all lanes take
//     the same accept/reject/step decisions without a broadcast);
//   * state, STM, covariance, stage derivatives and stage A-matrices live in shared memory (one slab per warp); the 9x9
//     algebra of the filter (Phi P Phi^T, Joseph update) is spread over the lanes entry by entry.
// Same semantics as the per-thread kernel nyxb_k_od (nyxb_od.cu), which remains the STRICT (oracle-order) path; this
// kernel reorders floating-point sums (tolerance parity, tests/test_gpu_stm_od.py).
#include "nyxb_od_device.cuh"

#define ODC_KMAX 4           // columns per lane (>= ceil((N+1)/32) + 1)
#define ODC_WPB 4            // warps (filters) per block
#define FULL 0xffffffffu

struct WarpS {
    double phi[81], nphi[81];          // STM (column-major like the ABI) and its candidate
    double P[81], T[81], Pb[81], F[81];
    double k[NYXB_MAX_STAGES][6];
    double Ai[NYXB_MAX_STAGES][12];
    double PHt[18], K[18], xdev[9], xhat[9];
};

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ D3 wsum(D3 a) { return D3{wsum(a.v), wsum(a.x), wsum(a.y), wsum(a.z)}; }
__device__ __forceinline__ D3 dfma(D3 acc, D3 t, double c) { return D3{fma(t.v, c, acc.v), fma(t.x, c, acc.x), fma(t.y, c, acc.y), fma(t.z, c, acc.z)}; }

__device__ __forceinline__ D3 dsel(bool c, D3 a, D3 b) { return c ? a : b; }
// complex dual product (ar + i ai)(br + i bi)
__device__ __forceinline__ void cmul(const D3& ar, const D3& ai, const D3& br, const D3& bi, D3& rr, D3& ri) {
    rr = ar * br - ai * bi;
    ri = ar * bi + ai * br;
}

// GravityField::gradient split by columns over the lanes of a warp.  pw: per-warp D3 tables RM/IM/RP of N+2 entries each.
__device__ static void grav_gradient_coop(const DevGrav& g, const int* __restrict__ mycols, long long t_ns, const double r_in[3],
                                          D3* __restrict__ pw, int lane, double acc[3], double Gm[9]) {
    const int N = g.N;
    D3* RM = pw;
    D3* IM = pw + (N + 2);
    D3* RP = pw + 2 * (N + 2);
    double R[9];
    rotation_dcm(g.rot, t_ns, R);
    double rb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = (R[3 * i] * r_in[0] + R[3 * i + 1] * r_in[1]) + R[3 * i + 2] * r_in[2];
    const D3 rx = dvar(rb[0], 0), ry = dvar(rb[1], 1), rz = dvar(rb[2], 2);
    const D3 r_ = dnorm(rx, ry, rz);
    const D3 s_ = rx / r_, t_ = ry / r_, u_ = rz / r_;
    const D3 rho = dc(g.r_eq) / r_;
    {   // powers z^j = (s + i t)^j and (mu / r) rho^(j+1), j = 0..N, in log depth: lane l forms z^l from the binary digits of l
        // (the squarings z, z^2, .., z^16 are uniform), then z^(l+32), z^(l+64), .. by the uniform factor z^32.
        D3 zr = s_, zi = t_, pr = dc(1.0), pi = dc(0.0), qr = rho, qp = dc(1.0);
#pragma unroll 1
        for (int b = 0; b < 5; ++b) {
            D3 nr, ni;
            cmul(pr, pi, zr, zi, nr, ni);
            const bool on = (lane >> b) & 1;
            pr = dsel(on, nr, pr); pi = dsel(on, ni, pi);
            qp = dsel(on, qp * qr, qp);
            cmul(zr, zi, zr, zi, nr, ni);
            zr = nr; zi = ni;
            qr = qr * qr;
        }
        const D3 c0 = (dc(g.mu) / r_) * rho;   // (mu / r) rho^(0+1)
        __syncwarp();
        for (int j = lane; j <= N; j += 32) {
            RM[j] = pr; IM[j] = pi; RP[j] = c0 * qp;
            D3 nr, ni;
            cmul(pr, pi, zr, zi, nr, ni);
            pr = nr; pi = ni;
            qp = qp * qr;
        }
        __syncwarp();
    }
    D3 p0 = dc(0.0), p1 = dc(0.0), p2 = dc(0.0), p3 = dc(0.0);
    const double sq2 = sqrt(2.0);
    for (int kc = 0; kc < ODC_KMAX; ++kc) {
        const int m = mycols[kc];
        if (m < 0) break;
        const int n0 = m > 0 ? m : 1;
        D3 a, am1, b0, b1;
        if (m == 0) {
            am1 = dc(1.0);
            a = dscale(u_, sqrt(3.0));
            b0 = dc(__ldg(g.a_diag + 1));
            b1 = (dc(__ldg(g.offdiag + 1)) * u_) * b0;
        } else {
            am1 = dc(0.0);
            a = dc(__ldg(g.a_diag + m));
            b0 = dc(0.0);
            b1 = dc(__ldg(g.a_diag + m + 1));
        }
        D3 rhop = RP[n0];
        D3 XC = dc(0.0), XS = dc(0.0), YC = dc(0.0), YS = dc(0.0), ZC = dc(0.0), ZS = dc(0.0);
        const DevHarm* rec = g.tab + tri(n0, m);
        for (int n = n0; n <= N; ++n) {
            const double C = __ldg(&rec->cbar), Sv = __ldg(&rec->sbar), v01 = __ldg(&rec->vr01), v11 = __ldg(&rec->vr11);
            const D3 rr = dscale(rhop, g.inv_r_eq);
            const D3 t1 = rr * a;
            XC = dfma(XC, t1, C); XS = dfma(XS, t1, Sv);
            const D3 t2 = dscale(rr * b0, v01);
            YC = dfma(YC, t2, C); YS = dfma(YS, t2, Sv);
            const D3 t3 = dscale(rr * b1, v11);
            ZC = dfma(ZC, t3, C); ZS = dfma(ZS, t3, Sv);
            if (n < N) {
                const DevHarm* rec1 = g.tab + tri(n + 1, m);        // row n+1, column m
                const DevHarm* rec2 = g.tab + tri(n + 2, m + 1);    // row n+2, column m+1
                D3 an, bn;
                if (n == m) {
                    an = (dc(__ldg(g.offdiag + m)) * u_) * a;                                // A[m+1][m]
                    bn = (dc(__ldg(g.offdiag + m + 1)) * u_) * b1;                           // A[m+2][m+1]
                } else {
                    an = dscale(u_, __ldg(&rec1->b)) * a - dscale(am1, __ldg(&rec1->c));
                    bn = dscale(u_, __ldg(&rec2->b)) * b1 - dscale(b0, __ldg(&rec2->c));
                }
                am1 = a; a = an;
                b0 = b1; b1 = bn;
                rhop = rhop * rho;
                rec = rec1;
            }
        }
        const D3 rmm = RM[m], imm = IM[m];
        p2 = p2 + dscale(YC * rmm + YS * imm, sq2);
        p3 = p3 + dscale(ZC * rmm + ZS * imm, sq2);
        if (m > 0) {
            const D3 r1 = RM[m - 1], i1 = IM[m - 1];
            const double mf = (double)m * sq2;
            p0 = p0 + dscale(XC * r1 + XS * i1, mf);
            p1 = p1 + dscale(XS * r1 - XC * i1, mf);
        }
    }
    const D3 a0 = wsum(p0), a1 = wsum(p1), a2 = wsum(p2), a3n = wsum(p3);
    const D3 a3 = D3{-a3n.v, -a3n.x, -a3n.y, -a3n.z};
    const D3 al[3] = { a0 + a3 * s_, a1 + a3 * t_, a2 + a3 * u_ };
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[i] = (R[i] * al[0].v + R[3 + i] * al[1].v) + R[6 + i] * al[2].v;
    double tmp9[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            tmp9[3 * i + j] = (R[i] * dpart(al[0], j) + R[3 + i] * dpart(al[1], j)) + R[6 + i] * dpart(al[2], j);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            Gm[3 * i + j] = (tmp9[3 * i] * R[j] + tmp9[3 * i + 1] * R[3 + j]) + tmp9[3 * i + 2] * R[6 + j];
}

// per-filter scalars, identical in every lane of the warp
struct InstC {
    double y[9];
    long long epoch_ns, step_ns;
    int fixed, status;
    long long det_step_ns;
    double det_error;
    int det_attempts;
    long long n_steps, n_rejected, n_rhs;
    double dry_mass, extra_mass, srp_area;
};

struct Ctx {
    const DevSetup* S;
    const int* mycols;
    D3* pw;
    WarpS* W;
    int lane;
};

// one RHS: stage slot `slot` of the shared k / Ai arrays receives (v, a) and the A-matrix parts
// __noinline__: called from two places in derive_coop; one copy keeps the kernel's instruction footprint (and the
// instruction-cache misses ncu shows as `no_inst` stalls) down
__device__ __noinline__ static int eom_coop(const Ctx& cx, InstC& in, double delta_t_s, const double ys[9], int slot) {
    const DevSetup& S = *cx.S;
    long long t_ns = in.epoch_ns + dur_from_seconds(delta_t_s);
    double yy[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) yy[e] = ys[e];
    yy[6] = yy[6] < 0.0 ? 0.0 : (yy[6] > 2.0 ? 2.0 : yy[6]);
    double mass = in.dry_mass + yy[8] + in.extra_mass;
    if (S.has_srp && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3], Gm[9], gcr[3];
    int rc = dual_eom_dev<false>(S, t_ns, yy, mass, in.srp_area, acc, Gm, gcr);
    in.n_rhs++;
    if (rc) return rc;
    if (S.has_grav) {
        double ga[3], gg[9];
        grav_gradient_coop(S.grav, cx.mycols, t_ns, yy, cx.pw, cx.lane, ga, gg);
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i] += ga[i];
#pragma unroll
        for (int q = 0; q < 9; ++q) Gm[q] += gg[q];
    }
    if (cx.lane == 0) {
        double* k = cx.W->k[slot];
        double* A = cx.W->Ai[slot];
        k[0] = yy[3]; k[1] = yy[4]; k[2] = yy[5]; k[3] = acc[0]; k[4] = acc[1]; k[5] = acc[2];
#pragma unroll
        for (int q = 0; q < 9; ++q) A[q] = Gm[q];
        A[9] = gcr[0]; A[10] = gcr[1]; A[11] = gcr[2];
    }
    __syncwarp();
    return 0;
}

// instance.rs:358-493 (see derive_stm in nyxb_od.cu); the candidate STM goes to W->nphi
__device__ static int derive_coop(const Ctx& cx, InstC& in, long long& dt_ns, double next[9]) {
    const DevSetup& S = *cx.S;
    WarpS& W = *cx.W;
    const int stages = S.tb.stages;
    in.det_attempts = 1;
    double h = dur_to_seconds(in.step_ns);
    for (;;) {
        int rc = eom_coop(cx, in, 0.0, in.y, 0);
        if (rc) return rc;
        for (int i = 0; i < stages - 1; ++i) {
            double wi[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            const double* arow = &S.tb.a[i * NYXB_MAX_STAGES];
            for (int j = 0; j <= i; ++j) {
                double a_ij = arow[j];
                if (a_ij == 0.0) continue;
#pragma unroll
                for (int e = 0; e < 6; ++e) wi[e] += a_ij * W.k[j][e];
            }
            double ys[9];
#pragma unroll
            for (int e = 0; e < 6; ++e) ys[e] = in.y[e] + h * wi[e];
            ys[6] = in.y[6]; ys[7] = in.y[7]; ys[8] = in.y[8];
            rc = eom_coop(cx, in, S.tb.c[i] * h, ys, i + 1);
            if (rc) return rc;
        }
        double err_est[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int e = 0; e < 9; ++e) next[e] = in.y[e];
        for (int i = 0; i < stages; ++i) {
            if (!in.fixed) {
                double cf = h * S.tb.e[i];
#pragma unroll
                for (int e = 0; e < 6; ++e) err_est[e] += cf * W.k[i][e];
            }
            double cb = h * S.tb.b[i];
#pragma unroll
            for (int e = 0; e < 6; ++e) next[e] += cb * W.k[i][e];
        }
        // candidate STM: entry (r, c) = phi(r, c) + sum_i (h b_i) (phi A_i)(r, c), one entry per lane and pass
        bool bad = false;
        for (int e = cx.lane; e < 81; e += 32) {
            const int c = e / 9, r = e - 9 * c;
            double v = W.phi[e];
            if (c < 7) {
                const double p3 = W.phi[27 + r], p4 = W.phi[36 + r], p5 = W.phi[45 + r], pc = (c >= 3 && c < 6) ? W.phi[(c - 3) * 9 + r] : 0.0;
                for (int i = 0; i < stages; ++i) {
                    const double cb = h * S.tb.b[i];
                    const double* Gi = W.Ai[i];
                    double d;
                    if (c < 3) d = (p3 * Gi[c] + p4 * Gi[3 + c]) + p5 * Gi[6 + c];
                    else if (c < 6) d = pc;
                    else d = (p3 * Gi[9] + p4 * Gi[10]) + p5 * Gi[11];
                    v += cb * d;
                }
            }
            W.nphi[e] = v;
            bad = bad || (v != v);
        }
        __syncwarp();
        if (in.fixed) {
            in.det_step_ns = in.step_ns;
            dt_ns = in.step_ns;
            return 0;
        }
        in.det_error = error_estimate(S.error_ctrl, err_est, next, in.y);
        if (ctl_accept(S, in.det_error, h, in.det_attempts)) {
            for (int e = 0; e < 9; ++e) bad = bad || (next[e] != next[e]);
            if (__any_sync(FULL, bad)) return NYXB_ERR_PROP_MATH;
            in.step_ns = ctl_accepted<pow_inv_int>(S, in.det_error, h, in.det_attempts, in.status, in.det_step_ns);
            dt_ns = in.det_step_ns;
            return 0;
        }
        in.det_attempts += 1;
        in.n_rejected += 1;
        h = ctl_retry<pow_inv_int>(S, in.det_error, h);
    }
}

__device__ static int single_step_coop(const Ctx& cx, InstC& in) {
    long long dt;
    double next[9];
    int rc = derive_coop(cx, in, dt, next);
    if (rc) return rc;
    in.epoch_ns += dt;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = next[e];
    for (int e = cx.lane; e < 81; e += 32) cx.W->phi[e] = cx.W->nphi[e];
    __syncwarp();
    in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
    in.n_steps += 1;
    return (in.y[8] < 0.0) ? NYXB_ERR_FUEL_EXHAUSTED : 0;
}

__device__ static int propagate_coop(const Ctx& cx, InstC& in, long long duration_ns) {
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
            int rc = single_step_coop(cx, in);
            if (rc) return rc;
            in.step_ns = prev_step;
            in.fixed = prev_fixed;
            if (backprop) in.step_ns = -in.step_ns;
            return 0;
        }
        int rc = single_step_coop(cx, in);
        if (rc) return rc;
    }
}

// ---- lane-parallel 9x9 algebra on the warp's shared slab (row-major unless noted)
__device__ __forceinline__ void w_identity_phi(WarpS& W, int lane) {
    for (int e = lane; e < 81; e += 32) W.phi[e] = ((e / 9) == (e % 9)) ? 1.0 : 0.0;
    __syncwarp();
}

// Pb = Phi P Phi^T (+ SNC), Phi = W.phi (column-major)
__device__ static void w_covar_bar(const DevOd& od, const InstC& in, long long prev_epoch, WarpS& W, int lane) {
    for (int e = lane; e < 81; e += 32) {   // T = Phi P
        const int r = e / 9, c = e - 9 * r;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) s += W.phi[k * 9 + r] * W.P[k * 9 + c];
        W.T[e] = s;
    }
    __syncwarp();
    for (int e = lane; e < 81; e += 32) {   // Pb = T Phi^T
        const int r = e / 9, c = e - 9 * r;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) s += W.T[r * 9 + k] * W.phi[k * 9 + c];
        W.Pb[e] = s;
    }
    __syncwarp();
    if (od.snc_enabled) {
        long long delta = in.epoch_ns - prev_epoch;
        if (delta <= od.snc_disable_ns) {
            double s[3] = { od.snc_diag[0], od.snc_diag[1], od.snc_diag[2] };
            if (od.snc_frame == 1) {
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
            if (lane < 3) {
                const int i = lane;
                W.Pb[i * 9 + i] += (g1 * s[i]) * g1;
                W.Pb[i * 9 + 3 + i] += (g1 * s[i]) * g2;
                W.Pb[(3 + i) * 9 + i] += (g2 * s[i]) * g1;
                W.Pb[(3 + i) * 9 + 3 + i] += (g2 * s[i]) * g2;
            }
            __syncwarp();
        }
    }
}

__device__ static void w_time_update(const DevOd& od, const InstC& in, long long& prev_epoch, WarpS& W, int lane) {
    w_covar_bar(od, in, prev_epoch, W, lane);
    double nx = 0.0;
    if (lane < 9 && od.variant == NYXB_KF_DEVIATION_TRACKING)
        for (int k = 0; k < 9; ++k) nx += W.phi[k * 9 + lane] * W.xdev[k];
    __syncwarp();
    if (lane < 9) W.xdev[lane] = nx;
    for (int e = lane; e < 81; e += 32) W.P[e] = W.Pb[e];
    __syncwarp();
    prev_epoch = in.epoch_ns;
}

__global__ void __launch_bounds__(32 * ODC_WPB)
nyxb_k_od_coop(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, const int* __restrict__ cols, size_t n,
               const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
               double* __restrict__ out_state, long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details,
               int* __restrict__ out_status) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const size_t i = (size_t)blockIdx.x * ODC_WPB + wib;
    if (i >= n) return;   // whole warps leave together
    const int npw = S.has_grav ? 3 * (S.grav.N + 2) : 0;
    const size_t slab = (sizeof(WarpS) + sizeof(D3) * (size_t)npw + 15) & ~(size_t)15;
    WarpS& W = *reinterpret_cast<WarpS*>(smem + slab * wib);
    Ctx cx;
    cx.S = &S; cx.mycols = cols + lane * ODC_KMAX; cx.W = &W; cx.lane = lane;
    cx.pw = reinterpret_cast<D3*>(smem + slab * wib + sizeof(WarpS));
    InstC in;
#pragma unroll
    for (int e = 0; e < 9; ++e) in.y[e] = state[(size_t)e * n + i];
    in.dry_mass = consts[i]; in.extra_mass = consts[n + i]; in.srp_area = consts[2 * n + i];
    in.epoch_ns = epoch0[i];
    in.step_ns = S.init_step_ns;
    in.fixed = S.fixed_step;
    in.status = 0;
    in.det_step_ns = S.init_step_ns; in.det_error = 0.0; in.det_attempts = 1;
    in.n_steps = 0; in.n_rejected = 0; in.n_rhs = 0;
    if (!in.fixed) in.step_ns = od.max_step_ns;
    for (int e = lane; e < 81; e += 32) {
        const int r = e / 9, c = e - 9 * r;
        W.P[e] = od.covar0[(size_t)(c * 9 + r) * n + i];
    }
    if (lane < 9) W.xdev[lane] = 0.0;
    w_identity_phi(W, lane);
    long long prev_epoch = in.epoch_ns;
    long long epoch = in.epoch_ns;
    int rc = 0;
    const bool ekf = od.variant == NYXB_KF_REFERENCE_UPDATE;
    const int M = od.msr_size;
    for (long long k = 0; k < od.n_msr && rc == 0; ++k) {
        const long long t_k = od.msr_epoch[k];
        const double o[2] = { od.obs[((size_t)k * 2 + 0) * n + i], od.obs[((size_t)k * 2 + 1) * n + i] };
        int flags = 0;
        if (o[0] != o[0] && o[1] != o[1]) {
            if (od.flags && lane == 0) od.flags[(size_t)k * n + i] = NYXB_MSRF_ABSENT;
            continue;
        }
        for (;;) {
            long long delta_t = t_k - epoch;
            long long next_step = delta_t;
            if (in.step_ns < next_step) next_step = in.step_ns;
            if (od.max_step_ns < next_step) next_step = od.max_step_ns;
            rc = propagate_coop(cx, in, next_step);
            if (rc) break;
            epoch = in.epoch_ns;
            long long gap = in.epoch_ns - t_k;
            if (gap < 0) gap = -gap;
            if (gap < od.eps_ns) {
                in.epoch_ns = t_k;
                const int trk = od.msr_tracker[k];
                if (trk < 0 || trk >= od.n_stations) break;
                const DevStation& gs = od.stations[trk];
                const int windows = gs.n_types / M;
                for (int wno = 0; wno <= windows; ++wno) {
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
                    // ---- measurement_update
                    w_covar_bar(od, in, prev_epoch, W, lane);
                    if (lane < 18) {   // PHt[r][q], r = lane / 2, q = lane % 2
                        const int r = lane >> 1, q = lane & 1;
                        double s = 0.0;
                        if (q < M)
                            for (int c = 0; c < 9; ++c) s += W.Pb[r * 9 + c] * H[q][c];
                        W.PHt[lane] = s;
                    }
                    __syncwarp();
                    double Sk[2][2] = { {0.0, 0.0}, {0.0, 0.0} }, pre[2] = { 0.0, 0.0 };
                    for (int a = 0; a < M; ++a)
                        for (int b = 0; b < M; ++b) {
                            double s = 0.0;
                            for (int c = 0; c < 9; ++c) s += H[a][c] * W.PHt[c * 2 + b];
                            Sk[a][b] = s + ((a == b) ? Rk[a] : 0.0);
                        }
                    for (int q = 0; q < M; ++q) pre[q] = real_obs[q] - comp[q];
                    double ratio;
                    if (!od_ratio(M, Sk, Rk, pre, ratio)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularNoiseRk
                    const int rslot = (M == 1) ? wno : 0;
                    if (lane == 0) {
                        if (od.ratio) od.ratio[((size_t)k * 2 + rslot) * n + i] = ratio;
                        if (od.prefit) for (int q = 0; q < ncur; ++q) od.prefit[((size_t)k * 2 + wno * M + q) * n + i] = pre[q];
                    }
                    flags |= NYXB_MSRF_PROCESSED;
                    if (od.reject >= 0.0 && ratio > od.reject) {
                        w_time_update(od, in, prev_epoch, W, lane);
                        flags |= NYXB_MSRF_REJECTED;
                    } else {
                        double Si[2][2];
                        if (!od_sinv(M, Sk, Si)) { rc = NYXB_ERR_PROP_MATH; break; }   // SingularKalmanGain
                        if (lane < 18) {   // K[r][q]
                            const int r = lane >> 1, q = lane & 1;
                            double s = 0.0;
                            if (q < M)
                                for (int b = 0; b < M; ++b) s += W.PHt[r * 2 + b] * Si[b][q];
                            W.K[lane] = s;
                        }
                        __syncwarp();
                        double post[2] = { 0.0, 0.0 };
                        // xhat (uniform): every lane computes all nine (cheap) so that the state replacement stays in registers
                        double xhat[9];
                        if (ekf) {
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += W.K[r * 2 + q] * pre[q]; xhat[r] = s; }
                            for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xhat[c]; post[q] = pre[q] - s; }
                        } else {
                            double xbar[9];
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int c = 0; c < 9; ++c) s += W.phi[c * 9 + r] * W.xdev[c]; xbar[r] = s; }
                            for (int q = 0; q < M; ++q) { double s = 0.0; for (int c = 0; c < 9; ++c) s += H[q][c] * xbar[c]; post[q] = pre[q] - s; }
                            for (int r = 0; r < 9; ++r) { double s = 0.0; for (int q = 0; q < M; ++q) s += W.K[r * 2 + q] * post[q]; xhat[r] = xbar[r] + s; }
                        }
                        __syncwarp();
                        for (int e = lane; e < 81; e += 32) {   // F = I - K H
                            const int r = e / 9, c = e - 9 * r;
                            double s = 0.0;
                            for (int q = 0; q < M; ++q) s += W.K[r * 2 + q] * H[q][c];
                            W.F[e] = ((r == c) ? 1.0 : 0.0) - s;
                        }
                        __syncwarp();
                        for (int e = lane; e < 81; e += 32) {   // T = F Pb
                            const int r = e / 9, c = e - 9 * r;
                            double s = 0.0;
#pragma unroll
                            for (int kk = 0; kk < 9; ++kk) s += W.F[r * 9 + kk] * W.Pb[kk * 9 + c];
                            W.T[e] = s;
                        }
                        __syncwarp();
                        for (int e = lane; e < 81; e += 32) {   // Pb <- T F^T + K R K^T   (Pb is dead after T)
                            const int r = e / 9, c = e - 9 * r;
                            double s = 0.0;
#pragma unroll
                            for (int kk = 0; kk < 9; ++kk) s += W.T[r * 9 + kk] * W.F[c * 9 + kk];
                            double s2 = 0.0;
                            for (int q = 0; q < M; ++q) s2 += (W.K[r * 2 + q] * Rk[q]) * W.K[c * 2 + q];
                            W.nphi[e] = s + s2;   // scratch (the STM is reset right after)
                        }
                        __syncwarp();
                        for (int e = lane; e < 81; e += 32) {
                            const int r = e / 9, c = e - 9 * r;
                            W.P[e] = 0.5 * (W.nphi[e] + W.nphi[c * 9 + r]);
                        }
                        if (lane < 9) W.xdev[lane] = xhat[lane];
                        __syncwarp();
                        prev_epoch = in.epoch_ns;
                        if (lane == 0 && od.postfit) for (int q = 0; q < ncur; ++q) od.postfit[((size_t)k * 2 + wno * M + q) * n + i] = post[q];
                        if (ekf) {
                            for (int r = 0; r < 9; ++r) in.y[r] = in.y[r] + xhat[r];
                            in.y[6] = in.y[6] < 0.0 ? 0.0 : (in.y[6] > 2.0 ? 2.0 : in.y[6]);
                        }
                    }
                    w_identity_phi(W, lane);
                }
                if (lane < 9) {
                    if (od.est_state) od.est_state[((size_t)k * 9 + lane) * n + i] = in.y[lane];
                    if (od.est_cov) od.est_cov[((size_t)k * 9 + lane) * n + i] = W.P[lane * 9 + lane];
                }
                break;
            } else {
                w_time_update(od, in, prev_epoch, W, lane);
                w_identity_phi(W, lane);
            }
        }
        if (od.flags && lane == 0) od.flags[(size_t)k * n + i] = flags;
    }
    __syncwarp();
    for (int e = lane; e < 81; e += 32) {
        const int r = e / 9, c = e - 9 * r;
        od.covar[(size_t)(c * 9 + r) * n + i] = W.P[e];
    }
    if (lane < 9) {
        if (od.state_dev) od.state_dev[(size_t)lane * n + i] = W.xdev[lane];
        out_state[(size_t)lane * n + i] = in.y[lane];
    }
    if (lane == 0) {
        out_epoch[i] = in.epoch_ns;
        if (out_details) {
            nyxb_details d;
            d.step_ns = in.det_step_ns; d.error = in.det_error; d.attempts = in.det_attempts; d._pad = 0;
            d.n_steps = in.n_steps; d.n_rejected = in.n_rejected; d.n_rhs = in.n_rhs;
            out_details[i] = d;
        }
        out_status[i] = (in.status & NYXB_WARN_MAX_ATTEMPTS) | rc;
    }
}

extern "C" size_t nyxb_od_coop_smem_bytes(int degree_or_zero) {
    const size_t npw = degree_or_zero > 0 ? 3 * (size_t)(degree_or_zero + 2) : 0;
    const size_t slab = (sizeof(WarpS) + sizeof(D3) * npw + 15) & ~(size_t)15;
    return slab * ODC_WPB;
}

extern "C" int nyxb_od_coop_kmax(void) { return ODC_KMAX; }

extern "C" cudaError_t nyxb_launch_od_coop(const DevSetup* S, const DevOd* od, const int* cols, size_t n, const double* state,
                                           const double* consts, const long long* epoch0, double* out_state, long long* out_epoch,
                                           nyxb_details* out_details, int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const size_t smem = nyxb_od_coop_smem_bytes(S->has_grav ? S->grav.N : 0);
    cudaError_t e = cudaFuncSetAttribute(nyxb_k_od_coop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    unsigned grid = (unsigned)((n + ODC_WPB - 1) / ODC_WPB);
    nyxb_k_od_coop<<<grid, 32 * ODC_WPB, smem, stream>>>(*S, *od, cols, n, state, consts, epoch0, out_state, out_epoch, out_details,
                                                         out_status);
    return cudaGetLastError();
}
