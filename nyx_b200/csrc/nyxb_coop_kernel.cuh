// nyxb_coop_kernel.cuh — lane-cooperative, register-blocked propagation kernel (FAST mode).
//
//   * G lanes of one warp integrate one trajectory together.  The spherical-harmonic
//     double sum (gravity_field.rs:217-249; >98 % of the arithmetic for a 21x21 field) is split across
//     the lanes by COLUMNS of the derived-Legendre triangle: every A[n][m] is produced by its own column
//     recursion (gravity_field.rs:175-181) in a register, and the four partial sums are regrouped so that
//     each A[n][m] is consumed exactly once, by the lane that produced it:
//         X += rr_n   m A[n][m] E(n,m)               Y += rr_n m A[n][m] F(n,m)
//         Z += rr_n   vr01[n][m-1] A[n][m] D(n,m-1)   W -= rr_{n-1} vr11[n-1][m-1] A[n][m] D(n-1,m-1)
//     (E, F, D share the per-column constant (cos,sin)((m-1) lambda)): no A matrix in memory, no cross-lane
//     traffic inside the sum, one butterfly reduction at the end.
//   * The shared-memory return path (128 B/clk/SM) is the scarce resource of this loop, so the per-entry record is
//     compressed to 40 bytes: the column recursion runs on the un-normalised Q[n][m] = (n-m)! d^m P_n/du^m whose
//     coefficients (2n+1), (n+m)(n-m) are generated in registers, the normalisation is folded into the stored
//     coefficients, and the W term reuses the Z term of the entry above (one ratio instead of two coefficients).
//     The record is fetched ONCE (2 x LDS.128 + LDS.64 from the TMA-staged table).
//   * RK stage vectors live in shared memory ([stage][6] per trajectory), lane c < 6 owns state component c;
//     the error norm and the step-size controller are evaluated redundantly by every lane of the group.
//   * The trajectory of a group advances by ONE step attempt per outer iteration; a rejected attempt simply
//     retries in the next iteration while the other groups of the warp move on (derive() loop, instance.rs:358-493).
//   * HBM is touched only to read the initial state and write the final one.
//
// Reference behaviour: instance.rs:87-262, 343-352, 358-493 (propagate/single_step/derive) and
// spacecraft.rs:191-310 (eom).  FMA contraction and the regrouped summation make this a tolerance-parity
// path (tests assert < 1e-6 km, the north-star's sub-mm bound; 5e-9 km with a fixed step).
#pragma once
#include "nyxb_coop.h"

#ifndef COOP_CTA
#define COOP_CTA 128
#endif
#define COOP_SM_FIXED 122  // kst[16*6] + ys[6] + ycur[6] + nxt[6] + er[6] + event {previous value, crossings}

// doubles of shared memory per trajectory, padded to 8 (mod 16) doubles so that consecutive trajectories
// start 64 B apart modulo the 128-B bank row instead of on the same banks
__host__ __device__ inline int coop_traj_stride(int N) {
    int s = COOP_SM_FIXED + 3 * (N + 3);
    return s + ((8 - (s & 15)) & 15);
}
// bytes of the CTA-shared table region: records [(L+2)/2 pairs][5 x 16 B][G], then colseed[N+3][4] (row N+2 zero: the seed of
// the stop column, see nyxb_coop_build_host), col_start/col_m [G][kmax+2]
__host__ __device__ inline size_t coop_rec_bytes(int L, int G) { return (size_t)(L + 2) * G * NYXB_COOP_REC_BYTES; }
__host__ __device__ inline size_t coop_meta_bytes(int N, int G, int kmax) {
    size_t b = (size_t)(N + 3) * 32 + (size_t)2 * G * (kmax + 2) * 4;
    return (b + 15) & ~(size_t)15;
}

__device__ __forceinline__ double shfl_d(unsigned mask, double v, int src, int width) { return __shfl_sync(mask, v, src, width); }
__device__ __forceinline__ double shfl_xor_d(unsigned mask, double v, int lanemask, int width) { return __shfl_xor_sync(mask, v, lanemask, width); }

__device__ __forceinline__ double lds_f64(unsigned addr) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ int lds_s32(unsigned addr) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// per-trajectory view of the group's shared memory + constants of motion
struct TrajCtx {
    double* kst; double* ys; double* ycur; double* nxt; double* er;
    double* ev;  // [0] previous event value, [1] crossings so far (kept out of registers: cold path)
    double* rm; double* im; double* rp;
    double dry_mass, extra_mass, srp_area, drag_area;
    double cr, cd, pm;  // y[6..8]: constant without guidance (spacecraft.rs:248)
    double hz;          // h * 0.0 of the current attempt: NaN-propagating stand-in for y[6..8] + h*0 (instance.rs:394)
};

// sin/cos of the three orientation angles at the step epoch; the per-stage DCM is obtained by a first-order
// update of the (slow) pole angles and an exact angle addition for the prime-meridian angle W.
struct RotBase { double sa, ca, sd, cd, sw, cw; };

// Cooperative SpacecraftDynamics::eom for the stage state held in g.ys; lane c < 6 receives dy[c].  Returns 0 or an nyxb_status error.
template <int G, bool NC>   // NC ("general fields"): the primary field may belong to another body, further fields may exist
__device__ __forceinline__ int coop_rhs(const DevSetup& S, const double* __restrict__ recs, int L,
                                        const double* __restrict__ colseed, unsigned a_cs, unsigned cm_off,
                                        TrajCtx& g, const RotBase& rb, double dt_s, long long t_ns, int lane, double& dyc) {
    constexpr unsigned FULL = 0xffffffffu;  // the caller keeps the warp converged (see nyxb_k_coop)
    const DevGrav& gv = S.grav;
    const double ra_dot = gv.rot.ra_dot, dec_dot = gv.rot.dec_dot;  // rad/s, precomputed on the host
    double inv_r, rho, ub, r2;
    {
        // ---- inertial -> body-fixed DCM at the stage time (angle addition from the step-epoch base)
        double R[9];
        if (gv.rot.kind == 0) {
            R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        } else {
            const double da = ra_dot * dt_s, dd = dec_dot * dt_s, dw = gv.rot.wdot * dt_s;
            const double sa = fma(rb.ca, da, rb.sa), ca = fma(-rb.sa, da, rb.ca);
            const double sd = fma(rb.cd, dd, rb.sd), cd = fma(-rb.sd, dd, rb.cd);
            double sdl, cdl;
            if (fabs(dw) < 0.02) {
                const double z = dw * dw;
                sdl = dw * fma(z, fma(z, 1.0 / 120.0, -1.0 / 6.0), 1.0);
                cdl = fma(z, fma(z, fma(z, -1.0 / 720.0, 1.0 / 24.0), -0.5), 1.0);
            } else {
                det_sincos(dw, sdl, cdl);
            }
            const double sw = fma(rb.sw, cdl, rb.cw * sdl), cw = fma(rb.cw, cdl, -(rb.sw * sdl));
            const double b00 = -sa, b01 = ca;
            const double b10 = -(sd * ca), b11 = -(sd * sa), b12 = cd;
            R[0] = fma(cw, b00, sw * b10); R[1] = fma(cw, b01, sw * b11); R[2] = sw * b12;
            R[3] = fma(cw, b10, -(sw * b00)); R[4] = fma(cw, b11, -(sw * b01)); R[5] = cw * b12;
            R[6] = cd * ca; R[7] = cd * sa; R[8] = sd;
        }
        double y0 = g.ys[0], y1 = g.ys[1], y2 = g.ys[2];
        if (NC && S.grav_body >= 0) field_offset(S, t_ns, y0, y1, y2);   // field of another body: the state is translated to it first
        const double rb0 = fma(R[2], y2, fma(R[1], y1, R[0] * y0));
        const double rb1 = fma(R[5], y2, fma(R[4], y1, R[3] * y0));
        const double rb2 = fma(R[8], y2, fma(R[7], y1, R[6] * y0));
        inv_r = rsqrt(fma(rb2, rb2, fma(rb1, rb1, rb0 * rb0)));  // one Newton chain instead of sqrt + division
        rho = gv.r_eq * inv_r;
        ub = (rb2 * inv_r) * rho;
        r2 = rho * rho;
        // park the DCM in the trajectory's scratch (nxt/er are idle during the stages): it is needed again only
        // after the column walk, and keeping it in registers would push the walk's live set past the occupancy target
        if (lane == 0) {
#pragma unroll
            for (int q = 0; q < 9; ++q) g.nxt[q] = R[q];
        }
        // power tables (cos,sin)(k lambda) cos^k(phi) and rho^k A[k][k]: lane computes k = lane, lane+G, ...
        double zr = 1.0, zi = 0.0, pr = 1.0;
        double bzr = rb0 * inv_r, bzi = rb1 * inv_r, bp = rho;
#pragma unroll
        for (int bit = 1; bit < G; bit <<= 1) {
            if (lane & bit) {
                const double nzr = fma(zr, bzr, -(zi * bzi));
                zi = fma(zr, bzi, zi * bzr);
                zr = nzr;
                pr *= bp;
            }
            const double nb = fma(bzr, bzr, -(bzi * bzi));
            bzi = 2.0 * bzr * bzi;
            bzr = nb;
            bp *= bp;
        }
        const int top = gv.N + 2;   // N + 2: the stop column's (zero) seed
        for (int k = lane; k <= top; k += G) {
            g.rm[k] = zr; g.im[k] = zi; g.rp[k] = pr * colseed[4 * k];  // rho^k (2k-1)!!: the seed Q[k][k] of column k
            const double nzr = fma(zr, bzr, -(zi * bzi));
            zi = fma(zr, bzi, zi * bzr);
            zr = nzr;
            pr *= bp;
        }
    }
    __syncwarp(FULL);

    // ---- column walk, two entries per iteration.  Per pair: one 80-byte record (5 x LDS.128) and 26 FP64 instructions;
    // the recursion coefficients (2n+1) and (n+m)(n-m) are generated in registers.  The per-column sums
    // S1..S6 carry no (cos, sin)((m-1) lambda) factor: it is applied once, when the lane switches to its next column
    // (columns have an even number of entries, so the switch is tested once per pair).  Loop invariants are pinned with
    // empty asm: ptxas otherwise rematerialises them inside the loop.
    unsigned a_rm = smem_u32(g.rm), a_seed = smem_u32(colseed);
    asm volatile("" : "+r"(a_rm), "+r"(a_cs), "+r"(a_seed));
    asm volatile("" : "+d"(r2), "+d"(ub));
    const unsigned pw8 = (unsigned)(gv.N + 3) * 8u;  // rm -> im -> rp stride in bytes
    double X = 0.0, Y = 0.0, Z = 0.0, W = 0.0, Q1 = 0.0, Q2 = 0.0, rr = 0.0, ii = 0.0;
    double S1 = 0.0, S2 = 0.0, S3 = 0.0, S4 = 0.0, S5 = 0.0, S6 = 0.0;
    double al = 0.0, be = 0.0;
    int ci = 0;
    int next_start = lds_s32(a_cs);
    unsigned a_col = a_rm + lds_s32(a_cs + cm_off) * 8;  // &rm[m] of the lane's next column
    const double2* rec = reinterpret_cast<const double2*>(recs) + lane;  // five 16-byte pieces per pair and lane
    // Software pipeline over two register sets (A, B): the records of the NEXT pair are requested before the current
    // pair is consumed, so no LDS latency is exposed; the macro is instantiated twice to avoid register-rotation moves.
#define COOP_WALK_PAIR(a0, a1, b0, b1, kk, na0, na1, nb0, nb1, nkk)                                                     \
    {                                                                                                                   \
        if (e == next_start) {                                                                                          \
            /* column switch (about three per lane and RHS): seeds are loaded here, not prefetched */                   \
            ++ci;                                                                                                       \
            const unsigned a_sd = a_seed + ((a_col - a_rm) >> 3) * 32;                                                  \
            const double pd1 = lds_f64(a_sd + 8), pd2 = lds_f64(a_sd + 16);                                             \
            al = lds_f64(a_sd + 24); be = 0.0;                                                                          \
            const double q = lds_f64(a_col + 2 * pw8), rn = lds_f64(a_col - 8), in_ = lds_f64(a_col + pw8 - 8);         \
            /* close the previous column: apply its (cos, sin)((m-1) lambda) */                                         \
            X = fma(rr, S1, fma(ii, S2, X));                                                                            \
            Y = fma(rr, S2, fma(-ii, S1, Y));                                                                           \
            Z = fma(rr, S3, fma(ii, S4, Z));                                                                            \
            W = fma(rr, S5, fma(ii, S6, W));                                                                            \
            Q1 = q; rr = rn; ii = in_; Q2 = 0.0;                                                                        \
            S1 = S2 = S3 = S4 = 0.0;                                                                                    \
            S5 = q * pd1; S6 = q * pd2; /* W term of the column's first degree (seed record, kappa = 1) */              \
            next_start = lds_s32(a_cs + ci * 4);                /* sentinel L+1 after the last column */                \
            a_col = a_rm + lds_s32(a_cs + cm_off + ci * 4) * 8; /* sentinel column 1 */                                 \
        }                                                                                                               \
        rec += 5 * G;                                                                                                   \
        na0 = rec[0]; na1 = rec[G]; nb0 = rec[2 * G]; nb1 = rec[3 * G]; nkk = rec[4 * G]; /* table ends with a null pair */ \
        const double be1 = be + al, al1 = al + 2.0; /* (n+1)^2 - m^2 = n^2 - m^2 + (2n+1) */                             \
        /* entry a (degree n): Q1 = Q[n], Q2 = Q[n-1] */                                                                \
        S1 = fma(Q1, a0.x, S1);                                                                                         \
        S2 = fma(Q1, a0.y, S2);                                                                                         \
        S3 = fma(Q1, a1.x, S3);                                                                                         \
        S4 = fma(Q1, a1.y, S4);                                                                                         \
        const double Qa = fma(al * ub, Q1, -((be * r2) * Q2)); /* Q[n+1] = (2n+1) u Q[n] - (n+m)(n-m) Q[n-1] */         \
        const double wa = kk.x * Qa;                                                                                    \
        S5 = fma(wa, a1.x, S5);                                                                                         \
        S6 = fma(wa, a1.y, S6);                                                                                         \
        /* entry b (degree n+1) */                                                                                      \
        S1 = fma(Qa, b0.x, S1);                                                                                         \
        S2 = fma(Qa, b0.y, S2);                                                                                         \
        S3 = fma(Qa, b1.x, S3);                                                                                         \
        S4 = fma(Qa, b1.y, S4);                                                                                         \
        const double Qb = fma(al1 * ub, Qa, -((be1 * r2) * Q1));                                                        \
        const double wb = kk.y * Qb;                                                                                    \
        S5 = fma(wb, b1.x, S5);                                                                                         \
        S6 = fma(wb, b1.y, S6);                                                                                         \
        Q2 = Qa;                                                                                                        \
        Q1 = Qb;                                                                                                        \
        be = be1 + al1;                                                                                                 \
        al = al1 + 2.0;                                                                                                 \
        e += 2;                                                                                                         \
    }
    double2 A0 = rec[0], A1 = rec[G], A2 = rec[2 * G], A3 = rec[3 * G], A4 = rec[4 * G];
    double2 B0, B1, B2, B3, B4;
    int e = 0;
#pragma unroll 1
    while (e < L) {
        COOP_WALK_PAIR(A0, A1, A2, A3, A4, B0, B1, B2, B3, B4)
        if (e >= L) break;
        COOP_WALK_PAIR(B0, B1, B2, B3, B4, A0, A1, A2, A3, A4)
    }
#undef COOP_WALK_PAIR
    // close the last column
    X = fma(rr, S1, fma(ii, S2, X));
    Y = fma(rr, S2, fma(-ii, S1, Y));
    Z = fma(rr, S3, fma(ii, S4, Z));
    W = fma(rr, S5, fma(ii, S6, W));
#pragma unroll
    for (int off = G / 2; off >= 1; off >>= 1) {
        X += shfl_xor_d(FULL, X, off, G);
        Y += shfl_xor_d(FULL, Y, off, G);
        Z += shfl_xor_d(FULL, Z, off, G);
        W += shfl_xor_d(FULL, W, off, G);
    }
    // ---- reload the stage state and the DCM, assemble the acceleration
    double y[9];
#pragma unroll
    for (int e = 0; e < 6; ++e) y[e] = g.ys[e];
    y[6] = g.cr + g.hz; y[7] = g.cd + g.hz; y[8] = g.pm + g.hz;
    double R[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) R[q] = g.nxt[q];
    double s_, t_, u_;
    if (NC) {
        double q0 = y[0], q1 = y[1], q2 = y[2];   // position relative to the field's body
        if (S.grav_body >= 0) field_offset(S, t_ns, q0, q1, q2);
        s_ = fma(R[2], q2, fma(R[1], q1, R[0] * q0)) * inv_r;
        t_ = fma(R[5], q2, fma(R[4], q1, R[3] * q0)) * inv_r;
        u_ = fma(R[8], q2, fma(R[7], q1, R[6] * q0)) * inv_r;
    } else {
        s_ = fma(R[2], y[2], fma(R[1], y[1], R[0] * y[0])) * inv_r;
        t_ = fma(R[5], y[2], fma(R[4], y[1], R[3] * y[0])) * inv_r;
        u_ = fma(R[8], y[2], fma(R[7], y[1], R[6] * y[0])) * inv_r;
    }
    // rr_n A[n][m] = K0 rho (rho^n A),  rr_{n-1} A[n][m] = K0 (rho^n A),  K0 = mu / (r R_eq)
    const double K0 = (gv.mu * gv.inv_r_eq) * inv_r;
    const double K1 = K0 * rho;
    const double aw = -K0 * W;
    const double ab0 = fma(aw, s_, K1 * X), ab1 = fma(aw, t_, K1 * Y), ab2 = fma(aw, u_, K1 * Z);
    // two-body (orbital.rs:86-92): from the same 1/r when the field belongs to the centre
    const double ir_c = (NC && S.grav_body >= 0) ? rsqrt(fma(y[2], y[2], fma(y[1], y[1], y[0] * y[0]))) : inv_r;
    const double fac = -S.mu_central * ir_c * ir_c * ir_c;
    double acc[3];
    acc[0] = fma(fac, y[0], fma(R[6], ab2, fma(R[3], ab1, R[0] * ab0)));
    acc[1] = fma(fac, y[1], fma(R[7], ab2, fma(R[4], ab1, R[1] * ab0)));
    acc[2] = fma(fac, y[2], fma(R[8], ab2, fma(R[5], ab1, R[2] * ab0)));
    int rc = 0;
    if (S.n_bodies > 0 || S.has_srp || S.has_drag || (NC && S.n_xgrav > 0)) {
        // cold path: private copies, so that y/acc of the common path are never address-taken (they stay in registers)
        double yy[9], aa[3];
#pragma unroll
        for (int e = 0; e < 9; ++e) yy[e] = y[e];
        aa[0] = acc[0]; aa[1] = acc[1]; aa[2] = acc[2];
        rc = accel_cold<NC>(S, g.dry_mass, g.extra_mass, g.srp_area, g.drag_area, t_ns, yy, aa);
        acc[0] = aa[0]; acc[1] = aa[1]; acc[2] = aa[2];
    }
    // lane c < 3 keeps the velocity component c, lanes 3..5 the acceleration components (selects, no jump table)
    const int c3 = lane >= 3 ? lane - 3 : lane;
    const double vsel = c3 == 0 ? y[3] : (c3 == 1 ? y[4] : y[5]);
    const double asel = c3 == 0 ? acc[0] : (c3 == 1 ? acc[1] : acc[2]);
    dyc = lane >= 3 ? asel : vsel;
    return rc;
}

template <int G, bool SMEM_TABLE, bool NC = false>
#ifndef COOP_MINB1
#define COOP_MINB1 5
#endif
__global__ void __launch_bounds__(COOP_CTA, COOP_MINB1)
nyxb_k_coop(const __grid_constant__ DevSetup S, const __grid_constant__ DevCoop Cp, size_t n,
            const double* __restrict__ state, const double* __restrict__ consts,
            const long long* __restrict__ epoch0, long long end_epoch, long long* __restrict__ step_io,
            double* __restrict__ out_state, long long* __restrict__ out_epoch,
            nyxb_details* __restrict__ out_details, int* __restrict__ out_status, const DevSink sink) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long tma_bar;
    const int tid = threadIdx.x;
    const int lane = tid % G, grp = tid / G;
    const int N = S.grav.N;

    // ---- CTA-shared tables: records via one TMA bulk copy (SMEM_TABLE), small metadata via plain loads
    const size_t rec_bytes = SMEM_TABLE ? coop_rec_bytes(Cp.L, G) : 0;
    unsigned char* meta = smem_raw + rec_bytes;
    double* sm_seed = reinterpret_cast<double*>(meta);
    int* sm_cs = reinterpret_cast<int*>(meta + (size_t)(N + 3) * 32);
    int* sm_cm = sm_cs + G * (Cp.kmax + 2);
    if (SMEM_TABLE) {
        if (tid == 0) mbar_init(&tma_bar, 1);
        __syncthreads();
        if (tid == 0) {
            mbar_expect_tx(&tma_bar, (unsigned)rec_bytes);
            tma_bulk_g2s(smem_raw, Cp.recs, (unsigned)rec_bytes, &tma_bar);
        }
    }
    for (int k = tid; k < (N + 3) * 4; k += COOP_CTA) sm_seed[k] = k < (N + 2) * 4 ? __ldg(Cp.colseed + k) : 0.0;
    for (int k = tid; k < G * (Cp.kmax + 2); k += COOP_CTA) {
        const int l = k / (Cp.kmax + 2), q = k % (Cp.kmax + 2);
        sm_cs[k] = (q < Cp.kmax) ? __ldg(Cp.col_start + l * Cp.kmax + q) : Cp.L + 1;
        sm_cm[k] = (q < Cp.kmax) ? __ldg(Cp.col_m + l * Cp.kmax + q) : 1;
    }
    if (SMEM_TABLE) mbar_wait(&tma_bar, 0);
    __syncthreads();
    const double* recs = SMEM_TABLE ? reinterpret_cast<const double*>(smem_raw) : Cp.recs;
    const unsigned a_cs = smem_u32(sm_cs + lane * (Cp.kmax + 2));
    const unsigned cm_off = (unsigned)(G * (Cp.kmax + 2) * 4);

    // ---- the trajectory of this group: whole warps are strided over the grid (every SM gets the same number of FULL warps,
    // surplus warps exit)
    const int gpw = 32 / G;
    const size_t traj0 = ((size_t)blockIdx.x + (size_t)gridDim.x * (tid >> 5)) * gpw;  // first trajectory of this WARP
    if (traj0 >= n) return;  // uniform per warp; no block-wide barrier below this point
    // The control flow below is WARP-uniform: every group of the warp runs the same sequence of attempts until all of them
    // are done (a finished or absent group keeps executing on its own scratch without committing anything), so all
    // synchronisation uses the full mask -- sub-warp masks cost a MATCH/REDUX/VOTE sequence per shuffle group.
    const size_t traj_raw = traj0 + (tid & 31) / G;
    const bool valid = traj_raw < n;
    const size_t traj = valid ? traj_raw : 0;  // an absent group shadows trajectory 0 and is never committed
    const int tstride = coop_traj_stride(N);
    double* sm = reinterpret_cast<double*>(meta + coop_meta_bytes(N, G, Cp.kmax)) + (size_t)grp * tstride;
    const int pw = N + 3;
    const unsigned lw = tid & 31;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lw - lane));  // cold, group-divergent paths only
    constexpr unsigned FULL = 0xffffffffu;

    TrajCtx g;
    g.kst = sm; g.ys = sm + 96; g.ycur = sm + 102; g.nxt = sm + 108; g.er = sm + 114; g.ev = sm + 120;
    g.rm = sm + COOP_SM_FIXED; g.im = g.rm + pw; g.rp = g.im + pw;
    g.hz = 0.0;
    // every lane of the group reads the same addresses (broadcast within the request)
    const int cidx = lane < 6 ? lane : 0;
    double yc = state[(size_t)cidx * n + traj];
    g.cr = state[6 * n + traj]; g.cd = state[7 * n + traj]; g.pm = state[8 * n + traj];
    g.dry_mass = consts[traj]; g.extra_mass = consts[n + traj];
    g.srp_area = consts[2 * n + traj]; g.drag_area = consts[3 * n + traj];
    long long epoch = epoch0[traj];
    long long step_ns = step_io ? step_io[traj] : S.init_step_ns;
    int fixed = S.fixed_step;
    int status = 0, rc = 0;
    long long det_step = S.init_step_ns;
    int n_steps = 0, n_rej = 0, n_rhs = 0;
    double det_error = 0.0;
    int det_attempts = 1;
    bool retry = false, last = false;
    double h = 0.0, nx = 0.0;
    long long prev_step = step_ns;
    int prev_fixed = fixed;
    RotBase rbase;
    rbase.sa = 0; rbase.ca = 1; rbase.sd = 1; rbase.cd = 0; rbase.sw = 0; rbase.cw = 1;
    if (lane < 6) g.ycur[lane] = yc;
    if (sink.ev_kind && lane == 0) {
        g.ev[0] = event_eval(sink.ev_kind, sink.ev_value, state[traj], state[n + traj], state[2 * n + traj],
                             state[3 * n + traj], state[4 * n + traj], state[5 * n + traj]);
        g.ev[1] = 0.0;
    }
    if (valid && sink.cap > 0) {  // start state (instance.rs:307, 321)
        if (lane < 6) sink.state[((size_t)lane * sink.cap) * n + traj] = yc;
        if (lane == 6) sink.epoch[traj] = epoch;
    }
    // instance.rs:96-115
    const long long duration = end_epoch - epoch;
    const bool backprop = duration < 0;
    bool done = !valid || (duration == 0);
    if (!done && g.pm < 0.0) { rc = NYXB_ERR_FUEL_EXHAUSTED; done = true; }
    if (!done && duration < 0) step_ns = -step_ns;
    __syncwarp(FULL);
    const int stages = S.tb.stages;
    const long long stop = end_epoch;

    for (;;) {
        if (!done && !retry) {
            // ---- instance.rs:149-196: pick this step (regular, or the final fixed step to the stop time)
            last = false;
            prev_step = step_ns;
            prev_fixed = fixed;
            if (ctl_past_stop(epoch, step_ns, stop, backprop)) {
                if (stop == epoch) {
                    done = true;
                } else {
                    step_ns = stop - epoch;
                    fixed = 1;
                    last = true;
                }
            }
            if (!done) {
                det_attempts = 1;
                h = dur_to_seconds(step_ns);
            }
        }
        if (__all_sync(FULL, done)) break;
        // ---- orientation angles at the step epoch: lanes 0..2 evaluate one sin/cos pair each
        if (S.grav.rot.kind != 0) {
            const double t_s = dur_to_seconds(epoch);
            const double d = t_s / 86400.0;
            const double Tc = d / 36525.0;
            double ang;
            if (lane == 0) ang = (S.grav.rot.ra0 + S.grav.rot.ra1 * Tc) * NYXB_DEG2RAD;
            else if (lane == 1) ang = (S.grav.rot.dec0 + S.grav.rot.dec1 * Tc) * NYXB_DEG2RAD;
            else ang = fmod(S.grav.rot.w0 + S.grav.rot.w1 * d, 360.0) * NYXB_DEG2RAD;
            double sv, cv;
            det_sincos(ang, sv, cv);
            rbase.sa = shfl_d(FULL, sv, 0, G); rbase.ca = shfl_d(FULL, cv, 0, G);
            rbase.sd = shfl_d(FULL, sv, 1, G); rbase.cd = shfl_d(FULL, cv, 1, G);
            rbase.sw = shfl_d(FULL, sv, 2, G); rbase.cw = shfl_d(FULL, cv, 2, G);
        }
        // ---- derive(): one attempt (instance.rs:358-493)
        for (int i = 0; i < stages; ++i) {
            // stage state y + h * sum_j a_ij k_j (instance.rs:376-394); stage 0 is y itself
            if (lane < 6) {
                double ysv = yc;
                if (i > 0) {
                    const double* arow = &S.tb.a[(i - 1) * NYXB_MAX_STAGES];
                    double w0 = 0.0, w1 = 0.0;  // two chains: the sum is latency-bound otherwise
                    int j = 0;
                    for (; j + 1 < i; j += 2) {
                        w0 = fma(arow[j], g.kst[j * 6 + lane], w0);
                        w1 = fma(arow[j + 1], g.kst[(j + 1) * 6 + lane], w1);
                    }
                    if (j < i) w0 = fma(arow[j], g.kst[j * 6 + lane], w0);
                    ysv = fma(h, w0 + w1, yc);
                }
                g.ys[lane] = ysv;
            }
            g.hz = (i > 0) ? h * 0.0 : 0.0;
            const long long off_ns = (i > 0) ? dur_from_seconds(S.tb.c[i - 1] * h) : 0;  // stage epoch is ns-truncated
            const double dt_s = (double)off_ns * 1e-9;
            const long long t_ns = epoch + off_ns;
            __syncwarp(FULL);
            double dyc;
            const int rcs = coop_rhs<G, NC>(S, recs, Cp.L, sm_seed, a_cs, cm_off, g, rbase, dt_s, t_ns, lane, dyc);
            if (!done) {
                ++n_rhs;
                if (rcs) { rc = rcs; done = true; }
                else if (lane < 6) g.kst[i * 6 + lane] = dyc;
            }
            // every lane read the stage state (ys) and the parked DCM (nxt) at the end of coop_rhs: order those reads before the
            // next stage's writes (compute-sanitizer racecheck found a write-after-read on ys without it)
            __syncwarp(FULL);
        }
        {
            double er = 0.0;
            nx = yc;
            if (lane < 6) {
                for (int i = 0; i < stages; ++i) {
                    const double ki = g.kst[i * 6 + lane];
                    if (!fixed) er = fma(h * S.tb.e[i], ki, er);
                    nx = fma(h * S.tb.b[i], ki, nx);
                }
                g.nxt[lane] = nx;
                g.er[lane] = er;
            }
        }
        __syncwarp(FULL);
        if (!done) {
            long long dt_ns = 0;
            bool accept = true;
            if (fixed) {
                det_step = step_ns; dt_ns = step_ns;
            } else {
                double e9[9], c9[9], y9[9];
#pragma unroll
                for (int e = 0; e < 6; ++e) { e9[e] = g.er[e]; c9[e] = g.nxt[e]; y9[e] = g.ycur[e]; }
                e9[6] = e9[7] = e9[8] = 0.0;
                y9[6] = g.cr; y9[7] = g.cd; y9[8] = g.pm;
                c9[6] = g.cr + g.hz; c9[7] = g.cd + g.hz; c9[8] = g.pm + g.hz;
                det_error = error_estimate(S.error_ctrl, e9, c9, y9);
                accept = ctl_accept(S, det_error, h, det_attempts);
                if (accept) {
                    bool bad = false;
#pragma unroll
                    for (int e = 0; e < 9; ++e) bad |= (c9[e] != c9[e]);
                    if (bad) {
                        rc = NYXB_ERR_PROP_MATH; done = true; accept = false;
                    } else {
                        step_ns = ctl_accepted<pow_inv_int>(S, det_error, h, det_attempts, status, det_step);
                        dt_ns = det_step;
                    }
                } else {
                    det_attempts += 1;
                    n_rej += 1;
                    h = ctl_retry<pow_inv_int>(S, det_error, h);
                    retry = true;
                }
            }
            if (accept) {
                // ---- single_step(): instance.rs:343-352
                retry = false;
                epoch += dt_ns;
                yc = nx;  // committed below, after every lane has finished reading ycur/nxt
                g.cr = g.cr < 0.0 ? 0.0 : (g.cr > 2.0 ? 2.0 : g.cr);  // cosmic/spacecraft.rs:494
                n_steps += 1;
                if (n_steps < sink.cap) {  // the channel send of instance.rs:186-193 / 255-259 (56 B per accepted step)
                    const size_t s = (size_t)n_steps;
                    if (lane < 6) sink.state[((size_t)lane * sink.cap + s) * n + traj] = nx;
                    if (lane == 6) sink.epoch[s * n + traj] = epoch;
                }
                if (g.pm < 0.0) { rc = NYXB_ERR_FUEL_EXHAUSTED; done = true; }
                if (sink.ev_kind && !last) {  // stop condition on non-final steps (instance.rs:243-252, event.rs:120-150); nxt = new state
                    const double yn = event_eval(sink.ev_kind, sink.ev_value, g.nxt[0], g.nxt[1], g.nxt[2], g.nxt[3], g.nxt[4], g.nxt[5]);
                    const double cnt = g.ev[1] + ((g.ev[0] * yn < 0.0) ? 1.0 : 0.0);
                    __syncwarp(gmask);
                    if (lane == 0) { g.ev[0] = yn; g.ev[1] = cnt; }
                    if (cnt >= (double)sink.ev_trigger) done = true;
                }
                if (last) {
                    step_ns = prev_step;
                    fixed = prev_fixed;
                    if (backprop) step_ns = -step_ns;
                    done = true;
                }
            }
        }
        __syncwarp(FULL);  // all lanes are done reading ycur/nxt/er
        if (lane < 6) g.ycur[lane] = yc;
    }
    __syncwarp(FULL);
    if (!valid) return;
    if (lane < 6) out_state[(size_t)lane * n + traj] = yc;
    if (lane == 6) {
        out_state[6 * n + traj] = g.cr; out_state[7 * n + traj] = g.cd; out_state[8 * n + traj] = g.pm;
        out_epoch[traj] = epoch;
        if (step_io) step_io[traj] = step_ns;
        out_status[traj] = ctl_finish(sink, traj, status, rc, (int)g.ev[1], n_steps);
    }
    if (lane == 7 && out_details) {
        nyxb_details d;
        d.step_ns = det_step; d.error = det_error; d.attempts = det_attempts; d._pad = 0;
        d.n_steps = n_steps; d.n_rejected = n_rej; d.n_rhs = n_rhs;
        out_details[traj] = d;
    }
}

template <int G, bool TAB, bool NC>
static cudaError_t launch_g(const DevSetup* S, const DevCoop* Cp, size_t n, size_t smem, const double* state,
                            const double* consts, const long long* epoch0, long long end_epoch, long long* step_io,
                            double* out_state, long long* out_epoch, nyxb_details* out_details, int* out_status,
                            const DevSink* sink, cudaStream_t stream) {
    cudaError_t e = cudaFuncSetAttribute(nyxb_k_coop<G, TAB, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int dev = 0, sms = 0, occ = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, nyxb_k_coop<G, TAB, NC>, COOP_CTA, smem);
    if (e != cudaSuccess) return e;
    if (occ < 1) occ = 1;
    const size_t groups = COOP_CTA / G;
    // one resident wave spread evenly over the SMs when the ensemble fits; otherwise plain tiling
    size_t grid = (n + groups - 1) / groups;
    const size_t wave = (size_t)sms * occ;
    if (grid <= wave) grid = ((grid + sms - 1) / sms) * sms;  // one resident wave, same CTA count on every SM
    nyxb_k_coop<G, TAB, NC><<<(unsigned)grid, COOP_CTA, smem, stream>>>(*S, *Cp, n, state, consts, epoch0, end_epoch, step_io,
                                                                        out_state, out_epoch, out_details, out_status, *sink);
    return cudaGetLastError();
}

template <int G>
cudaError_t nyxb_launch_coop_g(const DevSetup* S, const DevCoop* Cp, size_t n, const double* state, const double* consts,
                               const long long* epoch0, long long end_epoch, long long* step_io, double* out_state,
                               long long* out_epoch, nyxb_details* out_details, int* out_status, const DevSink* sink,
                               cudaStream_t stream) {
    const size_t groups = COOP_CTA / G;
    const size_t grp_bytes = groups * coop_traj_stride(S->grav.N) * sizeof(double) + coop_meta_bytes(S->grav.N, G, Cp->kmax);
    const size_t with_table = grp_bytes + coop_rec_bytes(Cp->L, G);
    // stage the record table in shared memory when at least two CTAs still fit per SM (227 KB usable)
    const bool tab = with_table * 2 <= 227 * 1024;
    const size_t smem = tab ? with_table : grp_bytes;
    if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;
#define NYXB_COOP_GO(TAB) ((S->grav_body >= 0 || S->n_xgrav > 0) ? launch_g<G, TAB, true>(S, Cp, n, smem, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream) : launch_g<G, TAB, false>(S, Cp, n, smem, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream))
    return tab ? NYXB_COOP_GO(true) : NYXB_COOP_GO(false);
#undef NYXB_COOP_GO
}
