// nyxb_device.cuh — device-side data model and right-hand side (force models) of the
// H100 batched propagator.  Shared by the per-thread kernel (nyxb_kernels.cu, built twice:
// STRICT = no FMA contraction / reference operation order, FAST = FMA allowed), the cooperative and
// transposed kernels (nyxb_coop_kernel.cuh, nyxb_coop_strict.cu, nyxb_tx.cu) and the STM / filter kernels
// (nyxb_od*.cu).  Every one of them calls the step-size controller defined at the end of this file.
//
// Reference behaviour implemented here (paths relative to /root/reference/nyx-core/src):
//   SpacecraftDynamics::eom   dynamics/spacecraft.rs:191-310
//   OrbitalDynamics::eom      dynamics/orbital.rs:80-114
//   PointMasses::eom          dynamics/orbital.rs:213-247
//   GravityField::eom         dynamics/gravity_field.rs:148-268
//   SolarPressure::eom        dynamics/solarpressure.rs:135-165 (+ cosmic/eclipse.rs:69-83)
//   Drag::eom                 dynamics/drag.rs:181-284
//   ErrorControl::estimate    propagators/error_ctrl.rs:79-230
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/nyxb.h"

#define NYXB_MAX_STAGES 16
#define NYXB_MAX_DEGREE 96 /* rows of the per-thread Legendre scratch: degree + 3 <= 99 */

struct DevRotation {
    int kind;
    double ra0, ra1, dec0, dec1, w0, w1;  // degrees
    double wdot;                           // rad/s
    double ra_dot, dec_dot;                // rad/s (FAST cooperative kernel: first-order pole update)
};

struct DevBody {
    double mu, radius;
    long long t0_ns, interval_ns;
    int n_intervals, n_coeffs;
    const double* coeffs;  // device [n_intervals][3][n_coeffs]
    double inv_interval;   // 1.0 / (double)interval_ns (FAST mode only)
};

// One record per (n, m), m <= n, n <= N+1, triangular index n(n+1)/2 + m.
struct __align__(16) DevHarm {
    double b, c;        // recursion factors   gravity_field.rs:69-81
    double vr01, vr11;  //                     gravity_field.rs:83-90
    double cbar, sbar;  // normalised coefficients (0 beyond N / beyond `order`)
};

struct DevGrav {
    int N, M;
    double mu, r_eq, inv_r_eq;
    DevRotation rot;
    const DevHarm* tab;      // (N+2)(N+3)/2 records
    const double* a_diag;    // [N+3]   gravity_field.rs:61-66
    const double* offdiag;   // [N+2]   sqrt(2n+3), n = 0..N+1   gravity_field.rs:168-173
    // FAST per-thread column walk (grav_accel_cols): 8 doubles per (column k, row j) in walk order — columns in pairs (k, k+1):
    // row k of column k, then rows j = k+1..N+1 of both columns interleaved; one null record at the end:
    // {q1..q6: the entry's coefficients of the six per-column sums (1/r_eq folded in), b, c: factors of A[j+1][k]}
    const double* colrec;
    int ncols;
};

struct DevSrp {
    double phi;
    int sun_body, n_shadow;
    int shadow_body[4];
    int estimate;  // Cr column of the STM A-matrix (solarpressure.rs:131-133)
};

struct DevDrag {
    int density;
    double rho0, r0, ref_alt_m, r_eq;
    DevRotation rot;
};

struct DevTableau {
    int stages, order;
    double a[NYXB_MAX_STAGES * NYXB_MAX_STAGES];  // dense, row i (stage i+1) uses a[i*16 + j], j <= i
    double c[NYXB_MAX_STAGES];                    // c[i] = sum_j a_ij accumulated left to right (instance.rs:379-386)
    double b[NYXB_MAX_STAGES];
    double e[NYXB_MAX_STAGES];                    // b_i - b*_i
};

struct DevSetup {
    // integrator
    DevTableau tb;
    int error_ctrl, attempts, fixed_step;
    long long init_step_ns, min_step_ns, max_step_ns;
    double tolerance, min_step_s, max_step_s;
    double inv_order, inv_order_m1;
    // dynamics
    double mu_central, central_radius;
    int n_bodies;
    unsigned point_mass_mask;
    int n_pm;                         // PointMasses members in summation order (orbital.rs:217)
    signed char pm_order[NYXB_MAX_BODIES];
    DevBody bodies[NYXB_MAX_BODIES];
    int has_grav, has_srp, has_drag;
    int grav_body;                    // body the primary field belongs to (NYXB_CENTRAL_BODY or an index into bodies)
    int n_xgrav;                      // further harmonic fields, evaluated per trajectory after the primary one
    int xgrav_body[NYXB_MAX_FIELDS - 1];
    int state_center;                 // integration_frame: -1 none, else the body the caller's states are relative to
    DevGrav grav;
    DevGrav xgrav[NYXB_MAX_FIELDS - 1];
    DevSrp srp;
    DevDrag drag;
};

// trajectory recording sink (device pointers; cap == 0: recording off)
struct DevSink {
    long long cap;
    long long* epoch;  // [cap][n]
    double* state;     // [6][cap][n]
    long long* count;  // [n]
    // stop condition of until_nth_event (event.rs:88-211); ev_kind == 0: none
    int ev_kind, ev_trigger;
    double ev_value;
    int* ev_crossings;  // [n]
};

// event scalar minus the desired value (closed set, see nyxb_event_kind)
__device__ __forceinline__ double event_eval(int kind, double value, double x, double y, double z, double vx, double vy, double vz) {
    double s;
    switch (kind) {
    case NYXB_EVENT_RMAG: s = sqrt((x * x + y * y) + z * z); break;
    case NYXB_EVENT_RDOTV: s = (x * vx + y * vy) + z * vz; break;
    case NYXB_EVENT_X: s = x; break;
    case NYXB_EVENT_Y: s = y; break;
    case NYXB_EVENT_Z: s = z; break;
    default: s = sqrt((vx * vx + vy * vy) + vz * vz); break;
    }
    return s - value;
}

#define NYXB_NS_PER_S 1000000000LL
#define NYXB_NS_PER_CENTURY 3155760000000000000LL

// hifitime Duration::to_seconds (see oracle/nyx_oracle.c for the pinning)
__device__ __forceinline__ double dur_to_seconds(long long total_ns) {
    long long cent = total_ns / NYXB_NS_PER_CENTURY;
    if (total_ns % NYXB_NS_PER_CENTURY < 0) cent -= 1;
    long long nanos = total_ns - cent * NYXB_NS_PER_CENTURY;
    long long sec = nanos / NYXB_NS_PER_S;
    long long sub = nanos - sec * NYXB_NS_PER_S;
    double s = __dadd_rn((double)sec, __dmul_rn((double)sub, 1e-9));
    if (cent == 0) return s;
    return __dadd_rn(__dadd_rn(__dmul_rn((double)cent, 3155760000.0), (double)sec), __dmul_rn((double)sub, 1e-9));
}

// f64 * Unit::Second -> Duration: truncation toward zero, NaN -> 0, saturating
__device__ __forceinline__ long long dur_from_seconds(double s) {
    double ns = __dmul_rn(s, 1e9);
    if (ns != ns) return 0;
    if (ns >= 9.2e18) return 0x7fffffffffffffffLL;
    if (ns <= -9.2e18) return (long long)0x8000000000000000ULL;
    return (long long)ns;  // cvt.rzi
}

__device__ __forceinline__ double norm3(double x, double y, double z) {
#if NYXB_STRICT
    return sqrt((x * x + y * y) + z * z);  // nalgebra order; -fmad=false build
#else
    return sqrt(fma(z, z, fma(y, y, x * x)));
#endif
}

// Deterministic sin/cos: same operation sequence as oracle/nyx_oracle.c::nyx_oracle_sincos.
__device__ __forceinline__ void det_sincos(double x, double& s, double& c) {
    const double two_over_pi = 6.36619772367581382433e-01;
    const double p1 = 1.57079632673412561417e+00;
    const double p2 = 6.07710050630396597660e-11;
    const double p3 = 2.02226624879595063154e-21;
    double kf = rint(x * two_over_pi);
    double r = ((x - kf * p1) - kf * p2) - kf * p3;
    double z = r * r;
    double ps = -1.66666666666666324348e-01 + z * (8.33333333332248946124e-03 + z * (-1.98412698298579493134e-04 + z * (2.75573137070700676789e-06 + z * (-2.50507602534068634195e-08 + z * 1.58969099521155010221e-10))));
    double sn = r + (r * z) * ps;
    double pc = 4.16666666666666019037e-02 + z * (-1.38888888888741095749e-03 + z * (2.48015872894767294178e-05 + z * (-2.75573143513906633035e-07 + z * (2.08757232129817482790e-09 + z * -1.13596475577881948265e-11))));
    double cs = (1.0 - 0.5 * z) + (z * z) * pc;
    long long k = (long long)kf;
    switch (k & 3) {
    case 0: s = sn; c = cs; break;
    case 1: s = cs; c = -sn; break;
    case 2: s = -sn; c = -cs; break;
    default: s = -cs; c = sn; break;
    }
}

// ---- step-size controller power: (tol/err)^(1/n), n = order or order-1 (instance.rs:451-454, 479-482).
// The reference calls libm `pow(x, fl(1/n))` (glibc: correctly rounded in all but a percent of cases).
// CUDA's pow is only 2-ulp accurate, and after a *rejected* attempt the raw f64 step is used
// unquantised (instance.rs:484-488), so a 1-ulp difference would perturb the whole trajectory.
// We therefore correct CUDA's result to the correctly rounded value: one Newton step on
// q^n = x evaluated in double-double, plus the first-order term for fl(1/n) != 1/n.
struct dd_t { double hi, lo; };
__device__ __forceinline__ dd_t dd_mul_d(dd_t a, double b) {
    double t = __dmul_rn(a.hi, b);
    double e = fma(a.hi, b, -t);
    double lo = fma(a.lo, b, e);
    double hi = __dadd_rn(t, lo);
    dd_t r; r.hi = hi; r.lo = __dsub_rn(lo, __dsub_rn(hi, t));
    return r;
}
__device__ __forceinline__ double pow_inv_int(double x, int n) {
    // eps_n = fl(1/n) - 1/n
    const double eps_tab[10] = {0.0, 0.0, 0.0, -1.850371707708594e-17, 0.0, 1.1102230246251566e-17,
                                -9.25185853854297e-18, -7.93016446160826e-18, 0.0, -6.1679056923619804e-18};
    double yinv = __ddiv_rn(1.0, (double)n);
    double q0 = pow(x, yinv);
    if (!(x > 0.0) || !(x < 1.0e300) || n < 2 || n > 9 || !(q0 > 0.0) || !(q0 < 1.0e300)) return q0;
    dd_t p; p.hi = q0; p.lo = 0.0;
    for (int i = 1; i < n; ++i) p = dd_mul_d(p, q0);
    double r = __dadd_rn(__dsub_rn(p.hi, x), p.lo);              // q0^n - x
    double delta = __ddiv_rn(__dmul_rn(r, q0), __dmul_rn((double)n, p.hi));
    double corr = __dmul_rn(__dmul_rn(q0, eps_tab[n]), log(x));  // x^y = x^(1/n) (1 + eps ln x)
    return __dadd_rn(q0, __dsub_rn(corr, delta));
}

#define NYXB_DEG2RAD 1.7453292519943295e-2

// inertial -> body-fixed DCM (row-major R[9]) of the orientation model in nyxb.h
__device__ __forceinline__ void rotation_dcm(const DevRotation& rot, long long t_ns, double R[9]) {
    if (rot.kind == 0) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        return;
    }
    double t_s = dur_to_seconds(t_ns);
    double d = t_s / 86400.0;
    double T = d / 36525.0;
    double ra = (rot.ra0 + rot.ra1 * T) * NYXB_DEG2RAD;
    double dec = (rot.dec0 + rot.dec1 * T) * NYXB_DEG2RAD;
    double w = fmod(rot.w0 + rot.w1 * d, 360.0) * NYXB_DEG2RAD;
    double sa, ca, sd, cd, sw, cw;
    det_sincos(ra, sa, ca);
    det_sincos(dec, sd, cd);
    det_sincos(w, sw, cw);
    double b00 = -sa, b01 = ca, b02 = 0.0;
    double b10 = -(sd * ca), b11 = -(sd * sa), b12 = cd;
    double b20 = cd * ca, b21 = cd * sa, b22 = sd;
    R[0] = cw * b00 + sw * b10; R[1] = cw * b01 + sw * b11; R[2] = cw * b02 + sw * b12;
    R[3] = cw * b10 - sw * b00; R[4] = cw * b11 - sw * b01; R[5] = cw * b12 - sw * b02;
    R[6] = b20; R[7] = b21; R[8] = b22;
}

// Piecewise-Chebyshev body position (Clenshaw); returns false when outside coverage.
__device__ __forceinline__ bool body_position(const DevBody& b, long long t_ns, double pos[3]) {
    long long dt = t_ns - b.t0_ns;
    if (dt < 0) return false;
#if NYXB_STRICT
    long long idx = dt / b.interval_ns;
    if (idx >= b.n_intervals) return false;
    long long off = dt - idx * b.interval_ns;
    double tau = 2.0 * ((double)off / (double)b.interval_ns) - 1.0;
    double tau2 = 2.0 * tau;
    int nc = b.n_coeffs;
    const double* c = b.coeffs + (size_t)idx * 3 * (size_t)nc;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
        const double* ca = c + ax * nc;
        double b1 = 0.0, b2 = 0.0;
        for (int k = nc - 1; k >= 1; --k) {
            double bk = (tau2 * b1 - b2) + __ldg(ca + k);
            b2 = b1; b1 = bk;
        }
        pos[ax] = (tau * b1 - b2) + __ldg(ca);
    }
#else
    // FAST: interval index from the reciprocal (no 64-bit division; +-1 corrected), the three axes share one Clenshaw loop
    long long idx = (long long)((double)dt * b.inv_interval);
    long long off = dt - idx * b.interval_ns;
    if (off < 0) { idx -= 1; off += b.interval_ns; }
    else if (off >= b.interval_ns) { idx += 1; off -= b.interval_ns; }
    if (idx >= b.n_intervals) return false;
    const double tau = fma(2.0 * (double)off, b.inv_interval, -1.0);
    const double tau2 = 2.0 * tau;
    const int nc = b.n_coeffs;
    const double* cx = b.coeffs + (size_t)idx * 3 * (size_t)nc;
    const double* cy = cx + nc;
    const double* cz = cy + nc;
    double x1 = 0.0, x2 = 0.0, y1 = 0.0, y2 = 0.0, z1 = 0.0, z2 = 0.0;
    for (int k = nc - 1; k >= 1; --k) {
        const double xk = fma(tau2, x1, __ldg(cx + k) - x2);
        const double yk = fma(tau2, y1, __ldg(cy + k) - y2);
        const double zk = fma(tau2, z1, __ldg(cz + k) - z2);
        x2 = x1; x1 = xk; y2 = y1; y1 = yk; z2 = z1; z1 = zk;
    }
    pos[0] = fma(tau, x1, __ldg(cx) - x2);
    pos[1] = fma(tau, y1, __ldg(cy) - y2);
    pos[2] = fma(tau, z1, __ldg(cz) - z2);
#endif
    return true;
}

// d/dt of the Chebyshev ephemeris (sum_k c_k T_k'(tau) * 2 / interval), reference operation order in every build: used where
// anise differentiates an SPK segment — frame translations (integration_frame, instance.rs:117-142) and tracking geometry
__device__ static bool body_velocity(const DevBody& b, long long t_ns, double vel[3]) {
    long long dt = t_ns - b.t0_ns;
    if (dt < 0) return false;
    long long idx = dt / b.interval_ns;
    if (idx >= b.n_intervals) return false;
    long long off = dt - idx * b.interval_ns;
    double tau = __dsub_rn(__dmul_rn(2.0, __ddiv_rn((double)off, (double)b.interval_ns)), 1.0);
    double tau2 = __dmul_rn(2.0, tau);
    int nc = b.n_coeffs;
    const double* c = b.coeffs + (size_t)idx * 3 * (size_t)nc;
    double scale = __ddiv_rn(2.0, __dmul_rn((double)b.interval_ns, 1e-9));
    for (int ax = 0; ax < 3; ++ax) {
        const double* ca = c + ax * nc;
        double b1 = 0.0, b2 = 0.0;
        for (int j = nc - 2; j >= 0; --j) {
            double bj = __dsub_rn(__dadd_rn(__dmul_rn((double)(j + 1), __ldg(ca + j + 1)), __dmul_rn(tau2, b1)), b2);
            b2 = b1; b1 = bj;
        }
        vel[ax] = __dmul_rn(b1, scale);
    }
    return true;
}

// anise `occultation` restated (see oracle/nyx_oracle.c::nyx_oracle_occultation)
__device__ __forceinline__ double circ_seg_area(double r, double d) {
    return (r * r) * acos(d / r) - d * sqrt(r * r - d * d);
}

__device__ inline double occultation(const double r_eb[3], const double r_ls[3], double light_radius, double body_radius) {
#if !NYXB_STRICT
    {   // FAST: the common case "the two disks are far apart" (d' > r_ls' + r_fobj', result 0) decided without asin/acos/division:
        // with s = sin of an apparent radius (< 1), d' > a + b  <=>  cos d' < cos a cos b - sin a sin b.  A 1e-9 guard band
        // sends everything near the boundary to the full evaluation below, so the returned values are unchanged.
        const double i_ls = rsqrt(fma(r_ls[2], r_ls[2], fma(r_ls[1], r_ls[1], r_ls[0] * r_ls[0])));
        const double i_eb = rsqrt(fma(r_eb[2], r_eb[2], fma(r_eb[1], r_eb[1], r_eb[0] * r_eb[0])));
        const double sl = light_radius * i_ls, sb = body_radius * i_eb;
        if (sl < 1.0 && sb < 1.0) {
            const double cd = -((r_ls[0] * r_eb[0] + r_ls[1] * r_eb[1]) + r_ls[2] * r_eb[2]) * (i_eb * i_ls);
            const double cs = sqrt((1.0 - sl * sl) * (1.0 - sb * sb)) - sl * sb;
            if (cd < cs - 1e-9) return 0.0;
        }
    }
#endif
    double n_ls = norm3(r_ls[0], r_ls[1], r_ls[2]), n_eb = norm3(r_eb[0], r_eb[1], r_eb[2]);
    double r_ls_prime = (light_radius >= n_ls) ? light_radius : asin(light_radius / n_ls);
    double r_fobj_prime = (body_radius >= n_eb) ? body_radius : asin(body_radius / n_eb);
    double dot = (r_ls[0] * r_eb[0] + r_ls[1] * r_eb[1]) + r_ls[2] * r_eb[2];
    double d_prime = acos(-dot / (n_eb * n_ls));
    if (d_prime - r_ls_prime > r_fobj_prime) return 0.0;
    if (r_fobj_prime > d_prime + r_ls_prime) return 1.0;
    if (fabs(r_ls_prime - r_fobj_prime) < d_prime && d_prime < r_ls_prime + r_fobj_prime) {
        double d1 = (d_prime * d_prime - r_ls_prime * r_ls_prime + r_fobj_prime * r_fobj_prime) / (2.0 * d_prime);
        double d2 = (d_prime * d_prime + r_ls_prime * r_ls_prime - r_fobj_prime * r_fobj_prime) / (2.0 * d_prime);
        double shadow_area = circ_seg_area(r_fobj_prime, d1) + circ_seg_area(r_ls_prime, d2);
        if (shadow_area != shadow_area) return 1.0;
        double nominal_area = 3.14159265358979323846 * (r_ls_prime * r_ls_prime);
        return shadow_area / nominal_area;
    }
    return (r_fobj_prime * r_fobj_prime) / (r_ls_prime * r_ls_prime);
}

__device__ __forceinline__ int tri(int n, int m) { return n * (n + 1) / 2 + m; }

// GravityField::eom (gravity_field.rs:148-268) — reference summation order, per-thread
// rolling rows of the derived-Legendre matrix: P = row n, Q = row n+1 (Q is overwritten
// in place from row n-1).  Only the values are rolled; every A[n][m] equals the
// reference's column-recursion value bit for bit (same recurrence, same operands).
__device__ inline void grav_accel_rows(const DevGrav& g, long long t_ns, const double r_in[3], double acc[3]) {
    const int N = g.N, M = g.M;
    double R[9];
    rotation_dcm(g.rot, t_ns, R);
    double rb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = (R[3 * i] * r_in[0] + R[3 * i + 1] * r_in[1]) + R[3 * i + 2] * r_in[2];
    double r_ = norm3(rb[0], rb[1], rb[2]);
    double s_ = rb[0] / r_, t_ = rb[1] / r_, u_ = rb[2] / r_;

    double rowA[NYXB_MAX_DEGREE + 3], rowB[NYXB_MAX_DEGREE + 3];
    double r_m[NYXB_MAX_DEGREE + 1], i_m[NYXB_MAX_DEGREE + 1];
    double* P = rowA;  // row n
    double* Q = rowB;  // row n-1, becomes row n+1
    for (int m = 0; m <= N + 2; ++m) { rowA[m] = 0.0; rowB[m] = 0.0; }
    // row 0 and row 1 (gravity_field.rs:61-66, 168)
    Q[0] = 1.0;
    P[0] = u_ * sqrt(3.0);
    P[1] = __ldg(g.a_diag + 1);
    const int mm = N < M ? N : M;
    r_m[0] = 1.0; i_m[0] = 0.0;
    for (int m = 1; m <= mm; ++m) {
        r_m[m] = s_ * r_m[m - 1] - t_ * i_m[m - 1];
        i_m[m] = s_ * i_m[m - 1] + t_ * r_m[m - 1];
    }
    double rho = g.r_eq / r_;
    double rho_np1 = g.mu / r_ * rho;
    double a4x = 0.0, a4y = 0.0, a4z = 0.0, a4w = 0.0;
    const double sqrt2 = sqrt(2.0);
    for (int n = 1; n <= N; ++n) {
        // ---- build row n+1 into Q (holds row n-1): gravity_field.rs:168-181
        {
            const int np1 = n + 1;
            const DevHarm* trow = g.tab + tri(np1, 0);
            int mrec = np1 - 2;  // m <= (n+1) - 2
            if (mrec > M + 1) mrec = M + 1;
            for (int m = 0; m <= mrec; ++m) {
                double bb = __ldg(&trow[m].b), cc = __ldg(&trow[m].c);
                Q[m] = u_ * bb * P[m] - cc * Q[m];
            }
            for (int m = mrec + 1; m <= np1 - 2; ++m) Q[m] = 0.0;  // never read (m > M+1)
            Q[n] = __ldg(g.offdiag + n) * u_ * __ldg(g.a_diag + n);  // A[n+1][n]
            Q[np1] = __ldg(g.a_diag + np1);                           // A[n+1][n+1]
        }
        // ---- degree-n partial sums: gravity_field.rs:217-249
        double sx = 0.0, sy = 0.0, sz = 0.0, sw = 0.0;
        rho_np1 *= rho;
        const DevHarm* trow = g.tab + tri(n, 0);
        int mtop = n < M ? n : M;
        for (int m = 0; m <= mtop; ++m) {
            double cv = __ldg(&trow[m].cbar), sv = __ldg(&trow[m].sbar);
            double d_ = (cv * r_m[m] + sv * i_m[m]) * sqrt2;
            double e_ = 0.0, f_ = 0.0;
            if (m != 0) {
                e_ = (cv * r_m[m - 1] + sv * i_m[m - 1]) * sqrt2;
                f_ = (sv * r_m[m - 1] - cv * i_m[m - 1]) * sqrt2;
            }
            double anm = P[m];
            sx += (double)m * anm * e_;
            sy += (double)m * anm * f_;
            sz += __ldg(&trow[m].vr01) * P[m + 1] * d_;
            sw -= __ldg(&trow[m].vr11) * Q[m + 1] * d_;
        }
        double rr = rho_np1 / g.r_eq;
        a4x += rr * sx; a4y += rr * sy; a4z += rr * sz; a4w += rr * sw;
        // roll: row n+1 becomes row n, row n becomes row n-1
        double* tmp = P; P = Q; Q = tmp;
    }
    double ab0 = a4x + a4w * s_, ab1 = a4y + a4w * t_, ab2 = a4z + a4w * u_;
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[i] = (R[i] * ab0 + R[3 + i] * ab1) + R[6 + i] * ab2;
}

#if !NYXB_STRICT
// GravityField::eom for one trajectory on one thread, FAST mode: the double sum walked by COLUMNS of the derived-Legendre
// triangle.  Each A[j][k] is produced by its column recursion in a register and consumed once: the four sums of the
// reference (gravity_field.rs:217-249) are regrouped per column k — sum2/sum3 re-indexed by k = m + 1 — so that all terms of
// a column share the pair (r_{k-1}, i_{k-1}) = (cos, sin)((k-1) lambda) cos^(k-1)(phi), applied once per column:
//   P1,P2 = sum_j rr_j     A[j][k] k sqrt2 (C,S)_{j,k}            -> a0 += r P1 + i P2,  a1 += r P2 - i P1
//   P3,P4 = sum_j rr_j     A[j][k] sqrt2 vr01(j,k-1) (C,S)_{j,k-1}    -> a2 += r P3 + i P4
//   P5,P6 = sum_j rr_{j-1} A[j][k] sqrt2 vr11(j-1,k-1) (C,S)_{j-1,k-1} -> a3 -= r P5 + i P6
// No Legendre rows in local memory, no trig/power tables: the running powers advance once per column.  Every thread of a
// warp walks the same (k, j) sequence, so the 64-byte records are warp-uniform loads.  12 FP64 instructions per entry.
__device__ inline void grav_accel_cols(const DevGrav& g, long long t_ns, const double r_in[3], double acc[3]) {
    const int N = g.N;
    double R[9];
    rotation_dcm(g.rot, t_ns, R);
    double rb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = fma(R[3 * i + 2], r_in[2], fma(R[3 * i + 1], r_in[1], R[3 * i] * r_in[0]));
    const double ir = rsqrt(fma(rb[2], rb[2], fma(rb[1], rb[1], rb[0] * rb[0])));
    const double s_ = rb[0] * ir, t_ = rb[1] * ir, u_ = rb[2] * ir;
    const double rho = g.r_eq * ir;
    const double irho = 1.0 / rho;
    double rk = 1.0, ik = 0.0;                 // (r_{k-1}, i_{k-1})
    double rho_k = (g.mu * ir) * rho * rho;    // (mu / r) rho^(k+1) at k = 1
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    // Columns are walked in PAIRS (k, k+1): two independent recursion chains per thread hide the FP64 latency, both use the same
    // rr_j.  Records come in walk order and are software-pipelined one entry ahead (the table ends with a null record).
    const double2* __restrict__ p = reinterpret_cast<const double2*>(g.colrec);
#define NYXB_REC_LD(x) __ldg(x)
    double2 n12 = NYXB_REC_LD(p), n34 = NYXB_REC_LD(p + 1), n56 = NYXB_REC_LD(p + 2), nbc = NYXB_REC_LD(p + 3);
    p += 4;
#ifndef NYXB_COLS_PF
#define NYXB_COLS_PF 1   /* prefetch distance in entries (1 or 2; the table ends with two null records) */
#endif
#if NYXB_COLS_PF == 2
    double2 m12 = NYXB_REC_LD(p), m34 = NYXB_REC_LD(p + 1), m56 = NYXB_REC_LD(p + 2), mbc = NYXB_REC_LD(p + 3);
    p += 4;
#define NYXB_COL_FETCH n12 = m12; n34 = m34; n56 = m56; nbc = mbc; m12 = NYXB_REC_LD(p); m34 = NYXB_REC_LD(p + 1); m56 = NYXB_REC_LD(p + 2); mbc = NYXB_REC_LD(p + 3);
#else
#define NYXB_COL_FETCH n12 = NYXB_REC_LD(p); n34 = NYXB_REC_LD(p + 1); n56 = NYXB_REC_LD(p + 2); nbc = NYXB_REC_LD(p + 3);
#endif
#define NYXB_COL_ENTRY(A, Ap, P1, P2, P3, P4, P5, P6)                                                            \
    {                                                                                                            \
        const double2 q12 = n12, q34 = n34, q56 = n56, bc = nbc;                                                 \
        NYXB_COL_FETCH                                                                                           \
        p += 4;                                                                                                  \
        const double t = rhop * A, tp = t * irho;                                                                \
        P1 = fma(t, q12.x, P1); P2 = fma(t, q12.y, P2);                                                          \
        P3 = fma(t, q34.x, P3); P4 = fma(t, q34.y, P4);                                                          \
        P5 = fma(tp, q56.x, P5); P6 = fma(tp, q56.y, P6);                                                        \
        const double An = fma(u_ * bc.x, A, -(bc.y * Ap));                                                       \
        Ap = A; A = An;                                                                                          \
    }
    for (int k = 1; k <= g.ncols; k += 2) {
        const bool two = k + 1 <= g.ncols;
        double A = __ldg(g.a_diag + k), Ap = 0.0, B = two ? __ldg(g.a_diag + k + 1) : 0.0, Bp = 0.0;
        double rhop = rho_k;
        double PA1 = 0.0, PA2 = 0.0, PA3 = 0.0, PA4 = 0.0, PA5 = 0.0, PA6 = 0.0;
        double PB1 = 0.0, PB2 = 0.0, PB3 = 0.0, PB4 = 0.0, PB5 = 0.0, PB6 = 0.0;
        NYXB_COL_ENTRY(A, Ap, PA1, PA2, PA3, PA4, PA5, PA6)   // row j = k belongs to column k alone
        rhop *= rho;
        if (two) {
            for (int j = k + 1; j <= N + 1; ++j) {
                NYXB_COL_ENTRY(A, Ap, PA1, PA2, PA3, PA4, PA5, PA6)
                NYXB_COL_ENTRY(B, Bp, PB1, PB2, PB3, PB4, PB5, PB6)
                rhop *= rho;
            }
        } else {
            for (int j = k + 1; j <= N + 1; ++j) {
                NYXB_COL_ENTRY(A, Ap, PA1, PA2, PA3, PA4, PA5, PA6)
                rhop *= rho;
            }
        }
        a0 = fma(rk, PA1, fma(ik, PA2, a0));
        a1 = fma(rk, PA2, fma(-ik, PA1, a1));
        a2 = fma(rk, PA3, fma(ik, PA4, a2));
        a3 -= fma(rk, PA5, ik * PA6);
        double nr = fma(s_, rk, -(t_ * ik)), ni = fma(s_, ik, t_ * rk);
        rk = nr; ik = ni;
        rho_k *= rho;
        if (two) {
            a0 = fma(rk, PB1, fma(ik, PB2, a0));
            a1 = fma(rk, PB2, fma(-ik, PB1, a1));
            a2 = fma(rk, PB3, fma(ik, PB4, a2));
            a3 -= fma(rk, PB5, ik * PB6);
            nr = fma(s_, rk, -(t_ * ik)); ni = fma(s_, ik, t_ * rk);
            rk = nr; ik = ni;
            rho_k *= rho;
        }
    }
#undef NYXB_COL_ENTRY
#undef NYXB_COL_FETCH
#undef NYXB_REC_LD
    const double ab0 = fma(a3, s_, a0), ab1 = fma(a3, t_, a1), ab2 = fma(a3, u_, a2);
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[i] = fma(R[6 + i], ab2, fma(R[3 + i], ab1, R[i] * ab0));
}
#endif

#define NYXB_AU_KM 149597870.700
#define NYXB_C_M_S (299792.458 * 1e3)

// ---- SpacecraftDynamics::eom split in three ordered parts so that the per-thread kernel
// (reference accumulation order) and the cooperative kernel (lanes share the harmonic sum)
// reuse the same force-model code:
//   accel_pre  : two-body + PointMasses                 orbital.rs:86-92, 213-247
//   (gravity)  : GravityField                           gravity_field.rs:148-268
//   accel_post : SolarPressure + Drag, each / mass      spacecraft.rs:238-243
__device__ __forceinline__ void accel_two_body(const DevSetup& S, const double y[9], double acc[3]) {
#if NYXB_STRICT
    double rmag = norm3(y[0], y[1], y[2]);
    double fac = -S.mu_central / (rmag * rmag * rmag);
#else
    const double ir = rsqrt(fma(y[2], y[2], fma(y[1], y[1], y[0] * y[0])));   // FAST: one rsqrt chain instead of sqrt + division
    double fac = -S.mu_central * (ir * ir * ir);
#endif
    acc[0] = fac * y[0]; acc[1] = fac * y[1]; acc[2] = fac * y[2];
}

// body positions at t_ns + PointMasses::eom added to acc (orbital.rs:213-247)
__device__ inline int accel_point_masses(const DevSetup& S, long long t_ns, const double y[9],
                                         double bpos[NYXB_MAX_BODIES][3], double acc[3]) {
    for (int j = 0; j < S.n_bodies; ++j)
        if (!body_position(S.bodies[j], t_ns, bpos[j])) return NYXB_ERR_EPHEMERIS;
    if (S.n_pm) {
        double dx[3] = {0.0, 0.0, 0.0};
        for (int q = 0; q < S.n_pm; ++q) {
            const int j = S.pm_order[q];
            double rj0 = y[0] - bpos[j][0], rj1 = y[1] - bpos[j][1], rj2 = y[2] - bpos[j][2];
            double nmu = -S.bodies[j].mu;
#if NYXB_STRICT
            double n_ij = norm3(bpos[j][0], bpos[j][1], bpos[j][2]);
            double r_ij3 = n_ij * n_ij * n_ij;
            double n_j = norm3(rj0, rj1, rj2);
            double r_j3 = n_j * n_j * n_j;
            dx[0] += nmu * (rj0 / r_j3 + bpos[j][0] / r_ij3);
            dx[1] += nmu * (rj1 / r_j3 + bpos[j][1] / r_ij3);
            dx[2] += nmu * (rj2 / r_j3 + bpos[j][2] / r_ij3);
#else
            // FAST: |r|^-3 from two rsqrt chains instead of two sqrt + six divisions
            const double i_ij = rsqrt(fma(bpos[j][2], bpos[j][2], fma(bpos[j][1], bpos[j][1], bpos[j][0] * bpos[j][0])));
            const double i_j = rsqrt(fma(rj2, rj2, fma(rj1, rj1, rj0 * rj0)));
            const double i_j3 = i_j * i_j * i_j, i_ij3 = i_ij * i_ij * i_ij;
            dx[0] += nmu * fma(rj0, i_j3, bpos[j][0] * i_ij3);
            dx[1] += nmu * fma(rj1, i_j3, bpos[j][1] * i_ij3);
            dx[2] += nmu * fma(rj2, i_j3, bpos[j][2] * i_ij3);
#endif
        }
        acc[0] += dx[0]; acc[1] += dx[1]; acc[2] += dx[2];
    }
    return 0;
}

__device__ inline int accel_pre(const DevSetup& S, long long t_ns, const double y[9],
                                double bpos[NYXB_MAX_BODIES][3], double acc[3]) {
    accel_two_body(S, y, acc);
    return accel_point_masses(S, t_ns, y, bpos, acc);
}

__device__ inline void accel_post(const DevSetup& S, long long t_ns, const double y[9],
                                  const double bpos[NYXB_MAX_BODIES][3], double mass, double srp_area,
                                  double drag_area, double acc[3]) {
    double cr = y[6] < 0.0 ? 0.0 : (y[6] > 2.0 ? 2.0 : y[6]);  // cosmic/spacecraft.rs:494
    double cd = y[7];
    if (S.has_srp) {
        const double* sun = bpos[S.srp.sun_body];
        double rs[3] = { y[0] - sun[0], y[1] - sun[1], y[2] - sun[2] };
#if NYXB_STRICT
        double n_sun = norm3(rs[0], rs[1], rs[2]);
        double unit[3] = { rs[0] / n_sun, rs[1] / n_sun, rs[2] / n_sun };
#else
        const double d2_sun = fma(rs[2], rs[2], fma(rs[1], rs[1], rs[0] * rs[0]));
        const double i_sun = rsqrt(d2_sun);
        double unit[3] = { rs[0] * i_sun, rs[1] * i_sun, rs[2] * i_sun };
#endif
        double occult = 0.0;
        double r_ls[3] = { -rs[0], -rs[1], -rs[2] };
        for (int q = 0; q < S.srp.n_shadow; ++q) {
            int bi = S.srp.shadow_body[q];
            double r_eb[3], rad;
            if (bi == NYXB_CENTRAL_BODY) { r_eb[0] = y[0]; r_eb[1] = y[1]; r_eb[2] = y[2]; rad = S.central_radius; }
            else { r_eb[0] = y[0] - bpos[bi][0]; r_eb[1] = y[1] - bpos[bi][1]; r_eb[2] = y[2] - bpos[bi][2]; rad = S.bodies[bi].radius; }
            double p = occultation(r_eb, r_ls, S.bodies[S.srp.sun_body].radius, rad);
            if (p > occult) occult = p;
        }
        double k = fabs(occult - 1.0);
#if NYXB_STRICT
        double r_sun_au = n_sun / NYXB_AU_KM;
        double inv = 1.0 / r_sun_au;
#else
        const double inv = NYXB_AU_KM * i_sun;
#endif
        double flux_pressure = (k * S.srp.phi / NYXB_C_M_S) * (inv * inv);
        double scal = 1e-3 * cr * srp_area * flux_pressure;
#if NYXB_STRICT
        acc[0] += (scal * unit[0]) / mass; acc[1] += (scal * unit[1]) / mass; acc[2] += (scal * unit[2]) / mass;
#else
        const double sm = scal / mass;
        acc[0] = fma(sm, unit[0], acc[0]); acc[1] = fma(sm, unit[1], acc[1]); acc[2] = fma(sm, unit[2], acc[2]);
#endif
    }
    if (S.has_drag) {
        double R[9];
        rotation_dcm(S.drag.rot, t_ns, R);
        double wdot = S.drag.rot.wdot;
        double rb[3], vb[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            rb[i] = (R[3 * i] * y[0] + R[3 * i + 1] * y[1]) + R[3 * i + 2] * y[2];
            vb[i] = (R[3 * i] * y[3] + R[3 * i + 1] * y[4]) + R[3 * i + 2] * y[5];
        }
        vb[0] = vb[0] + wdot * rb[1];
        vb[1] = vb[1] - wdot * rb[0];
        double rho, vel[3];
        if (S.drag.density == NYXB_DENSITY_CONSTANT) {
            rho = S.drag.rho0;
            vel[0] = vb[0]; vel[1] = vb[1]; vel[2] = vb[2];
        } else {
            double rmag_bf = norm3(rb[0], rb[1], rb[2]);
            if (S.drag.density == NYXB_DENSITY_EXPONENTIAL) {
                rho = S.drag.rho0 * exp(-(rmag_bf - (S.drag.r0 + S.drag.r_eq)) / S.drag.ref_alt_m);
            } else {
                double alt = rmag_bf - S.drag.r_eq;
                if (alt > S.drag.ref_alt_m / 1000.0) {
                    rho = pow(10.0, (-7e-5) * alt - 14.464);
                } else {
                    double sc = (alt - 526.8000) / 292.8563;
                    double s2 = sc * sc, s3 = s2 * sc, s4 = s3 * sc, s5 = s4 * sc, s6 = s5 * sc;
                    double logd = 0.34047 * s6 - 0.5889 * s5 - 0.5269 * s4 + 1.0036 * s3 + 0.60713 * s2 - 2.3024 * sc - 12.575;
                    rho = pow(10.0, logd);
                }
            }
            vel[0] = y[3] - vb[0]; vel[1] = y[4] - vb[1]; vel[2] = y[5] - vb[2];
        }
        double scal = -0.5 * 1e3 * rho * cd * drag_area * norm3(vel[0], vel[1], vel[2]);
        acc[0] += (scal * vel[0]) / mass; acc[1] += (scal * vel[1]) / mass; acc[2] += (scal * vel[2]) / mass;
    }
}

// position of the spacecraft relative to the body a harmonic field belongs to (gravity_field.rs:149-154: transform_to the
// field's frame; the body-fixed rotation follows inside the field evaluation)
__device__ __forceinline__ void grav_rel(int body, const double y[9], const double bpos[NYXB_MAX_BODIES][3], double rel[3]) {
    if (body < 0) { rel[0] = y[0]; rel[1] = y[1]; rel[2] = y[2]; }
    else { rel[0] = y[0] - bpos[body][0]; rel[1] = y[1] - bpos[body][1]; rel[2] = y[2] - bpos[body][2]; }
}

// harmonic fields beyond the primary one (OrbitalDynamics holds a Vec of accel models, orbital.rs:44-46, 102-107), summed per
// trajectory in list order
// (out of line: the per-thread harmonic evaluation carries a large register / stack footprint that must not leak into its callers)
static __device__ __noinline__ void accel_extra_fields(const DevSetup& S, long long t_ns, const double y[9],
                                                const double bpos[NYXB_MAX_BODIES][3], double acc[3]) {
    for (int f = 0; f < S.n_xgrav; ++f) {
        double rel[3], ga[3];
        grav_rel(S.xgrav_body[f], y, bpos, rel);
#if NYXB_STRICT
        grav_accel_rows(S.xgrav[f], t_ns, rel, ga);
#else
        grav_accel_cols(S.xgrav[f], t_ns, rel, ga);
#endif
        acc[0] += ga[0]; acc[1] += ga[1]; acc[2] += ga[2];
    }
}

// SpacecraftDynamics::eom for one trajectory on one thread: y[9] -> dy[0..5] (dy[6..8] == 0).
// Returns 0 or an nyxb_status error code.
template <bool GRAV = true>
__device__ inline int eom_full(const DevSetup& S, long long epoch_ns, double delta_t_s, const double y[9],
                               double dry_mass, double extra_mass, double srp_area, double drag_area, double dy[6]) {
    long long t_ns = epoch_ns + dur_from_seconds(delta_t_s);
    double mass = dry_mass + y[8] + extra_mass;
    bool has_force = S.has_srp || S.has_drag;
    if (has_force && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3];
    double bpos[NYXB_MAX_BODIES][3];
    int rc = accel_pre(S, t_ns, y, bpos, acc);
    if (rc) return rc;
    if (GRAV && S.has_grav) {
        double ga[3], rel[3];
        grav_rel(S.grav_body, y, bpos, rel);
#if NYXB_STRICT
        grav_accel_rows(S.grav, t_ns, rel, ga);
#else
        grav_accel_cols(S.grav, t_ns, rel, ga);
#endif
        acc[0] += ga[0]; acc[1] += ga[1]; acc[2] += ga[2];
        if (S.n_xgrav > 0) accel_extra_fields(S, t_ns, y, bpos, acc);
    }
    if (has_force) accel_post(S, t_ns, y, bpos, mass, srp_area, drag_area, acc);
    dy[0] = y[3]; dy[1] = y[4]; dy[2] = y[5];
    dy[3] = acc[0]; dy[4] = acc[1]; dy[5] = acc[2];
    return 0;
}

// Cold part of the right-hand side in the cooperative and transposed kernels, whose harmonic sum is evaluated apart: third bodies,
// further fields (GEN), SRP and drag added onto acc.  Out of line so that the ephemeris scratch does not inflate the register count
// of the harmonic sum (scalars, not a context struct, are passed: taking a struct's address would force it into local memory).
template <bool GEN>
static __device__ __noinline__ int accel_cold(const DevSetup& S, double dry_mass, double extra_mass, double srp_area, double drag_area,
                                              long long t_ns, const double y[9], double acc[3]) {
    const double mass = dry_mass + y[8] + extra_mass;
    const bool has_force = S.has_srp || S.has_drag;
    if (has_force && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double bpos[NYXB_MAX_BODIES][3];
    const int rc = accel_point_masses(S, t_ns, y, bpos, acc);
    if (rc) return rc;
    if (GEN && S.n_xgrav > 0) accel_extra_fields(S, t_ns, y, bpos, acc);
    if (has_force) accel_post(S, t_ns, y, bpos, mass, srp_area, drag_area, acc);
    return 0;
}

// position relative to the body the primary field belongs to (gravity_field.rs:149-154); out of line: the Clenshaw scratch must not
// inflate the register count of the harmonic sum.  An epoch outside the ephemeris is reported by accel_cold, which evaluates every body.
static __device__ __noinline__ void field_offset(const DevSetup& S, long long t_ns, double& y0, double& y1, double& y2) {
    double bp[3];
    if (body_position(S.bodies[S.grav_body], t_ns, bp)) { y0 -= bp[0]; y1 -= bp[1]; y2 -= bp[2]; }
}

// ---- ErrorControl::estimate (error_ctrl.rs:79-230); err/cand/cur are 9-vectors whose
// entries 6..8 carry zero error (their derivatives are zero without guidance).
__device__ __forceinline__ double rss_step3(const double* e, const double* cand, const double* cur) {
    double mag = norm3(cand[0] - cur[0], cand[1] - cur[1], cand[2] - cur[2]);
    double err = norm3(e[0], e[1], e[2]);
    return (mag > sqrt(0.1)) ? err / mag : err;
}
__device__ __forceinline__ double rss_state3(const double* e, const double* cand, const double* cur) {
    double mag = 0.5 * norm3(cand[0] + cur[0], cand[1] + cur[1], cand[2] + cur[2]);
    double err = norm3(e[0], e[1], e[2]);
    return (mag > 0.1) ? err / mag : err;
}
__device__ __forceinline__ double fmax_rust(double a, double b) { return (a > b || b != b) ? a : b; }
__device__ __forceinline__ double norm9_nalgebra(const double v[9]) {
    // nalgebra generic dot: 8 interleaved accumulators (see oracle/nyx_oracle.c)
    double a0 = __dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[8], v[8]));
    double res = 0.0;
    res = __dadd_rn(res, __dadd_rn(a0, __dmul_rn(v[4], v[4])));
    res = __dadd_rn(res, __dadd_rn(__dmul_rn(v[1], v[1]), __dmul_rn(v[5], v[5])));
    res = __dadd_rn(res, __dadd_rn(__dmul_rn(v[2], v[2]), __dmul_rn(v[6], v[6])));
    res = __dadd_rn(res, __dadd_rn(__dmul_rn(v[3], v[3]), __dmul_rn(v[7], v[7])));
    return sqrt(res);
}

__device__ inline double error_estimate(int ctrl, const double err[9], const double cand[9], const double cur[9]) {
    switch (ctrl) {
    case NYXB_RSS_CARTESIAN_STATE:
        return fmax_rust(rss_state3(err, cand, cur), rss_state3(err + 3, cand + 3, cur + 3));
    case NYXB_RSS_CARTESIAN_STEP:
        return fmax_rust(rss_step3(err, cand, cur), rss_step3(err + 3, cand + 3, cur + 3));
    case NYXB_RSS_STATE: {
        double s[9];
        for (int i = 0; i < 9; ++i) s[i] = cand[i] + cur[i];
        double mag = 0.5 * norm9_nalgebra(s), e = norm9_nalgebra(err);
        return (mag > 0.1) ? e / mag : e;
    }
    case NYXB_RSS_STEP: {
        double d[9];
        for (int i = 0; i < 9; ++i) d[i] = cand[i] - cur[i];
        double mag = norm9_nalgebra(d), e = norm9_nalgebra(err);
        return (mag > sqrt(0.1)) ? e / mag : e;
    }
    case NYXB_LARGEST_ERROR: {
        double max_err = 0.0;
        for (int i = 0; i < 9; ++i) {
            double delta = cand[i] - cur[i];
            double e = (delta > 0.1) ? fabs(err[i] / delta) : fabs(err[i]);
            if (e > max_err) max_err = e;
        }
        return max_err;
    }
    case NYXB_LARGEST_STATE: {
        double mag = 0.0, e = 0.0;
        for (int i = 0; i < 9; ++i) { mag += 0.5 * fabs(cand[i] + cur[i]); e += fabs(err[i]); }
        return (mag > 0.1) ? e / mag : e;
    }
    default: {
        double mag = 0.0, e = 0.0;
        for (int i = 0; i < 9; ++i) { mag += fabs(cand[i] - cur[i]); e += fabs(err[i]); }
        return (mag > 0.1) ? e / mag : e;
    }
    }
}

// ---- step-size controller of every kernel family (instance.rs:149-196, 416-490).  Each kernel keeps the controller state in its own
// storage and checks the candidate for NaN itself; ROOT is x^(1/n): pow_inv_int, or the transposed kernel's tx_pow_inv_int.
// The clamps are NaN-sensitive as written: (p < min) ? min : p is not fmax.

// the final step of a run: the regular step would pass the stop epoch (forward) or reach it (backward)
__device__ __forceinline__ bool ctl_past_stop(long long epoch, long long step_ns, long long stop, bool backprop) {
    return backprop ? epoch + step_ns <= stop : epoch + step_ns > stop;
}

// an attempt of h seconds with error estimate err is accepted
__device__ __forceinline__ bool ctl_accept(const DevSetup& S, double err, double h, int attempts) {
    return err <= S.tolerance || h <= S.min_step_s || attempts >= S.attempts;
}

// after an accepted attempt: the max-attempts warning, the step taken (det_step, ns) and, returned, the step of the next attempt (ns)
template <double (*ROOT)(double, int)>
__device__ __forceinline__ long long ctl_accepted(const DevSetup& S, double err, double h, int attempts, int& status, long long& det_step) {
    if (attempts >= S.attempts) status |= NYXB_WARN_MAX_ATTEMPTS;
    det_step = dur_from_seconds(h);
    if (err < S.tolerance) {
        const double proposed = 0.9 * h * ROOT(S.tolerance / err, S.tb.order);
        if (fabs(proposed) > fabs(S.max_step_s)) {
            const double sg = (proposed != proposed) ? proposed : (signbit(proposed) ? -1.0 : 1.0);
            h = S.max_step_s * sg;
        } else {
            h = proposed;
        }
    }
    long long step_ns = dur_from_seconds(h);
    const long long ab = step_ns < 0 ? -step_ns : step_ns;
    if (ab < S.min_step_ns) step_ns = (step_ns < 0) ? -S.min_step_ns : S.min_step_ns;
    return step_ns;
}

// the step (seconds, unquantised) of the retry after a rejected attempt
template <double (*ROOT)(double, int)>
__device__ __forceinline__ double ctl_retry(const DevSetup& S, double err, double h) {
    const double proposed = 0.9 * h * ROOT(S.tolerance / err, S.tb.order - 1);
    return (proposed < S.min_step_s) ? S.min_step_s : proposed;
}

// end of a run of trajectory i: event crossings and event-not-found (event.rs:177-182), the recorded count; returns the status word
__device__ __forceinline__ int ctl_finish(const DevSink& sink, size_t i, int status, int rc, int crossings, long long n_steps) {
    if (sink.ev_kind) {
        sink.ev_crossings[i] = crossings;
        if (rc == 0 && crossings < sink.ev_trigger) rc = NYXB_ERR_EVENT_NOT_FOUND;
    }
    if (sink.cap > 0) sink.count[i] = (n_steps + 1 < sink.cap) ? n_steps + 1 : sink.cap;
    return (status & NYXB_WARN_MAX_ATTEMPTS) | rc;
}

// ---- shared-memory addressing and the TMA 1-D bulk copy global -> shared with completion on an mbarrier (SASS: UBLKCP + SYNCS),
// used by the cooperative and transposed kernels to stage their coefficient tables
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
