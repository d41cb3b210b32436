// nyxb_target.h — the per-problem arithmetic of the finite-difference targeter (md/opti/raphson_finite_diff.rs:41-747, impulsive
// variables only) as host/device inline functions: objective values, the local-frame DCMs, applying a correction, and one correction
// step from the nominal and perturbed final states.  Used by the update kernels (nyxb_target.cu); plain C++ when not compiled by nvcc,
// so that a CPU test checks the same arithmetic against the restatement (tests/cpp/target_core_shim.cpp, tests/target_oracle.py).
// Both sides are built without FMA contraction; they then agree up to the libm ulps of acos / asin.
//
// The objective values follow nyx_b200/param.py operation by operation (anise's OrbitalElement is not in the reference tree).  The
// pseudo-inverse is the reference's (utils.rs:429-445): J^T (J J^T)^-1 when O < V, else (J^T J)^-1 J^T, with the m x m inverse
// from nyxb_inv9 on the matrix padded with an identity block (the padding neither pivots nor changes the leading block).
#pragma once
#include <math.h>

#include "../../include/nyxb.h"
#include "nyxb_smooth.h"

enum { NYXB_TGT_CONTINUE = -1 };

NYXB_SHD double nyxb_tgt_deg(double rad) { return rad * (180.0 / 3.14159265358979323846); }

// np.mod(a, 360.0) for a finite a
NYXB_SHD double nyxb_tgt_wrap360(double a) {
    double m = fmod(a, 360.0);
    if (m != 0.0 && m < 0.0) m += 360.0;
    if (m == 0.0) m = 0.0;
    return m;
}

NYXB_SHD double nyxb_tgt_angle(double c, bool flip) {
    const double cc = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c);
    const double ang = nyxb_tgt_deg(acos(cc));
    return flip ? 360.0 - ang : ang;
}

// value of parameter `param` (enum nyxb_tgt_param) of the Cartesian state rv[6] around a body of gravitational parameter mu
NYXB_SHD double nyxb_tgt_eval(int param, const double* rv, double mu) {
    if (param <= NYXB_TGT_VZ) return rv[param];
    const double* r = rv;
    const double* v = rv + 3;
    const double rmag = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    const double vmag = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (param == NYXB_TGT_RMAG) return rmag;
    if (param == NYXB_TGT_VMAG) return vmag;
    if (param == NYXB_TGT_DECLINATION) return nyxb_tgt_deg(asin(r[2] / rmag));
    const double energy = 0.5 * vmag * vmag - mu / rmag;
    if (param == NYXB_TGT_ENERGY) return energy;
    const double sma = -mu / (2.0 * energy);
    if (param == NYXB_TGT_SMA) return sma;
    if (param == NYXB_TGT_C3) return -mu / sma;
    if (param == NYXB_TGT_PERIOD) return 2.0 * 3.14159265358979323846 * sqrt(sma * sma * sma / mu);
    const double h[3] = {r[1] * v[2] - r[2] * v[1], r[2] * v[0] - r[0] * v[2], r[0] * v[1] - r[1] * v[0]};
    const double hmag = sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    if (param == NYXB_TGT_HMAG) return hmag;
    const double rdv = r[0] * v[0] + r[1] * v[1] + r[2] * v[2];
    const double k = vmag * vmag - mu / rmag;
    const double e[3] = {(k * r[0] - rdv * v[0]) / mu, (k * r[1] - rdv * v[1]) / mu, (k * r[2] - rdv * v[2]) / mu};
    const double ecc = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    if (param == NYXB_TGT_ECC) return ecc;
    if (param == NYXB_TGT_APOAPSIS) return sma * (1.0 + ecc);
    if (param == NYXB_TGT_PERIAPSIS) return sma * (1.0 - ecc);
    if (param == NYXB_TGT_INC) return nyxb_tgt_angle(h[2] / hmag, false);
    const double nd[3] = {-h[1], h[0], 0.0};   // z x h
    const double nmag = sqrt(nd[0] * nd[0] + nd[1] * nd[1] + nd[2] * nd[2]);
    const double raan = nyxb_tgt_angle(nd[0] / nmag, nd[1] < 0.0);
    if (param == NYXB_TGT_RAAN) return raan;
    const double aop = nyxb_tgt_angle((nd[0] * e[0] + nd[1] * e[1] + nd[2] * e[2]) / (nmag * ecc), e[2] < 0.0);
    if (param == NYXB_TGT_AOP) return aop;
    const double ta = nyxb_tgt_angle((e[0] * r[0] + e[1] * r[1] + e[2] * r[2]) / (ecc * rmag), rdv < 0.0);
    if (param == NYXB_TGT_TA) return ta;
    if (param == NYXB_TGT_AOL) return nyxb_tgt_wrap360(aop + ta);
    return nyxb_tgt_wrap360(aop + raan + ta);   // NYXB_TGT_TLONG
}

// Row-major local -> inertial DCM of rv for `frame` (VNC or RIC)
NYXB_SHD void nyxb_tgt_dcm(int frame, const double* rv, double* D) {
    const double* r = rv;
    const double* v = rv + 3;
    const double h[3] = {r[1] * v[2] - r[2] * v[1], r[2] * v[0] - r[0] * v[2], r[0] * v[1] - r[1] * v[0]};
    const double hm = sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    const double c[3] = {h[0] / hm, h[1] / hm, h[2] / hm};
    const double* a = (frame == NYXB_TGT_FRAME_VNC) ? v : r;
    const double am = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    const double u[3] = {a[0] / am, a[1] / am, a[2] / am};
    double col[3][3];
    if (frame == NYXB_TGT_FRAME_VNC) {   // V = v^, N = h^, C = V x N
        for (int i = 0; i < 3; ++i) { col[0][i] = u[i]; col[1][i] = c[i]; }
        col[2][0] = u[1] * c[2] - u[2] * c[1]; col[2][1] = u[2] * c[0] - u[0] * c[2]; col[2][2] = u[0] * c[1] - u[1] * c[0];
    } else {                             // R = r^, C = h^, I = C x R
        for (int i = 0; i < 3; ++i) { col[0][i] = u[i]; col[2][i] = c[i]; }
        col[1][0] = c[1] * u[2] - c[2] * u[1]; col[1][1] = c[2] * u[0] - c[0] * u[2]; col[1][2] = c[0] * u[1] - c[1] * u[0];
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) D[i * 3 + j] = col[j][i];
}

// Apply the state correction sc[6] to rv[6]: with a frame as the Δv D sc[3..6] with D the DCM of rv itself (apply_dv_km_s), without
// one to r and v (`Spacecraft + Vector6`, cosmic/spacecraft.rs:698-711)
NYXB_SHD void nyxb_tgt_apply(int frame, const double* sc, double* rv) {
    if (frame == NYXB_TGT_FRAME_NONE) {
        for (int i = 0; i < 6; ++i) rv[i] += sc[i];
        return;
    }
    double D[9];
    nyxb_tgt_dcm(frame, rv, D);
    double dv[3];
    for (int i = 0; i < 3; ++i) dv[i] = D[i * 3 + 0] * sc[3] + D[i * 3 + 1] * sc[4] + D[i * 3 + 2] * sc[5];
    for (int i = 0; i < 3; ++i) rv[3 + i] += dv[i];
}

// rv + the correction x[V] (one entry per variable, duplicates add up), applied once
NYXB_SHD void nyxb_tgt_apply_vars(const nyxb_target_config& cfg, const double* x, double* rv) {
    double sc[6] = {0, 0, 0, 0, 0, 0};
    for (int j = 0; j < cfg.n_vars; ++j) sc[cfg.vars[j].component] += x[j];
    nyxb_tgt_apply(cfg.correction_frame, sc, rv);
}

// start state of perturbed propagation j (0..V-1): xi with variable j's perturbation
NYXB_SHD void nyxb_tgt_perturbed(const nyxb_target_config& cfg, int j, const double* xi, double* out) {
    for (int i = 0; i < 6; ++i) out[i] = xi[i];
    double sc[6] = {0, 0, 0, 0, 0, 0};
    sc[cfg.vars[j].component] += cfg.vars[j].perturbation;
    nyxb_tgt_apply(cfg.correction_frame, sc, out);
}

// One iteration from the final states xf (nominal at xf[0..6], perturbation j at xf[6 (j + 1)..]) of propagations that all
// succeeded.  Writes err[O]; returns 0 (converged), NYXB_ERR_TGT_NON_FINITE, _CORRECTION_INEFFECTIVE or _SINGULAR_JACOBIAN (xi,
// total, prev_norm unchanged), or, after the step has updated xi[6], total[V] and prev_norm: NYXB_ERR_TGT_TOO_MANY_ITERATIONS when
// it == cfg.iterations, else NYXB_TGT_CONTINUE.
NYXB_SHD int nyxb_tgt_step(const nyxb_target_config& cfg, double mu, int it, const double* xf, double* xi, double* total, double* err,
                           double* prev_norm) {
    const int V = cfg.n_vars, O = cfg.n_objs;
    double ach[6], J[36];
    for (int i = 0; i < O; ++i) err[i] = NAN;
    for (int i = 0; i < O; ++i) {
        ach[i] = nyxb_tgt_eval(cfg.objs[i].parameter, xf, mu);
        if (!isfinite(ach[i])) return NYXB_ERR_TGT_NON_FINITE;
    }
    for (int j = 0; j < V; ++j)
        for (int i = 0; i < O; ++i) {
            const double a = nyxb_tgt_eval(cfg.objs[i].parameter, xf + 6 * (j + 1), mu);
            const double d = (a - ach[i]) / cfg.vars[j].perturbation;
            if (!isfinite(a) || !isfinite(d)) return NYXB_ERR_TGT_NON_FINITE;
            J[i * V + j] = d;
        }
    bool converged = true;
    for (int i = 0; i < O; ++i) {
        const nyxb_tgt_objective& o = cfg.objs[i];
        err[i] = o.multiplicative_factor * (o.desired - ach[i]) + o.additive_factor;
        if (!(fabs(err[i]) <= o.tolerance)) converged = false;
    }
    if (converged) return 0;
    double nsq = 0.0;
    for (int i = 0; i < O; ++i) nsq += err[i] * err[i];
    const double norm = sqrt(nsq);
    if (fabs(norm - *prev_norm) < 1e-10) return NYXB_ERR_TGT_CORRECTION_INEFFECTIVE;
    *prev_norm = norm;
    // pseudo-inverse P [V][O]
    const int m = O < V ? O : V;
    double A[81], LU[81], Ai[81], P[36];
    for (int e = 0; e < 81; ++e) A[e] = (e % 10 == 0) ? 1.0 : 0.0;
    for (int a = 0; a < m; ++a)
        for (int b = 0; b < m; ++b) {
            double s = 0.0;
            if (O < V) for (int k = 0; k < V; ++k) s += J[a * V + k] * J[b * V + k];   // J J^T
            else       for (int k = 0; k < O; ++k) s += J[k * V + a] * J[k * V + b];   // J^T J
            A[a * 9 + b] = s;
        }
    if (!nyxb_inv9(A, LU, Ai)) return NYXB_ERR_TGT_SINGULAR_JACOBIAN;
    for (int r = 0; r < V; ++r)
        for (int c = 0; c < O; ++c) {
            double s = 0.0;
            if (O < V) for (int k = 0; k < O; ++k) s += J[k * V + r] * Ai[k * 9 + c];   // J^T M^-1
            else       for (int k = 0; k < V; ++k) s += Ai[r * 9 + k] * J[c * V + k];   // M^-1 J^T
            P[r * O + c] = s;
        }
    double delta[6];
    for (int r = 0; r < V; ++r) {
        double s = 0.0;
        for (int c = 0; c < O; ++c) s += P[r * O + c] * err[c];
        // the clip and the bounds apply to the step, not to the total (raphson_finite_diff.rs:710-717)
        const nyxb_tgt_variable& var = cfg.vars[r];
        if (fabs(s) > fabs(var.max_step)) s = fabs(var.max_step) * (s < 0.0 ? -1.0 : 1.0);
        else if (s > var.max_value) s = var.max_value;
        else if (s < var.min_value) s = var.min_value;
        delta[r] = s;
    }
    nyxb_tgt_apply_vars(cfg, delta, xi);
    for (int r = 0; r < V; ++r) total[r] += delta[r];
    return it >= cfg.iterations ? (int)NYXB_ERR_TGT_TOO_MANY_ITERATIONS : (int)NYXB_TGT_CONTINUE;
}
