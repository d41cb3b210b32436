// nyxb_od_device.cuh — device code shared by the per-thread (nyxb_od.cu) and the warp-cooperative (nyxb_od_coop.cu)
// STM / filter kernels: 3-partial dual numbers, the dual right-hand side (spacecraft.rs:312-363 and what it calls) and
// the tracking geometry (trk_device.rs:150-200).
#pragma once
#include "nyxb_od.cuh"

// ------------------------------------------------------------------------- dual numbers (value + d/dx, d/dy, d/dz)
struct D3 { double v, x, y, z; };
__device__ __forceinline__ D3 dc(double v) { return D3{v, 0.0, 0.0, 0.0}; }
__device__ __forceinline__ D3 dvar(double v, int i) { return D3{v, i == 0 ? 1.0 : 0.0, i == 1 ? 1.0 : 0.0, i == 2 ? 1.0 : 0.0}; }
__device__ __forceinline__ D3 operator+(D3 a, D3 b) { return D3{a.v + b.v, a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ D3 operator-(D3 a, D3 b) { return D3{a.v - b.v, a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ D3 operator*(D3 a, D3 b) {
    return D3{a.v * b.v, b.v * a.x + a.v * b.x, b.v * a.y + a.v * b.y, b.v * a.z + a.v * b.z};
}
__device__ __forceinline__ D3 operator/(D3 a, D3 b) {
#if NYXB_STRICT
    double den = b.v * b.v;
    return D3{a.v / b.v, (b.v * a.x - a.v * b.x) / den, (b.v * a.y - a.v * b.y) / den, (b.v * a.z - a.v * b.z) / den};
#else
    const double r = 1.0 / b.v, q = a.v * r;   // FAST: one division; d(a/b) = (da - (a/b) db) / b
    return D3{q, (a.x - q * b.x) * r, (a.y - q * b.y) * r, (a.z - q * b.z) * r};
#endif
}
__device__ __forceinline__ D3 dscale(D3 a, double c) { return D3{a.v * c, a.x * c, a.y * c, a.z * c}; }
__device__ __forceinline__ D3 ddivs(D3 a, double c) { return D3{a.v / c, a.x / c, a.y / c, a.z / c}; }
__device__ __forceinline__ D3 dsq(D3 a) { double p = 2.0 * a.v; return D3{a.v * a.v, p * a.x, p * a.y, p * a.z}; }
__device__ __forceinline__ D3 dcube(D3 a) { double p = 3.0 * (a.v * a.v); return D3{(a.v * a.v) * a.v, p * a.x, p * a.y, p * a.z}; }
__device__ __forceinline__ D3 dsqrt(D3 a) {
    double r = sqrt(a.v), dd = 1.0 / (2.0 * r);
    return D3{r, a.x * dd, a.y * dd, a.z * dd};
}
__device__ __forceinline__ D3 dnorm(D3 a, D3 b, D3 c) { return dsqrt(((dc(0.0) + dsq(a)) + dsq(b)) + dsq(c)); }
__device__ __forceinline__ double dpart(const D3& a, int j) { return j == 0 ? a.x : (j == 1 ? a.y : a.z); }

// ------------------------------------------------------------------------- GravityField::gradient (gravity_field.rs:273-431)
// rolling rows of the derived-Legendre triangle in dual numbers: P = row n, Q = row n-1 -> row n+1
__device__ static void grav_gradient(const DevGrav& g, long long t_ns, const double r_in[3], double acc[3], double G[9]) {
    const int N = g.N, M = g.M;
    double R[9];
    rotation_dcm(g.rot, t_ns, R);
    double rb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = (R[3 * i] * r_in[0] + R[3 * i + 1] * r_in[1]) + R[3 * i + 2] * r_in[2];
    D3 rx = dvar(rb[0], 0), ry = dvar(rb[1], 1), rz = dvar(rb[2], 2);
    D3 r_ = dnorm(rx, ry, rz);
    D3 s_ = rx / r_, t_ = ry / r_, u_ = rz / r_;
    D3 rowA[NYXB_MAX_DEGREE + 3], rowB[NYXB_MAX_DEGREE + 3];
    D3 r_m[NYXB_MAX_DEGREE + 1], i_m[NYXB_MAX_DEGREE + 1];
    D3* P = rowA;
    D3* Q = rowB;
    for (int m = 0; m <= N + 2; ++m) { rowA[m] = dc(0.0); rowB[m] = dc(0.0); }
    Q[0] = dc(1.0);
    P[0] = dscale(u_, sqrt(3.0));
    P[1] = dc(__ldg(g.a_diag + 1));
    const int mm = N < M ? N : M;
    r_m[0] = dc(1.0); i_m[0] = dc(0.0);
    for (int m = 1; m <= mm; ++m) {
        r_m[m] = s_ * r_m[m - 1] - t_ * i_m[m - 1];
        i_m[m] = s_ * i_m[m - 1] + t_ * r_m[m - 1];
    }
    D3 eq_radius = dc(g.r_eq);
    D3 rho = eq_radius / r_;
    D3 rho_np1 = (dc(g.mu) / r_) * rho;
    D3 a0 = dc(0.0), a1 = dc(0.0), a2 = dc(0.0), a3 = dc(0.0);
    const D3 sqrt2 = dc(sqrt(2.0));
    for (int n = 1; n <= N; ++n) {
        {   // row n+1 into Q (holds row n-1): gravity_field.rs:305-317
            const int np1 = n + 1;
            const DevHarm* trow = g.tab + tri(np1, 0);
            int mrec = np1 - 2;
            if (mrec > M + 1) mrec = M + 1;
            for (int m = 0; m <= mrec; ++m) {
                double bb = __ldg(&trow[m].b), cc = __ldg(&trow[m].c);
                Q[m] = (u_ * dc(bb)) * P[m] - dc(cc) * Q[m];
            }
            for (int m = mrec + 1; m <= np1 - 2; ++m) Q[m] = dc(0.0);
            Q[n] = (dc(__ldg(g.offdiag + n)) * u_) * dc(__ldg(g.a_diag + n));
            Q[np1] = dc(__ldg(g.a_diag + np1));
        }
        D3 sum0 = dc(0.0), sum1 = dc(0.0), sum2 = dc(0.0), sum3 = dc(0.0);
        rho_np1 = rho_np1 * rho;
        const DevHarm* trow = g.tab + tri(n, 0);
        int mtop = n < M ? n : M;
        for (int m = 0; m <= mtop; ++m) {
            D3 cv = dc(__ldg(&trow[m].cbar)), sv = dc(__ldg(&trow[m].sbar));
            D3 d_ = (cv * r_m[m] + sv * i_m[m]) * sqrt2;
            D3 e_ = dc(0.0), f_ = dc(0.0);
            if (m != 0) {
                e_ = (cv * r_m[m - 1] + sv * i_m[m - 1]) * sqrt2;
                f_ = (sv * r_m[m - 1] - cv * i_m[m - 1]) * sqrt2;
            }
            D3 mf = dc((double)m);
            sum0 = sum0 + (mf * P[m]) * e_;
            sum1 = sum1 + (mf * P[m]) * f_;
            sum2 = sum2 + (dc(__ldg(&trow[m].vr01)) * P[m + 1]) * d_;
            sum3 = sum3 + (dc(__ldg(&trow[m].vr11)) * Q[m + 1]) * d_;
        }
        D3 rr = rho_np1 / eq_radius;
        a0 = a0 + rr * sum0;
        a1 = a1 + rr * sum1;
        a2 = a2 + rr * sum2;
        a3 = a3 - rr * sum3;
        D3* tmp = P; P = Q; Q = tmp;
    }
    D3 al[3] = { a0 + a3 * s_, a1 + a3 * t_, a2 + a3 * u_ };
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
            G[3 * i + j] = (tmp9[3 * i] * R[j] + tmp9[3 * i + 1] * R[3 + j]) + tmp9[3 * i + 2] * R[6 + j];
}

// ------------------------------------------------------------------------- dual_eom (spacecraft.rs:312-363)
// y[9] with Cr already clamped; outputs: acc[3], G[9] = d(acc)/d(r) row-major, gcr[3] = d(acc)/d(Cr)
template <bool WITH_GRAV>
__device__ static int dual_eom_dev(const DevSetup& S, long long t_ns, const double y[9], double total_mass, double srp_area,
                                   double acc[3], double G[9], double gcr[3]) {
    // OrbitalDynamics::dual_eom, orbital.rs:116-172
    D3 rad[3] = { dvar(y[0], 0), dvar(y[1], 1), dvar(y[2], 2) };
    D3 rmag = dnorm(rad[0], rad[1], rad[2]);
    D3 fac = dc(-S.mu_central) / dcube(rmag);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        D3 ba = rad[i] * fac;
        acc[i] = ba.v;
        G[3 * i] = ba.x; G[3 * i + 1] = ba.y; G[3 * i + 2] = ba.z;
        gcr[i] = 0.0;
    }
    double bpos[NYXB_MAX_BODIES][3];
    for (int j = 0; j < S.n_bodies; ++j)
        if (!body_position(S.bodies[j], t_ns, bpos[j])) return NYXB_ERR_EPHEMERIS;
    if (S.point_mass_mask) {  // PointMasses::gradient, orbital.rs:249-307 (r_ij carries identity partials, as coded)
        double fx[3] = {0.0, 0.0, 0.0}, gp[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int j = 0; j < S.n_bodies; ++j) {
            if (!((S.point_mass_mask >> j) & 1u)) continue;
            D3 gm_d = dc(-S.bodies[j].mu);
            D3 rij[3] = { dvar(bpos[j][0], 0), dvar(bpos[j][1], 1), dvar(bpos[j][2], 2) };
            D3 rij3 = dcube(dnorm(rij[0], rij[1], rij[2]));
            D3 rj[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) { rj[i] = rad[i] - rij[i]; }
            rj[0].x = 1.0; rj[1].y = 1.0; rj[2].z = 1.0;
            D3 rj3 = dcube(dnorm(rj[0], rj[1], rj[2]));
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                D3 t = (rj[i] / rj3 + rij[i] / rij3) * gm_d;
                fx[i] += t.v;
                gp[3 * i] += t.x; gp[3 * i + 1] += t.y; gp[3 * i + 2] += t.z;
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i] += fx[i];
#pragma unroll
        for (int q = 0; q < 9; ++q) G[q] += gp[q];
    }
    if (WITH_GRAV && S.has_grav) {
        double ga[3], gg[9];
        grav_gradient(S.grav, t_ns, y, ga, gg);
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i] += ga[i];
#pragma unroll
        for (int q = 0; q < 9; ++q) G[q] += gg[q];
    }
    if (S.has_srp) {  // SolarPressure::gradient, solarpressure.rs:167-233
        const double cr = y[6];
        const double* sun = bpos[S.srp.sun_body];
        double rs[3] = { y[0] - sun[0], y[1] - sun[1], y[2] - sun[2] };
        D3 rsd[3] = { dvar(rs[0], 0), dvar(rs[1], 1), dvar(rs[2], 2) };
        D3 n_d = dnorm(rsd[0], rsd[1], rsd[2]);
        double occult = 0.0;
        double r_ls[3] = { -rs[0], -rs[1], -rs[2] };
        for (int q = 0; q < S.srp.n_shadow; ++q) {
            int bi = S.srp.shadow_body[q];
            double r_eb[3], radb;
            if (bi == NYXB_CENTRAL_BODY) { r_eb[0] = y[0]; r_eb[1] = y[1]; r_eb[2] = y[2]; radb = S.central_radius; }
            else { r_eb[0] = y[0] - bpos[bi][0]; r_eb[1] = y[1] - bpos[bi][1]; r_eb[2] = y[2] - bpos[bi][2]; radb = S.bodies[bi].radius; }
            double p = occultation(r_eb, r_ls, S.bodies[S.srp.sun_body].radius, radb);
            if (p > occult) occult = p;
        }
        double k = fabs(occult - 1.0);
        D3 r_sun_au = ddivs(n_d, NYXB_AU_KM);
        D3 inv = dc(1.0) / r_sun_au;
        D3 flux = dc(k * S.srp.phi / NYXB_C_M_S) * dsq(inv);
        D3 scal = dc(1e-3 * cr * srp_area);
        double n_sun = norm3(rs[0], rs[1], rs[2]);
        double r_au = n_sun / NYXB_AU_KM, inv_s = 1.0 / r_au;
        double flux_s = (k * S.srp.phi / NYXB_C_M_S) * (inv_s * inv_s);
        double scal_s = 1e-3 * cr * srp_area * flux_s;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            D3 f = (scal * flux) * (rsd[i] / n_d);
            acc[i] += f.v / total_mass;
            G[3 * i] += f.x / total_mass; G[3 * i + 1] += f.y / total_mass; G[3 * i + 2] += f.z / total_mass;
            if (S.srp.estimate) gcr[i] += ((scal_s * (rs[i] / n_sun)) / cr) / total_mass;
        }
    }
    return 0;
}

// ------------------------------------------------------------------------- tracking geometry
// trk_device.rs:150-152 `location`: antenna position / velocity in the integration frame and the inertial zenith.  St: DevStation, or
// DevAerStation, whose body-fixed north and east are rotated alike into ne[0] and ne[1].
template <class St>
__device__ static bool station_state(const DevSetup& S, const St& st, long long t_ns, double r[3], double v[3], double up[3], double ne[2][3]) {
    double R[9];
    rotation_dcm(st.rot, t_ns, R);
    const double wdot = st.rot.kind ? st.rot.wdot : 0.0;
    double vf[3] = { -(wdot * st.pos[1]), wdot * st.pos[0], 0.0 };
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        r[i] = (R[i] * st.pos[0] + R[3 + i] * st.pos[1]) + R[6 + i] * st.pos[2];
        v[i] = (R[i] * vf[0] + R[3 + i] * vf[1]) + R[6 + i] * vf[2];
        up[i] = (R[i] * st.up[0] + R[3 + i] * st.up[1]) + R[6 + i] * st.up[2];
        if constexpr (St::NS == 4) {
            ne[0][i] = (R[i] * st.north[0] + R[3 + i] * st.north[1]) + R[6 + i] * st.north[2];
            ne[1][i] = (R[i] * st.east[0] + R[3 + i] * st.east[1]) + R[6 + i] * st.east[2];
        }
    }
    if (st.body != NYXB_CENTRAL_BODY) {
        double bp[3], bv[3];
        if (!body_position(S.bodies[st.body], t_ns, bp) || !body_velocity(S.bodies[st.body], t_ns, bv)) return false;
#pragma unroll
        for (int i = 0; i < 3; ++i) { r[i] += bp[i]; v[i] += bv[i]; }
    }
    return true;
}

// ------------------------------------------------------------------------- one residual window of a measurement
// What od/process/mod.rs:270-352 prepares before `measurement_update`: the window's measurement types, the real observation,
// the tracker geometry (range, range rate, elevation mask, line-of-sight obstruction), `h_tilde` (msr/sensitivity.rs:88-239:
// identity rows unless the type is in msr.data; the observed range / Doppler in the denominators, as coded), the measurement
// noise and the computed observation minus the device bias.  Shared by the per-thread and the warp-cooperative filter kernels.
// SUB_BIAS = false leaves the bias in: the batch least-squares estimator compares with measure_instantaneous(state, None), which
// has no noise and no bias (blse/mod.rs:248-249).
// NS: observation slots of the tracker kind (2 for the ground station, 3 for position fixes, 4 for a station with angles)
template <int NS>
struct OdWindowT {
    int ncur;
    int cur[NS];
    bool avail[NS];
    double real_obs[NS], Rk[NS], comp[NS];
    double H[NS][9];
};
using OdWindow = OdWindowT<2>;
// OD_WIN_TX_NO_DATA and OD_WIN_NO_RANGE: interlink windows only (od_link_window_setup)
enum { OD_WIN_OK = 0, OD_WIN_EMPTY = 1, OD_WIN_UNAVAILABLE = 2, OD_WIN_NOT_VISIBLE = 3, OD_WIN_EPHEMERIS = 4, OD_WIN_TX_NO_DATA = 5,
       OD_WIN_NO_RANGE = 6 };

// St: DevStation (range, Doppler) or DevAerStation, which adds azimuth and elevation (trk_device.rs:158-208, msr/types.rs:102-117,
// sensitivity.rs:188-226).  The observation slot of a type is its value.  The angles, in degrees, come from rho = r_sc - r_station in
// the integration frame: elevation asin(rho.up / |rho|), the very value the mask test reads; azimuth atan2(rho.E, rho.N) mapped into
// [0, 360) (anise's atan2(rho_SEZ.y, -rho_SEZ.x) and between_0_360), with E and N the geodetic east and north.  Their h_tilde rows are
// the reference's as coded: in rad/km, from the integration-frame rho, with r^2 = |rho|^2 formed as (sqrt(sum))^2.
template <bool SUB_BIAS = true, class St>
__device__ static int od_window_setup(const DevSetup& S, const St& gs, int M, int wno, const double o[St::NS], long long t_k,
                                      const double y[9], OdWindowT<St::NS>& w) {
    constexpr int NS = St::NS;
    w.ncur = 0;
    for (int q = wno * M; q < (wno + 1) * M && q < gs.n_types; ++q) w.cur[w.ncur++] = gs.types[q];
    if (w.ncur == 0) return OD_WIN_EMPTY;
    bool any = false;
#pragma unroll
    for (int q = 0; q < NS; ++q) w.avail[q] = false;
    for (int q = 0; q < w.ncur; ++q) { w.avail[q] = (o[w.cur[q]] == o[w.cur[q]]); any = any || w.avail[q]; }
    if (!any) return OD_WIN_UNAVAILABLE;
#pragma unroll
    for (int q = 0; q < NS; ++q) w.real_obs[q] = 0.0;
    for (int q = 0; q < w.ncur; ++q) if (w.avail[q]) w.real_obs[q] = o[w.cur[q]];
    double r_tx[3], v_tx[3], up[3], ne[2][3];
    if (!station_state(S, gs, t_k, r_tx, v_tx, up, ne)) return OD_WIN_EPHEMERIS;
    const double dr[3] = { y[0] - r_tx[0], y[1] - r_tx[1], y[2] - r_tx[2] };
    const double dv[3] = { y[3] - v_tx[0], y[4] - v_tx[1], y[5] - v_tx[2] };
    const double rng = sqrt((dr[0] * dr[0] + dr[1] * dr[1]) + dr[2] * dr[2]);
    const double rr = ((dr[0] * dv[0] + dr[1] * dv[1]) + dr[2] * dv[2]) / rng;
    const double elev = asin(((dr[0] * up[0] + dr[1] * up[1]) + dr[2] * up[2]) / rng) * (180.0 / 3.14159265358979323846);
    bool visible = !(elev - gs.mask_deg < 0.0);
    if (visible && gs.body != NYXB_CENTRAL_BODY && gs.body_radius > 0.0) {   // Vallado SIGHT (anise line_of_sight_obstructed)
        double r1sq = (y[0] * y[0] + y[1] * y[1]) + y[2] * y[2];
        double r2sq = (r_tx[0] * r_tx[0] + r_tx[1] * r_tx[1]) + r_tx[2] * r_tx[2];
        double r12 = (y[0] * r_tx[0] + y[1] * r_tx[1]) + y[2] * r_tx[2];
        double tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12);
        if (tau >= 0.0 && tau <= 1.0 && (1.0 - tau) * r1sq + r12 * tau <= gs.body_radius * gs.body_radius) visible = false;
    }
    if (!visible) return OD_WIN_NOT_VISIBLE;   // device.measure() -> None (process/mod.rs:386-392)
#pragma unroll
    for (int q = 0; q < NS; ++q)
#pragma unroll
        for (int c = 0; c < 9; ++c) w.H[q][c] = (q == c) ? 1.0 : 0.0;
#pragma unroll
    for (int q = 0; q < NS; ++q) { w.Rk[q] = 0.0; w.comp[q] = 0.0; }
    for (int q = 0; q < w.ncur; ++q) {
        const int slot = wno * M + q;  // position of the type in the device's list
        const int t = w.cur[q];
        w.Rk[q] = gs.noise_var[slot];
        w.comp[q] = ((t == NYXB_MSR_RANGE) ? rng : rr);
        if constexpr (NS == 4) {
            if (t == NYXB_MSR_ELEVATION) w.comp[q] = elev;
            if (t == NYXB_MSR_AZIMUTH) {
                const double rn = (dr[0] * ne[0][0] + dr[1] * ne[0][1]) + dr[2] * ne[0][2];
                const double re = (dr[0] * ne[1][0] + dr[1] * ne[1][1]) + dr[2] * ne[1][2];
                double az = fmod(atan2(re, rn) * (180.0 / 3.14159265358979323846), 360.0);
                if (az < 0.0) az += 360.0;
                w.comp[q] = az;
            }
        }
        if (SUB_BIAS) w.comp[q] -= gs.bias[slot];
        if (!w.avail[q]) continue;
        if (t == NYXB_MSR_DOPPLER) {
            const double rho = rng, rho_dot = o[NYXB_MSR_DOPPLER], rho2 = rho * rho;
            w.H[q][0] = dv[0] / rho - rho_dot * dr[0] / rho2;
            w.H[q][1] = dv[1] / rho - rho_dot * dr[1] / rho2;
            w.H[q][2] = dv[2] / rho - rho_dot * dr[2] / rho2;
            w.H[q][3] = dr[0] / rho; w.H[q][4] = dr[1] / rho; w.H[q][5] = dr[2] / rho;
            w.H[q][6] = 0.0; w.H[q][7] = 0.0; w.H[q][8] = 0.0;
        } else if (NS == 4 && (t == NYXB_MSR_AZIMUTH || t == NYXB_MSR_ELEVATION)) {
            const double xy2 = dr[0] * dr[0] + dr[1] * dr[1];
            for (int c = 0; c < 9; ++c) w.H[q][c] = 0.0;
            if (t == NYXB_MSR_AZIMUTH) {
                w.H[q][0] = -dr[1] / xy2;
                w.H[q][1] = dr[0] / xy2;
            } else {
                const double nrm = sqrt(xy2 + dr[2] * dr[2]), r2 = nrm * nrm, z2 = dr[2] * dr[2];
                w.H[q][0] = -(dr[0] * dr[2]) / (r2 * sqrt(r2 - z2));
                w.H[q][1] = -(dr[1] * dr[2]) / (r2 * sqrt(r2 - z2));
                w.H[q][2] = sqrt(xy2) / r2;
            }
        } else {
            const double rho = o[NYXB_MSR_RANGE];
            w.H[q][0] = dr[0] / rho; w.H[q][1] = dr[1] / rho; w.H[q][2] = dr[2] / rho;
            for (int c = 3; c < 9; ++c) w.H[q][c] = 0.0;
        }
    }
    return OD_WIN_OK;
}

// Innovation statistics (filtering.rs:152-167): S = H P H^T + R (given), Cholesky of S (fallback: of R), whitened residual ratio.
// Returns false on SingularNoiseRk.
__device__ static bool od_ratio(int M, const double Sk[2][2], const double Rk[2], const double pre[2], double& ratio) {
    double L00 = 1.0, L10 = 0.0, L11 = 1.0;
    bool chol_ok = Sk[0][0] > 0.0;
    if (chol_ok) {
        L00 = sqrt(Sk[0][0]);
        if (M == 2) {
            L10 = Sk[1][0] / L00;
            const double d = Sk[1][1] - L10 * L10;
            if (d > 0.0) L11 = sqrt(d); else chol_ok = false;
        }
    }
    double W00 = L00, W10 = L10, W11 = L11;
    if (!chol_ok) {
        if (!(Rk[0] > 0.0) || (M == 2 && !(Rk[1] > 0.0))) return false;
        W00 = sqrt(Rk[0]); W10 = 0.0; W11 = (M == 2) ? sqrt(Rk[1]) : 1.0;
    }
    const double w0 = pre[0] / W00, w1 = (M == 2) ? (pre[1] - W10 * w0) / W11 : 0.0;
    ratio = sqrt(((M == 2) ? (w0 * w0 + w1 * w1) : (w0 * w0)) / (double)M);
    return true;
}

// S^-1 for M = 1, 2 (the gain K = P H^T S^-1, filtering.rs:206-231); false on SingularKalmanGain
__device__ static bool od_sinv(int M, const double Sk[2][2], double Si[2][2]) {
    if (M == 1) { Si[0][0] = 1.0 / Sk[0][0]; Si[0][1] = Si[1][0] = 0.0; Si[1][1] = 0.0; return true; }
    const double det = Sk[0][0] * Sk[1][1] - Sk[0][1] * Sk[1][0];
    if (det == 0.0 || det != det) return false;
    Si[0][0] = Sk[1][1] / det; Si[0][1] = -Sk[0][1] / det; Si[1][0] = -Sk[1][0] / det; Si[1][1] = Sk[0][0] / det;
    return true;
}

// ------------------------------------------------------------------------- tracker kinds of the filter loop (od_process_arc's TRK)
// TRK::NS      observation slots per measurement: obs, ratio, prefit and postfit are [m][NS][n], and slot wno*M + q is the position of
//              the window's type in the device's list (the ratio takes slot ratio_slot(M, wno));
// TRK::Dev     the device struct of DevOdT;
// absent(o)    no type of the measurement is in this filter's arc;
// setup(..)    the window (od_window_setup's contract) at the measurement epoch t_k, which is the nominal state's; the propagator's
//              epoch before it was set to t_k (within epoch_precision of it) comes next, for the interlink's computed observation;
// ratio(..)    residual ratio of filtering.rs:152-167, false on SingularNoiseRk;
// gain_setup / gain_entry   K = P H^T S^-1 (filtering.rs:206-231): gain_setup factors S (false on SingularKalmanGain), gain_entry gives
//              entry q of row r of K from row r of P H^T;
// ratio_slot   the ratio's slot of window wno;
// tag(..)      the estimate record's tag, and tag_msr / tag_window its measurement index and window.
struct GroundTrk {
    using Dev = DevStation;
    static constexpr int NS = Dev::NS;
    using Win = OdWindow;
    struct Gain { double Si[2][2]; };
    __device__ __forceinline__ static bool absent(const double o[2]) { return o[0] != o[0] && o[1] != o[1]; }
    __device__ __forceinline__ static int setup(const DevSetup& S, const Dev& gs, int M, int wno, const double o[2], long long t_k, long long,
                                const double y[9], Win& w) {
        return od_window_setup(S, gs, M, wno, o, t_k, y, w);
    }
    __device__ __forceinline__ static bool ratio(int M, const double Sk[2][2], const double Rk[2], const double pre[2], double& r) {
        return od_ratio(M, Sk, Rk, pre, r);
    }
    __device__ __forceinline__ static bool gain_setup(int M, const double Sk[2][2], Gain& g) { return od_sinv(M, Sk, g.Si); }
    __device__ __forceinline__ static double gain_entry(int M, const Gain& g, const double* pht, int q) {
        double s = 0.0;
        if (q < M)
            for (int bb = 0; bb < M; ++bb) s += pht[bb] * g.Si[bb][q];
        return s;
    }
    __device__ __forceinline__ static int ratio_slot(int M, int wno) { return (M == 1) ? wno : 0; }
    __device__ __forceinline__ static long long tag(long long k, int wno, int rej, int M) { return ((k * 2 + wno) * 2 + rej) * 2 + (M - 1); }
    __device__ __forceinline__ static long long tag_msr(long long tg) { return tg >> 3; }
    __device__ __forceinline__ static int tag_window(long long tg) { return (int)((tg >> 2) & 1); }
};

// PositionDevice (od/position): the type at list position ii measures component ii of the nominal position (trk_device.rs:76-83, the
// list position, not the type), while h_tilde puts its unit row at the TYPE's component X -> 0, Y -> 1, Z -> 2 (sensitivity.rs:55-75)
// and starts from zeros (sensitivity.rs:32): a window slot without a type, or whose type is absent, keeps a zero row, R keeps the
// type's variance (trackdata.rs:84-102) and the real observation is 0 (measurement.rs:84-96).  The computed observation is
// measure()'s ((r_ii + 0) + bias) minus the bias vector (process/mod.rs:324-333): the bias cancels.  No visibility test.
__device__ static int od_pos_window_setup(const DevPosDevice& d, int M, int wno, const double o[3], const double y[9], OdWindowT<3>& w) {
    w.ncur = 0;
    for (int q = wno * M; q < (wno + 1) * M && q < d.n_types; ++q) w.cur[w.ncur++] = d.types[q];
    if (w.ncur == 0) return OD_WIN_EMPTY;
    bool any = false;
    for (int q = 0; q < 3; ++q) w.avail[q] = false;
    for (int q = 0; q < w.ncur; ++q) { const double v = o[w.cur[q] - NYXB_MSR_X]; w.avail[q] = (v == v); any = any || w.avail[q]; }
    if (!any) return OD_WIN_UNAVAILABLE;
    for (int q = 0; q < 3; ++q) {
        w.real_obs[q] = 0.0; w.Rk[q] = 0.0; w.comp[q] = 0.0;
        for (int c = 0; c < 9; ++c) w.H[q][c] = 0.0;
    }
    for (int q = 0; q < w.ncur; ++q) {
        const int slot = wno * M + q;
        w.Rk[q] = d.noise_var[slot];
        w.comp[q] = ((y[slot] + 0.0) + d.bias[slot]) - d.bias[slot];
        if (!w.avail[q]) continue;
        w.real_obs[q] = o[w.cur[q] - NYXB_MSR_X];
        w.H[q][w.cur[q] - NYXB_MSR_X] = 1.0;
    }
    return OD_WIN_OK;
}

// Lower Cholesky factor of a symmetric 3x3 S, column by column; false when a pivot is not positive.
__device__ static bool od_chol3(const double A[3][3], double L[3][3]) {
    L[0][1] = L[0][2] = L[1][2] = 0.0;
    if (!(A[0][0] > 0.0)) return false;
    L[0][0] = sqrt(A[0][0]);
    L[1][0] = A[1][0] / L[0][0];
    L[2][0] = A[2][0] / L[0][0];
    const double d1 = A[1][1] - L[1][0] * L[1][0];
    if (!(d1 > 0.0)) return false;
    L[1][1] = sqrt(d1);
    L[2][1] = (A[2][1] - L[2][0] * L[1][0]) / L[1][1];
    const double d2 = (A[2][2] - L[2][0] * L[2][0]) - L[2][1] * L[2][1];
    if (!(d2 > 0.0)) return false;
    L[2][2] = sqrt(d2);
    return true;
}

// y = L^-1 b (forward substitution, column-oriented as nalgebra's solve_lower_triangular)
__device__ __forceinline__ void od_fwd3(const double L[3][3], const double b[3], double y[3]) {
    double t1 = b[1], t2 = b[2];
    y[0] = b[0] / L[0][0];
    t1 = t1 - y[0] * L[1][0]; t2 = t2 - y[0] * L[2][0];
    y[1] = t1 / L[1][1];
    t2 = t2 - y[1] * L[2][1];
    y[2] = t2 / L[2][2];
}

struct PosTrk {
    using Dev = DevPosDevice;
    static constexpr int NS = Dev::NS;
    using Win = OdWindowT<3>;
    // chol: S = L L^T (M = 3), else Si: S^-1 (M <= 2: od_sinv, M = 3: the closed-form 3x3 inverse after a failed Cholesky)
    struct Gain { bool chol; double L[3][3]; double Si[3][3]; };
    __device__ __forceinline__ static bool absent(const double o[3]) { return o[0] != o[0] && o[1] != o[1] && o[2] != o[2]; }
    __device__ __forceinline__ static int setup(const DevSetup&, const Dev& d, int M, int wno, const double o[3], long long, long long,
                                const double y[9], Win& w) {
        return od_pos_window_setup(d, M, wno, o, y, w);
    }
    // M <= 2: od_ratio on the leading 2x2 block, the ground station's arithmetic
    __device__ __forceinline__ static bool ratio(int M, const double Sk[3][3], const double Rk[3], const double pre[3], double& r) {
        if (M < 3) {
            const double S2[2][2] = { { Sk[0][0], Sk[0][1] }, { Sk[1][0], Sk[1][1] } };
            const double R2[2] = { Rk[0], Rk[1] }, p2[2] = { pre[0], pre[1] };
            return od_ratio(M, S2, R2, p2, r);
        }
        double L[3][3];
        if (!od_chol3(Sk, L)) {                                   // fall back to the Cholesky factor of the diagonal R
            if (!(Rk[0] > 0.0) || !(Rk[1] > 0.0) || !(Rk[2] > 0.0)) return false;
            for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) L[a][c] = 0.0;
            L[0][0] = sqrt(Rk[0]); L[1][1] = sqrt(Rk[1]); L[2][2] = sqrt(Rk[2]);
        }
        double w[3];
        od_fwd3(L, pre, w);
        r = sqrt(((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]) / 3.0);
        return true;
    }
    __device__ __forceinline__ static bool gain_setup(int M, const double Sk[3][3], Gain& g) {
        g.chol = false;
        if (M < 3) {
            const double S2[2][2] = { { Sk[0][0], Sk[0][1] }, { Sk[1][0], Sk[1][1] } };
            double Si[2][2];
            if (!od_sinv(M, S2, Si)) return false;
            for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) g.Si[a][c] = (a < 2 && c < 2) ? Si[a][c] : 0.0;
            return true;
        }
        if (od_chol3(Sk, g.L)) { g.chol = true; return true; }
        // try_inverse: the closed-form inverse (cofactors over the determinant); not pinned to nalgebra's
        const double m11 = Sk[0][0], m12 = Sk[0][1], m13 = Sk[0][2], m21 = Sk[1][0], m22 = Sk[1][1], m23 = Sk[1][2];
        const double m31 = Sk[2][0], m32 = Sk[2][1], m33 = Sk[2][2];
        const double c11 = m22 * m33 - m32 * m23, c12 = m21 * m33 - m31 * m23, c13 = m21 * m32 - m31 * m22;
        const double det = (m11 * c11 - m12 * c12) + m13 * c13;
        if (det == 0.0 || det != det) return false;
        g.Si[0][0] = c11 / det;
        g.Si[0][1] = (m13 * m32 - m33 * m12) / det;
        g.Si[0][2] = (m12 * m23 - m22 * m13) / det;
        g.Si[1][0] = -c12 / det;
        g.Si[1][1] = (m11 * m33 - m31 * m13) / det;
        g.Si[1][2] = (m13 * m21 - m23 * m11) / det;
        g.Si[2][0] = c13 / det;
        g.Si[2][1] = (m12 * m31 - m32 * m11) / det;
        g.Si[2][2] = (m11 * m22 - m21 * m12) / det;
        return true;
    }
    // Cholesky solve S k = (row r of P H^T): forward, then back substitution with L^T
    __device__ __forceinline__ static double gain_entry(int M, const Gain& g, const double* pht, int q) {
        if (g.chol) {
            const double b[3] = { pht[0], pht[1], pht[2] };
            double y[3], x[3];
            od_fwd3(g.L, b, y);
            x[2] = y[2] / g.L[2][2];
            x[1] = (y[1] - g.L[2][1] * x[2]) / g.L[1][1];
            x[0] = (y[0] - (g.L[1][0] * x[1] + g.L[2][0] * x[2])) / g.L[0][0];
            return x[q];
        }
        double s = 0.0;
        if (q < M)
            for (int bb = 0; bb < M; ++bb) s += pht[bb] * g.Si[bb][q];
        return s;
    }
    __device__ __forceinline__ static int ratio_slot(int M, int wno) { return (M == 1) ? wno : 0; }
    __device__ __forceinline__ static long long tag(long long k, int wno, int rej, int M) { return ((k * 4 + wno) * 2 + rej) * 4 + (M - 1); }
    __device__ __forceinline__ static long long tag_msr(long long tg) { return tg >> 5; }
    __device__ __forceinline__ static int tag_window(long long tg) { return (int)((tg >> 3) & 3); }
};

// A ground station with angles (DevAerStation): the window of od_window_setup over four slots, msr_size 1 or 2.  Ratio and gain are the
// ground station's (od_ratio, od_sinv) on the leading 2x2 block.  The ratio takes slot wno: four types at msr_size 2 make two windows.
// Record tags use the position filter's layout (window 0..3).
struct AerTrk {
    using Dev = DevAerStation;
    static constexpr int NS = Dev::NS;
    using Win = OdWindowT<4>;
    using Gain = GroundTrk::Gain;
    __device__ __forceinline__ static bool absent(const double o[4]) { return o[0] != o[0] && o[1] != o[1] && o[2] != o[2] && o[3] != o[3]; }
    __device__ __forceinline__ static int setup(const DevSetup& S, const Dev& gs, int M, int wno, const double o[4], long long t_k, long long,
                                const double y[9], Win& w) {
        return od_window_setup(S, gs, M, wno, o, t_k, y, w);
    }
    __device__ __forceinline__ static bool ratio(int M, const double Sk[4][4], const double Rk[4], const double pre[4], double& r) {
        const double S2[2][2] = { { Sk[0][0], Sk[0][1] }, { Sk[1][0], Sk[1][1] } };
        const double R2[2] = { Rk[0], Rk[1] }, p2[2] = { pre[0], pre[1] };
        return od_ratio(M, S2, R2, p2, r);
    }
    __device__ __forceinline__ static bool gain_setup(int M, const double Sk[4][4], Gain& g) {
        const double S2[2][2] = { { Sk[0][0], Sk[0][1] }, { Sk[1][0], Sk[1][1] } };
        return od_sinv(M, S2, g.Si);
    }
    __device__ __forceinline__ static double gain_entry(int M, const Gain& g, const double* pht, int q) { return GroundTrk::gain_entry(M, g, pht, q); }
    __device__ __forceinline__ static int ratio_slot(int, int wno) { return wno; }
    __device__ __forceinline__ static long long tag(long long k, int wno, int rej, int M) { return PosTrk::tag(k, wno, rej, M); }
    __device__ __forceinline__ static long long tag_msr(long long tg) { return PosTrk::tag_msr(tg); }
    __device__ __forceinline__ static int tag_window(long long tg) { return PosTrk::tag_window(tg); }
};

// An interlink transmitter (DevLink; interlink/trk_device.rs:180-232, interlink/sensitivity.rs:50-172, process/mod.rs:300-330), as
// coded.  h_tilde runs first, with the transmitter at the nominal state's epoch t_nom: dr = r_rx - r_tx, dv = v_rx - v_tx, and the
// OBSERVED range and Doppler in the rows; identity rows for types absent from the measurement, OD_WIN_NO_RANGE for a Doppler row without
// an observed range.  Then measure_instantaneous at the propagator's epoch t_prop: the transmitter again, the line of sight against the
// body at the frame's centre (Vallado's SIGHT, the receiver as r1), range |rho| and range rate rho . v_rx / |rho|: the transmitter's
// velocity is not subtracted.  A transmitter epoch outside the recording is OD_WIN_TX_NO_DATA, before any obstruction test.
__device__ static int od_link_window_setup(const DevLink& d, int M, int wno, const double o[2], long long t_nom, long long t_prop,
                                           const double y[9], OdWindow& w) {
    w.ncur = 0;
    for (int q = wno * M; q < (wno + 1) * M && q < d.n_types; ++q) w.cur[w.ncur++] = d.types[q];
    if (w.ncur == 0) return OD_WIN_EMPTY;
    bool any = false;
    w.avail[0] = w.avail[1] = false;
    for (int q = 0; q < w.ncur; ++q) { w.avail[q] = (o[w.cur[q]] == o[w.cur[q]]); any = any || w.avail[q]; }
    if (!any) return OD_WIN_UNAVAILABLE;
    for (int q = 0; q < 2; ++q) {
        w.real_obs[q] = 0.0; w.Rk[q] = 0.0; w.comp[q] = 0.0;
        for (int c = 0; c < 9; ++c) w.H[q][c] = (q == c) ? 1.0 : 0.0;
    }
    for (int q = 0; q < w.ncur; ++q) if (w.avail[q]) w.real_obs[q] = o[w.cur[q]];
    double tx[6];
    if (nyxb_traj_at(d.tx, (size_t)d.tx_n, (size_t)d.col, t_nom, tx)) return OD_WIN_TX_NO_DATA;   // `location(..).unwrap()`
    const double dr[3] = { y[0] - tx[0], y[1] - tx[1], y[2] - tx[2] };
    const double dv[3] = { y[3] - tx[3], y[4] - tx[4], y[5] - tx[5] };
    for (int q = 0; q < w.ncur; ++q) {
        if (!w.avail[q]) continue;
        const double rho = o[NYXB_MSR_RANGE];
        if (w.cur[q] == NYXB_MSR_DOPPLER) {
            if (rho != rho) return OD_WIN_NO_RANGE;
            const double rho_dot = o[NYXB_MSR_DOPPLER], rho2 = rho * rho;
            w.H[q][0] = dv[0] / rho - rho_dot * dr[0] / rho2;
            w.H[q][1] = dv[1] / rho - rho_dot * dr[1] / rho2;
            w.H[q][2] = dv[2] / rho - rho_dot * dr[2] / rho2;
            w.H[q][3] = dr[0] / rho; w.H[q][4] = dr[1] / rho; w.H[q][5] = dr[2] / rho;
        } else {
            w.H[q][0] = dr[0] / rho; w.H[q][1] = dr[1] / rho; w.H[q][2] = dr[2] / rho;
            for (int c = 3; c < 9; ++c) w.H[q][c] = 0.0;
        }
        w.H[q][6] = 0.0; w.H[q][7] = 0.0; w.H[q][8] = 0.0;
    }
    if (nyxb_traj_at(d.tx, (size_t)d.tx_n, (size_t)d.col, t_prop, tx)) return OD_WIN_TX_NO_DATA;  // `self.traj.at(rx.epoch())?`
    if (d.body_radius > 0.0) {                 // r1 = the receiver, r2 = the transmitter: od_window_setup's order for the same test
        const double r1sq = (y[0] * y[0] + y[1] * y[1]) + y[2] * y[2];
        const double r2sq = (tx[0] * tx[0] + tx[1] * tx[1]) + tx[2] * tx[2];
        const double r12 = (y[0] * tx[0] + y[1] * tx[1]) + y[2] * tx[2];
        const double tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12);
        if (tau >= 0.0 && tau <= 1.0 && (1.0 - tau) * r1sq + r12 * tau <= d.body_radius * d.body_radius) return OD_WIN_NOT_VISIBLE;
    }
    const double rho[3] = { y[0] - tx[0], y[1] - tx[1], y[2] - tx[2] };
    const double rng = sqrt((rho[0] * rho[0] + rho[1] * rho[1]) + rho[2] * rho[2]);
    const double rr = ((rho[0] * y[3] + rho[1] * y[4]) + rho[2] * y[5]) / rng;
    for (int q = 0; q < w.ncur; ++q) {
        const int slot = wno * M + q;
        w.Rk[q] = d.noise_var[slot];
        w.comp[q] = ((w.cur[q] == NYXB_MSR_RANGE) ? rng : rr) - d.bias[slot];
    }
    return OD_WIN_OK;
}

// The interlink transmitter: od_link_window_setup, and the ground station's slots, ratio, gain and record tags.
struct LinkTrk {
    using Dev = DevLink;
    static constexpr int NS = Dev::NS;
    using Win = OdWindow;
    using Gain = GroundTrk::Gain;
    __device__ __forceinline__ static bool absent(const double o[2]) { return GroundTrk::absent(o); }
    __device__ __forceinline__ static int setup(const DevSetup&, const Dev& d, int M, int wno, const double o[2], long long t_k, long long t_prop,
                                const double y[9], Win& w) {
        return od_link_window_setup(d, M, wno, o, t_k, t_prop, y, w);
    }
    __device__ __forceinline__ static bool ratio(int M, const double Sk[2][2], const double Rk[2], const double pre[2], double& r) {
        return od_ratio(M, Sk, Rk, pre, r);
    }
    __device__ __forceinline__ static bool gain_setup(int M, const double Sk[2][2], Gain& g) { return od_sinv(M, Sk, g.Si); }
    __device__ __forceinline__ static double gain_entry(int M, const Gain& g, const double* pht, int q) { return GroundTrk::gain_entry(M, g, pht, q); }
    __device__ __forceinline__ static int ratio_slot(int M, int wno) { return GroundTrk::ratio_slot(M, wno); }
    __device__ __forceinline__ static long long tag(long long k, int wno, int rej, int M) { return GroundTrk::tag(k, wno, rej, M); }
    __device__ __forceinline__ static long long tag_msr(long long tg) { return GroundTrk::tag_msr(tg); }
    __device__ __forceinline__ static int tag_window(long long tg) { return GroundTrk::tag_window(tg); }
};
