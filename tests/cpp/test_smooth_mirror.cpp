// C++ host-mirror test of the smoother: KalmanODProcess::process_arcs with estimate records and ODSolution::smooth through
// nyxb.hpp -> C ABI -> CUDA kernels.  Noise-free range + Doppler from a truth propagated with the same dynamics and step; a CKF started
// on the truth then has zero deviations, and so has every smoothed estimate (od_tb_val_ckf_fixed_step_perfect_stations in small).
#include <cmath>
#include <cstdio>

#include "nyxb.hpp"

using namespace nyxb;
static int failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++failures; } } while (0)

int main() {
    const Frame eme2k = EARTH_J2000();
    const Spacecraft truth = Spacecraft::cartesian(-2436.45, -2436.45, 6891.037, 5.088611, -5.088611, 0.0, 0, eme2k);
    const auto dynamics = SpacecraftDynamics::new_(OrbitalDynamics::two_body());
    auto setup = Propagator::rk89(dynamics, IntegratorOptions::with_fixed_step_s(10.0));
    GroundStation gs = GroundStation::dss65_madrid(-90.0, StochasticNoise{1e-6, 0.0}, StochasticNoise{1e-6, 0.0});
    gs.frame = eme2k;   // fixed in the integration frame: range and range rate are plain geometry
    double p[3], up[3];
    gs.body_fixed(p, up);
    const size_t n = 2;
    TrackingDataArc arc; arc.n = n;
    for (int k = 1; k <= 12; ++k) {
        const int64_t t = k * 30 * NS_PER_S;   // 30 s apart, 10 s steps, 60 s max_step: one time update and a window per gap
        const Spacecraft s = setup.with(truth).for_duration(t);
        const double dr[3] = {s.x_km - p[0], s.y_km - p[1], s.z_km - p[2]};
        const double rng = std::sqrt((dr[0] * dr[0] + dr[1] * dr[1]) + dr[2] * dr[2]);
        const double rr = ((dr[0] * s.vx_km_s + dr[1] * s.vy_km_s) + dr[2] * s.vz_km_s) / rng;
        arc.epoch_ns.push_back(t); arc.tracker.push_back(gs.name);
        for (size_t i = 0; i < n; ++i) arc.obs.push_back(rng);
        for (size_t i = 0; i < n; ++i) arc.obs.push_back(rr);
    }
    KalmanODProcess odp(setup, KalmanVariant::DeviationTracking, std::nullopt, {gs});
    const double d[9] = {1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0, 0, 0};
    std::vector<KfEstimate> ests{KfEstimate::from_diag(truth, d), KfEstimate::from_diag(truth, d)};
    const ODSolution plain = odp.process_arcs(ests, arc);
    const ODSolution sol = odp.process_arcs(ests, arc, 64);
    CHECK(sol.state == plain.state && sol.covar == plain.covar && sol.postfit == plain.postfit);
    CHECK(sol.status[0] == 0 && sol.n_estimates(0) == sol.rec_count[0] && sol.rec_count[0] >= 12);
    int meas = 0;
    for (int64_t k = 0; k < sol.n_estimates(0); ++k) meas += sol.rec_tag[(size_t)k * n] >= 0;
    CHECK(meas == 12);
    const ODSolution sm = sol.smooth(odp, arc);
    CHECK(sm.is_smoother_run() && !sol.is_smoother_run());
    for (size_t i = 0; i < n; ++i) {
        CHECK(sm.sm_status[i] == 0);
        const int64_t L = sm.n_estimates(i);
        double worst = 0.0;
        for (int64_t k = 0; k < L; ++k)
            for (int r = 0; r < 9; ++r) worst = std::fmax(worst, std::fabs(sm.sm_deviation[((size_t)k * 9 + r) * n + i]));
        CHECK(worst < 1e-9);
        // the last estimate is copied unchanged, without a ratio
        const size_t l = (size_t)(L - 1);
        for (int e = 0; e < 81; ++e) CHECK(sm.sm_covar[(l * 81 + e) * n + i] == sol.rec_covar[(l * 81 + e) * n + i]);
        CHECK(std::isnan(sm.sm_fs_ratio[(l * 9) * n + i]));
        CHECK(std::fabs(sm.sm_state[(l * 9) * n + i] - (sol.rec_nominal[(l * 9) * n + i] + sol.rec_deviation[(l * 9) * n + i])) == 0.0);
    }
    // the two filters are the same problem: the same bits
    for (size_t q = 0; q < sm.sm_covar.size(); q += n) CHECK(std::isnan(sm.sm_covar[q]) ? std::isnan(sm.sm_covar[q + 1]) : sm.sm_covar[q] == sm.sm_covar[q + 1]);
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
