// C++ host-mirror test of the position-fix filter: PositionKalmanODProcess::process_arcs (with and without estimate records) and
// ODSolution::smooth through nyxb.hpp -> C ABI -> CUDA kernels.  Noise-free X / Y / Z fixes from a truth propagated with the same
// dynamics and step; a CKF started on the truth then has zero prefits and deviations, and so has every smoothed estimate.
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
    PositionDevice gnss{"GNSS"};
    gnss.with_noise(MeasurementType::X, StochasticNoise{1e-6, 0.0}).with_noise(MeasurementType::Y, StochasticNoise{1e-6, 0.0})
        .with_noise(MeasurementType::Z, StochasticNoise{1e-6, 0.0});
    const size_t n = 2;
    TrackingDataArc arc; arc.n = n; arc.ns = 3;
    for (int k = 1; k <= 12; ++k) {
        const int64_t t = k * 30 * NS_PER_S;
        const Spacecraft s = setup.with(truth).for_duration(t);
        arc.epoch_ns.push_back(t); arc.tracker.push_back(gnss.name);
        const double xyz[3] = {s.x_km, s.y_km, s.z_km};
        for (int q = 0; q < 3; ++q) for (size_t i = 0; i < n; ++i) arc.obs.push_back(xyz[q]);
    }
    for (int32_t msr : {3, 1}) {
        PositionKalmanODProcess odp(setup, KalmanVariant::DeviationTracking, std::nullopt, {gnss}, msr);
        const double d[9] = {1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0, 0, 0};
        std::vector<KfEstimate> ests{KfEstimate::from_diag(truth, d), KfEstimate::from_diag(truth, d)};
        const ODSolution plain = odp.process_arcs(ests, arc);
        const ODSolution sol = odp.process_arcs(ests, arc, 128);
        CHECK(sol.ns == 3 && sol.prefit.size() == 12 * 3 * n);
        CHECK(sol.state == plain.state && sol.covar == plain.covar && sol.postfit == plain.postfit);
        CHECK(sol.status[0] == 0 && sol.status[1] == 0 && sol.n_estimates(0) == sol.rec_count[0]);
        int meas = 0;
        for (int64_t k = 0; k < sol.n_estimates(0); ++k) {
            const int64_t tg = sol.rec_tag[(size_t)k * n];
            if (tg < 0) continue;
            ++meas;
            CHECK(NYXB_OD_POS_TAG_MSR_SIZE(tg) == msr && NYXB_OD_POS_TAG_WINDOW(tg) < 3 / msr);
        }
        CHECK(meas == 12 * (3 / msr));
        for (size_t e = 0; e < sol.prefit.size(); ++e) CHECK(std::isnan(sol.prefit[e]) || std::fabs(sol.prefit[e]) < 1e-9);
        const ODSolution sm = sol.smooth(odp, arc);
        CHECK(sm.is_smoother_run() && sm.sm_postfit.size() == (size_t)128 * 3 * n);
        for (size_t i = 0; i < n; ++i) {
            CHECK(sm.sm_status[i] == 0);
            double worst = 0.0;
            for (int64_t k = 0; k < sm.n_estimates(i); ++k)
                for (int r = 0; r < 9; ++r) worst = std::fmax(worst, std::fabs(sm.sm_deviation[((size_t)k * 9 + r) * n + i]));
            CHECK(worst < 1e-9);
        }
    }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
