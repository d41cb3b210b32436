// C++ host-mirror test of the covariance mapping: KalmanODProcess::predict_until / predict_for through nyxb.hpp -> C ABI ->
// CUDA kernels.
#include <cmath>
#include <cstdio>

#include "nyxb.hpp"

using namespace nyxb;
static int failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++failures; } } while (0)

int main() {
    const Frame eme2k = EARTH_J2000();
    const Spacecraft init = Spacecraft::cartesian(-2436.45, -2436.45, 6891.037, 5.088611, -5.088611, 0.0, 0, eme2k);
    const auto dynamics = SpacecraftDynamics::new_(OrbitalDynamics::two_body());
    auto setup = Propagator::rk89(dynamics, IntegratorOptions::with_fixed_step_s(10.0));
    const double p0[9] = {1.0, 1.0, 1.0, 1e-6, 1e-6, 1e-6, 0.0, 0.0, 0.0};
    KfEstimate est = KfEstimate::from_diag(init, p0);
    est.state_deviation[0] = 0.1;
    est.state_deviation[4] = -1e-4;

    {   // CKF, no process noise: 10 min 30 s in chunks of 1 min -> 12 records, the last one 30 s past the end
        KalmanODProcess odp(setup, KalmanVariant::DeviationTracking, std::nullopt, {});
        auto sol = odp.predict_for(est, 630 * NS_PER_S);
        CHECK(sol.status == 0);
        CHECK(sol.count == 12);
        CHECK(sol.epoch == 660 * NS_PER_S && sol.record_epoch(sol.count - 1) == sol.epoch);
        CHECK(sol.rec_state[0] == init.x_km + 0.1 && sol.rec_state[4] == init.vy_km_s - 1e-4);   // record 0 = the initial estimate
        CHECK(sol.record_covar(0, 0, 0) == 1.0 && sol.record_covar(0, 3, 3) == 1e-6);
        double asym = 0.0;
        for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) asym = std::fmax(asym, std::fabs(sol.covar[c * 9 + r] - sol.covar[r * 9 + c]));
        CHECK(asym <= 1e-9 * sol.covar[0]);
        CHECK(sol.covar[0] + sol.covar[10] + sol.covar[20] > 3.0);   // position uncertainty grows along the orbit
        // the nominal state follows the plain propagation of the same steps
        auto fin = setup.with(init).for_duration(660 * NS_PER_S);
        CHECK(std::fabs(fin.x_km - sol.state[0]) < 1e-9 && std::fabs(fin.y_km - sol.state[1]) < 1e-9 && std::fabs(fin.z_km - sol.state[2]) < 1e-9);
        // CKF: the last record is nominal + deviation, the deviation mapped by the STM (non-zero, not the initial one)
        CHECK(std::fabs(sol.rec_state[(size_t)(sol.count - 1) * 9] - (sol.state[0] + sol.state_dev[0])) < 1e-12);
        CHECK(sol.state_dev[0] != 0.1 && sol.state_dev[0] != 0.0);
    }
    {   // EKF with RIC process noise; an end before the start still runs one chunk
        KalmanODProcess odp(setup, KalmanVariant::ReferenceUpdate, std::nullopt, {});
        const double q[3] = {1e-12, 1e-12, 1e-12};
        odp.with_process_noise(ProcessNoise3D::from_diagonal(q, 600 * NS_PER_S, true));
        auto sol = odp.predict_until(est, -NS_PER_S);
        CHECK(sol.status == 0 && sol.count == 2 && sol.epoch == 60 * NS_PER_S);
        for (int r = 0; r < 9; ++r) CHECK(sol.state_dev[r] == 0.0);
        CHECK(sol.rec_state[9] == sol.state[0]);
    }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
