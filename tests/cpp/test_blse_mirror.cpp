// C++ host-mirror test of the batch least-squares estimator: BatchLeastSquares::estimate / evaluate through nyxb.hpp -> C ABI ->
// CUDA kernels.  Noise-free range + Doppler from a truth propagated with the same dynamics, then a guess dispersed by 50 m / 5 cm/s.
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
    // Madrid's coordinates on a non-rotating Earth (frame = EME2000): the station is fixed in the integration frame, so range and
    // range rate are plain geometry; a -90 deg mask keeps every pass visible
    GroundStation gs = GroundStation::dss65_madrid(-90.0, StochasticNoise{1e-2, 0.0}, StochasticNoise{1e-5, 0.0});
    gs.frame = eme2k;
    double p[3], up[3];
    gs.body_fixed(p, up);
    TrackingDataArc arc; arc.n = 1;
    for (int k = 1; k <= 8; ++k) {
        const int64_t t = k * 10 * NS_PER_S;
        const Spacecraft s = setup.with(truth).for_duration(t);
        const double dr[3] = {s.x_km - p[0], s.y_km - p[1], s.z_km - p[2]};
        const double rng = std::sqrt((dr[0] * dr[0] + dr[1] * dr[1]) + dr[2] * dr[2]);
        const double rr = ((dr[0] * s.vx_km_s + dr[1] * s.vy_km_s) + dr[2] * s.vz_km_s) / rng;
        arc.epoch_ns.push_back(t); arc.tracker.push_back(gs.name); arc.obs.push_back(rng); arc.obs.push_back(rr);
    }
    BatchLeastSquares b(setup, {gs});
    CHECK(b.max_step == 30 * NS_PER_S && b.max_iterations == 10 && b.tolerance_pos_km == 1e-4 && b.lm_lambda_init == 10.0);
    {   // the truth: residuals at the integration error only, and the estimate does not move far
        const double rms = b.evaluate(truth, arc);
        CHECK(rms < 1e-3);
        auto sol = b.estimate(truth, arc);
        CHECK(sol.estimated_state.epoch() == truth.epoch());
        CHECK(std::fabs(sol.estimated_state.x_km - truth.x_km) < 1e-3);
    }
    {   // a dispersed guess: LM lowers the RMS of its final state below the guess's
        Spacecraft g = truth; g.x_km += 0.05; g.vy_km_s += 5e-5;
        b.solver = BLSSolver::LevenbergMarquardt; b.max_iterations = 3;
        auto sol = b.estimate(g, arc);
        CHECK(sol.num_iterations == 3 && sol.final_rms < b.evaluate(g, arc));
        CHECK(b.evaluate(sol.estimated_state, arc) < b.evaluate(g, arc));
        const KfEstimate kf = sol.to_kf_estimate();
        CHECK(kf.covar[60] == 0.0 && kf.covar[70] == 0.0 && kf.covar[80] == 0.0 && kf.covar[0] == sol.covariance[0]);
    }
    {   // one measurement: TooFewMeasurements for estimate, a value for evaluate
        TrackingDataArc one = arc; one.epoch_ns.resize(1); one.tracker.resize(1); one.obs.resize(2);
        bool threw = false;
        try { b.estimate(truth, one); } catch (const std::runtime_error& e) { threw = std::string(e.what()) == "TooFewMeasurements"; }
        CHECK(threw);
        CHECK(b.evaluate(truth, one) >= 0.0);
    }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
