// C++ host-mirror test of interlink tracking: InterlinkKalmanODProcess::process_arcs and ODSolution::smooth, through nyxb.hpp -> C ABI
// (nyxb_od_interlink_batch, nyxb_od_interlink_smooth_batch) -> CUDA kernels.  A transmitter on a Moon-centred NRHO-like orbit, recorded
// with Propagator::propagate_batch_traj, tracks a low lunar orbiter.  The observations are the filter's own computed values: a first CKF
// run from the truth gives obs - prefit = the computed range and Doppler to the last bit; a second run on them has zero prefits and
// deviations, and so has every smoothed estimate.  A Doppler-only device ends with NYXB_ERR_NO_RANGE, a recording that ends inside the
// arc with NYXB_ERR_TX_NO_DATA, and a device with an aberration correction throws.
#include <cmath>
#include <cstdio>

#include "nyxb.hpp"

using namespace nyxb;
static int failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++failures; } } while (0)

int main() {
    Frame moon; moon.ephemeris_id = 301; moon.mu_km3_s2 = 4902.800066163796; moon.mean_equatorial_radius_km = 1737.4;
    const Spacecraft tx0 = Spacecraft::cartesian(-7437.668796715336, -12882.420245780639, -40869.654144715205, 0.01311202708510157,
                                                 0.022710697101615124, -0.3016510044810502, 0, moon);
    const Spacecraft truth = Spacecraft::cartesian(-1415.2989082524969, 0.0, -1187.576791920277, 1.0471505397646481, 0.0, -1.2477825100469835, 0, moon);
    const auto dynamics = SpacecraftDynamics::new_(OrbitalDynamics::two_body());
    auto setup = Propagator::rk89(dynamics, IntegratorOptions::with_fixed_step_s(10.0));
    const size_t n = 2, m = 12;
    const int64_t end = (int64_t)(m + 1) * 60 * NS_PER_S;
    const auto rec = setup.propagate_batch_traj({tx0}, end, end / (10 * NS_PER_S) + 4);
    Traj traj; traj.name = "NRHO Tx SC"; traj.frame = moon;
    for (int64_t s = 0; s < rec.t_count[0]; ++s) {
        traj.epoch_ns.push_back(rec.epoch_at((size_t)s, 0));
        for (int c = 0; c < 6; ++c) traj.state.push_back(rec.state_at(c, (size_t)s, 0));
    }
    const StochasticNoise rn{1e-3, 0.0}, dn{1e-6, 0.0};
    InterlinkTxSpacecraft link{"NRHO", traj, {MeasurementType::Range, MeasurementType::Doppler}, {rn, dn}, std::nullopt, std::nullopt};
    CHECK(link.name() == "NRHO Tx SC");
    TrackingDataArc arc; arc.n = n; arc.ns = 2;
    for (size_t k = 1; k <= m; ++k) {
        arc.epoch_ns.push_back((int64_t)k * 60 * NS_PER_S);
        arc.tracker.push_back("NRHO");
        for (size_t e = 0; e < 2 * n; ++e) arc.obs.push_back(1.0);   // nonzero: the rows divide by the observed range
    }
    const double d[9] = {1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0, 0, 0};
    const std::vector<KfEstimate> ests{KfEstimate::from_diag(truth, d), KfEstimate::from_diag(truth, d)};
    {
        InterlinkKalmanODProcess sim(setup, KalmanVariant::DeviationTracking, std::nullopt, {link}, nullptr, 2);
        const ODSolution first = sim.process_arcs(ests, arc);
        CHECK(first.ns == 2 && first.status[0] == 0 && first.status[1] == 0);
        for (size_t k = 0; k < m; ++k) CHECK(first.msr_flags[k * n] == NYXB_MSRF_PROCESSED);
        for (size_t e = 0; e < arc.obs.size(); ++e) arc.obs[e] = arc.obs[e] - first.prefit[e];   // list [R, D]: slot = type
    }
    for (int32_t msr : {2, 1}) {
        InterlinkKalmanODProcess odp(setup, KalmanVariant::DeviationTracking, std::nullopt, {link}, nullptr, msr);
        const ODSolution plain = odp.process_arcs(ests, arc);
        const ODSolution sol = odp.process_arcs(ests, arc, 128);
        CHECK(sol.state == plain.state && sol.covar == plain.covar && sol.postfit == plain.postfit);
        CHECK(sol.status[0] == 0 && sol.status[1] == 0 && sol.n_estimates(0) == sol.rec_count[0]);
        int meas = 0;
        for (int64_t k = 0; k < sol.n_estimates(0); ++k) {
            const int64_t tg = sol.rec_tag[(size_t)k * n];
            if (tg < 0) continue;
            ++meas;
            CHECK(NYXB_OD_TAG_MSR_SIZE(tg) == msr);
        }
        CHECK(meas == (int)(m * (2 / msr)));
        for (size_t e = 0; e < sol.prefit.size(); ++e) CHECK(std::fabs(sol.prefit[e]) < 1e-9);
        const ODSolution sm = sol.smooth(odp, arc);
        CHECK(sm.is_smoother_run() && sm.sm_postfit.size() == (size_t)128 * 2 * n);
        for (size_t i = 0; i < n; ++i) {
            CHECK(sm.sm_status[i] == 0);
            double worst = 0.0;
            for (int64_t k = 0; k < sm.n_estimates(i); ++k)
                for (int r = 0; r < 9; ++r) worst = std::fmax(worst, std::fabs(sm.sm_deviation[((size_t)k * 9 + r) * n + i]));
            CHECK(worst < 1e-9);
        }
    }
    // a Doppler-only device: NYXB_ERR_NO_RANGE once filter 1's range is missing; a recording ending after 5 minutes: NYXB_ERR_TX_NO_DATA
    {
        TrackingDataArc a = arc;
        a.obs[(3 * 2 + 0) * n + 1] = NAN;
        InterlinkKalmanODProcess odp(setup, KalmanVariant::ReferenceUpdate, std::nullopt, {link}, nullptr, 2);
        const ODSolution s = odp.process_arcs(ests, a);
        CHECK(s.status[0] == 0 && s.status[1] == NYXB_ERR_NO_RANGE);
        InterlinkTxSpacecraft shortl = link;
        while (shortl.traj.epoch_ns.back() > 5 * 60 * NS_PER_S) { shortl.traj.epoch_ns.pop_back(); shortl.traj.state.resize(shortl.traj.state.size() - 6); }
        InterlinkKalmanODProcess odp2(setup, KalmanVariant::ReferenceUpdate, std::nullopt, {shortl}, nullptr, 2);
        const ODSolution s2 = odp2.process_arcs(ests, arc);
        CHECK(s2.status[0] == NYXB_ERR_TX_NO_DATA && s2.status[1] == NYXB_ERR_TX_NO_DATA);
        InterlinkTxSpacecraft lt = link; lt.ab_corr = "LT";
        InterlinkKalmanODProcess bad(setup, KalmanVariant::ReferenceUpdate, std::nullopt, {lt}, nullptr, 2);
        bool threw = false;
        try { bad.process_arcs(ests, arc); } catch (const std::runtime_error&) { threw = true; }
        CHECK(threw);
    }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
