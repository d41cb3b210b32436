// C++ host-mirror test of angle tracking: KalmanODProcess::process_arcs and ODSolution::smooth with ground stations that measure
// azimuth and elevation, through nyxb.hpp -> C ABI (nyxb_od_aer_batch, nyxb_od_aer_smooth_batch) -> CUDA kernels.  The observations
// are the filter's own computed values: a first CKF run from the truth (whose nominal is never replaced) gives obs - prefit = the
// computed range, Doppler, azimuth and elevation to the last bit; a second run on them then has zero prefits and deviations, and so has every
// smoothed estimate.  Range/Doppler-only stations give the same bits through either entry point (STRICT).
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
    const StochasticNoise mn{1e-6, 0.0};
    std::vector<GroundStation> stations{GroundStation::dss65_madrid(-90.0, mn, mn), GroundStation::dss34_canberra(-90.0, mn, mn),
                                        GroundStation::dss13_goldstone(-90.0, mn, mn)};
    for (auto& gs : stations) gs.with_msr_type(MeasurementType::Azimuth, mn).with_msr_type(MeasurementType::Elevation, mn);
    const size_t n = 2, m = 12;
    TrackingDataArc arc; arc.n = n; arc.ns = 4;
    for (size_t k = 1; k <= m; ++k) {
        arc.epoch_ns.push_back((int64_t)k * 30 * NS_PER_S);
        arc.tracker.push_back(stations[k % 3].name);
        for (size_t e = 0; e < 4 * n; ++e) arc.obs.push_back(1.0);   // nonzero: the range row divides by the observed range
    }
    const double d[9] = {1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0, 0, 0};
    const std::vector<KfEstimate> ests{KfEstimate::from_diag(truth, d), KfEstimate::from_diag(truth, d)};
    {
        KalmanODProcess sim(setup, KalmanVariant::DeviationTracking, std::nullopt, stations, nullptr, 2);
        const ODSolution first = sim.process_arcs(ests, arc);
        CHECK(first.ns == 4 && first.status[0] == 0 && first.status[1] == 0);
        for (size_t e = 0; e < arc.obs.size(); ++e) arc.obs[e] = arc.obs[e] - first.prefit[e];   // list [R, D, Az, El]: slot = type
    }
    for (int32_t msr : {2, 1}) {
        KalmanODProcess odp(setup, KalmanVariant::DeviationTracking, std::nullopt, stations, nullptr, msr);
        const ODSolution plain = odp.process_arcs(ests, arc);
        const ODSolution sol = odp.process_arcs(ests, arc, 128);
        CHECK(sol.ns == 4 && sol.prefit.size() == m * 4 * n);
        CHECK(sol.state == plain.state && sol.covar == plain.covar && sol.postfit == plain.postfit);
        CHECK(sol.status[0] == 0 && sol.status[1] == 0 && sol.n_estimates(0) == sol.rec_count[0]);
        int meas = 0;
        for (int64_t k = 0; k < sol.n_estimates(0); ++k) {
            const int64_t tg = sol.rec_tag[(size_t)k * n];
            if (tg < 0) continue;
            ++meas;
            CHECK(NYXB_OD_POS_TAG_MSR_SIZE(tg) == msr && NYXB_OD_POS_TAG_WINDOW(tg) < 4 / msr);
        }
        CHECK(meas == (int)(m * (4 / msr)));
        for (size_t e = 0; e < sol.prefit.size(); ++e) CHECK(std::fabs(sol.prefit[e]) < 1e-9);
        for (size_t k = 0; k < m; ++k)
            for (int w = 0; w < 4; ++w) CHECK(std::isnan(sol.resid_ratio[(k * 4 + w) * n]) == (w >= 4 / msr));   // ratio of window w in slot w
        const ODSolution sm = sol.smooth(odp, arc);
        CHECK(sm.is_smoother_run() && sm.sm_postfit.size() == (size_t)128 * 4 * n);
        for (size_t i = 0; i < n; ++i) {
            CHECK(sm.sm_status[i] == 0);
            double worst = 0.0;
            for (int64_t k = 0; k < sm.n_estimates(i); ++k)
                for (int r = 0; r < 9; ++r) worst = std::fmax(worst, std::fabs(sm.sm_deviation[((size_t)k * 9 + r) * n + i]));
            CHECK(worst < 1e-9);
        }
    }
    // range/Doppler-only stations: a two-slot arc (nyxb_od_ekf_batch) and the same data in four slots (nyxb_od_aer_batch)
    std::vector<GroundStation> rd{GroundStation::dss65_madrid(-90.0, mn, mn), GroundStation::dss34_canberra(-90.0, mn, mn),
                                  GroundStation::dss13_goldstone(-90.0, mn, mn)};
    TrackingDataArc arc2 = arc; arc2.ns = 2; arc2.obs.clear();
    TrackingDataArc arc4 = arc;
    for (size_t k = 0; k < m; ++k)
        for (size_t q = 0; q < 4; ++q)
            for (size_t i = 0; i < n; ++i) {
                const double v = arc.obs[(k * 4 + q) * n + i];
                if (q < 2) arc2.obs.push_back(v + 1e-3 * (double)(i + 1));
                arc4.obs[(k * 4 + q) * n + i] = q < 2 ? v + 1e-3 * (double)(i + 1) : NAN;
            }
    KalmanODProcess rdp(setup, KalmanVariant::ReferenceUpdate, std::nullopt, rd, nullptr, 2);
    const ODSolution a = rdp.process_arcs(ests, arc4), g = rdp.process_arcs(ests, arc2);
    CHECK(a.ns == 4 && g.ns == 2 && a.state == g.state && a.covar == g.covar && a.msr_flags == g.msr_flags);
    for (size_t k = 0; k < m; ++k)
        for (size_t q = 0; q < 2; ++q)
            for (size_t i = 0; i < n; ++i) {
                const double x = a.prefit[(k * 4 + q) * n + i], y = g.prefit[(k * 2 + q) * n + i];
                CHECK(x == y || (std::isnan(x) && std::isnan(y)));
            }
    CHECK(a.status[0] == 0 && a.status[1] == 0);
    // stations with angles need the four-slot arc
    KalmanODProcess bad(setup, KalmanVariant::ReferenceUpdate, std::nullopt, stations, nullptr, 2);
    bool threw = false;
    try { bad.process_arcs(ests, arc2); } catch (const std::runtime_error&) { threw = true; }
    CHECK(threw);
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
