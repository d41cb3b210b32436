// C++ host-mirror test of impulsive targeting: nyxb::Targeter through nyxb.hpp -> C ABI -> CUDA kernels, on the reference's two-body
// cases (tests/mission_design/targeter): SMA from apoapsis and C3 + declination in VNC, with their GMAT bounds, an ensemble with a failing
// problem, apply() and its Verification (also the one the corrected-state quirk causes in VNC), and the FrameError of a position variable with a frame.
#include <cmath>
#include <cstdio>

#include "nyxb.hpp"

using namespace nyxb;
static int failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++failures; } } while (0)

static double norm(const std::vector<double>& v) { double s = 0.0; for (double x : v) s += x * x; return std::sqrt(s); }

int main() {
    const Frame eme2k = EARTH_J2000();
    // Orbit::keplerian(8 000 km, 0.2, 30, 60, 60, TA) at apoapsis (TA 180) and periapsis (TA 0); half a period = 3 560.5 s
    Spacecraft apo = Spacecraft::cartesian(3835.3829072479552, -7756.921938165308, -4156.921938165305, 4.6568950360385735,
                                           3.0747337513619453, -1.4408483385016626, 0, eme2k);
    Spacecraft peri = Spacecraft::cartesian(-2556.9219381653043, 5171.281292110205, 2771.281292110203, -6.985342554057858,
                                            -4.612100627042918, 2.161272507752493, 0, eme2k);
    apo.dry_mass_kg = peri.dry_mass_kg = 100.0;
    const int64_t half = 3560540817212LL;
    const auto dynamics = SpacecraftDynamics::new_(OrbitalDynamics::two_body());
    const auto dp78 = Propagator::dp78(dynamics, IntegratorOptions::default_());

    // tgt_sma_from_apo
    Targeter sma = Targeter::delta_v(dp78, {Objective::new_(NYXB_TGT_SMA, 8100.0)});
    TargeterSolution sol = sma.try_achieve_from(apo, 0, half);
    CHECK(std::fabs(norm(sol.correction) - 0.05312024615278713) < 1e-6);
    CHECK(sol.corrected_state.epoch() == 0 && sol.achieved_state.epoch() == half && sol.corrected_state.dry_mass_kg == 100.0);
    const Spacecraft fin = sma.apply(sol);
    CHECK(fin.epoch() == half);
    TargeterSolution bad = sol;
    bad.corrected_state = apo;
    bool verification = false;
    try { sma.apply(bad); } catch (const TargetingError& e) { verification = e.variant == "Verification"; }
    CHECK(verification);

    // tgt_vnc_c3_decl
    Targeter c3 = Targeter::vnc(Propagator::default_(dynamics),
                                {Objective::within_tolerance(NYXB_TGT_DECLINATION, 5.0, 0.1), Objective::within_tolerance(NYXB_TGT_C3, -5.0, 0.5)});
    TargeterSolution vs = c3.try_achieve_from(peri, 0, half);
    CHECK(std::fabs(norm(vs.correction) - 2.385704523944014) < 6e-3);
    // the corrected state applies the total correction once with the DCM of the start state, not the iterated one: in VNC and over
    // several iterations the two differ, and apply() fails Verification as the reference's does (its VNC test does not call apply)
    bool vnc_verification = false;
    try { c3.apply(vs); } catch (const TargetingError& e) { vnc_verification = e.variant == "Verification"; }
    CHECK(vs.iterations >= 2 && vnc_verification);

    // an ensemble: two converge, one runs out of iterations
    Targeter tight = Targeter::delta_v(dp78, {Objective::within_tolerance(NYXB_TGT_SMA, 8100.0, 1e-3)});
    tight.iterations = 2;
    Spacecraft far = apo; far.vx_km_s += 0.5;   // needs more than two clipped steps
    TargeterEnsembleSolution ens = tight.try_achieve_from_many({apo, far, apo}, 0, half);
    CHECK(ens.size() == 3 && ens.n_vars == 3 && ens.n_objs == 1);
    for (size_t i = 0; i < 3; ++i) std::printf("problem %zu: status %d iterations %d\n", i, ens.status[i], ens.iterations[i]);
    CHECK(!ens.error(0) && !ens.error(2) && ens.error(1) && *ens.error(1) == "TooManyIterations");
    CHECK(ens.iterations[0] == ens.iterations[2] && ens.correction[0] == ens.correction[2]);
    CHECK(std::fabs(norm(ens.solution(0).correction) - 0.05312024615278713) < 1e-6);

    // FrameError: a position variable in VNC is refused before any launch
    bool refused = false;
    try { Targeter::vnc_with_components(dp78, {Variable::from(Vary::PositionX)}, {Objective::new_(NYXB_TGT_SMA, 8100.0)}).try_achieve_from(apo, 0, half); }
    catch (const std::runtime_error& e) { refused = std::string(e.what()).find("FrameError") != std::string::npos; }
    CHECK(refused);

    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("OK\n");
    return 0;
}
