// nyxb.hpp — header-only C++17 host mirror of the reference's Rust surface for the propagation path,
// layered on the C ABI of nyxb.h (libnyxb.so).  The reference is compiled (Rust) code and its toolchain is not
// available in the build image, so this is the compiled-language host side a nyx maintainer would port 1:1 to a
// Rust shim (INTEGRATION.md).  Names, argument meaning and error behaviour follow the reference:
//
//   IntegratorMethod / ErrorControl / IntegratorOptions   propagators/rk_methods/mod.rs:65-79, error_ctrl.rs:30-71, options.rs:42-186
//   Propagator::{new_,rk89,dp78,default_,with}            propagators/propagator.rs:55-118
//   PropInstance::{for_duration,until_epoch,latest_details}   propagators/instance.rs:265-282, 495-498
//   SpacecraftDynamics / OrbitalDynamics / PointMasses / GravityField / SolarPressure / Drag   dynamics/*.rs
//   MonteCarlo::{generate_states,run_until_epoch,resume_run_until_epoch}   mc/montecarlo.rs:188-296
//   Propagator::propagate_batch_stm (Spacecraft::with_stm + propagate)       dynamics/spacecraft.rs:203-227, 312-363
//   GroundStation / StochasticNoise / ProcessNoise3D / SigmaRejection / KfEstimate / TrackingDataArc / KalmanODProcess
//                                                         od/ground_station, od/snc.rs, od/process/{mod,initializers,rejectcrit}.rs
//
// No arithmetic of the hot path lives here: every propagate call is one nyxb_propagate_batch on the GPU.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <memory>
#include <optional>
#include <random>
#include <stdexcept>
#include <string>
#include <variant>
#include <vector>

#include "nyxb.h"

namespace nyxb {

constexpr int64_t NS_PER_S = 1000000000LL;
// hifitime `f64 * Unit::Second`: truncation toward zero
inline int64_t seconds(double s) { return (int64_t)(s * 1e9); }
inline int64_t days(int64_t d) { return d * 86400 * NS_PER_S; }

enum class IntegratorMethod : int32_t { RungeKutta89 = NYXB_RK89, DormandPrince78 = NYXB_DP78, DormandPrince45 = NYXB_DP45,
                                        RungeKutta4 = NYXB_RK4, CashKarp45 = NYXB_CK45, Verner56 = NYXB_V56 };
enum class ErrorControl : int32_t { RSSCartesianState = NYXB_RSS_CARTESIAN_STATE, RSSCartesianStep = NYXB_RSS_CARTESIAN_STEP,
                                    RSSState = NYXB_RSS_STATE, RSSStep = NYXB_RSS_STEP, LargestError = NYXB_LARGEST_ERROR,
                                    LargestState = NYXB_LARGEST_STATE, LargestStep = NYXB_LARGEST_STEP };

// PropagationError (propagators/mod.rs:68-92) wrapping DynamicsError (dynamics/mod.rs:177-203)
struct PropagationError : std::runtime_error {
    int32_t status;
    explicit PropagationError(int32_t st) : std::runtime_error(describe(st)), status(st) {}
    static std::string describe(int32_t st) {
        switch (st & 0xff) {
        case NYXB_ERR_PROP_MATH: return "PropMathError: part of state vector is NaN";
        case NYXB_ERR_FUEL_EXHAUSTED: return "DynamicsError::FuelExhausted";
        case NYXB_ERR_MASSLESS: return "DynamicsError::MasslessSpacecraft";
        case NYXB_ERR_EPHEMERIS: return "DynamicsError::DynamicsAlmanacError (epoch outside ephemeris coverage)";
        default: return "propagation error " + std::to_string(st);
        }
    }
};

// IntegratorOptions (options.rs:42-186); durations in integer nanoseconds
struct IntegratorOptions {
    int64_t init_step = 60 * NS_PER_S, min_step = NS_PER_S / 1000, max_step = 2700 * NS_PER_S;
    double tolerance = 1e-12;
    int32_t attempts = 50;
    bool fixed_step = false;
    ErrorControl error_ctrl = ErrorControl::RSSCartesianStep;
    static IntegratorOptions default_() { return {}; }
    static IntegratorOptions with_adaptive_step(int64_t min_step, int64_t max_step, double tol, ErrorControl ctrl) {
        return {max_step, min_step, max_step, tol, 50, false, ctrl};  // options.rs:66-82
    }
    static IntegratorOptions with_adaptive_step_s(double mn, double mx, double tol, ErrorControl ctrl) {
        return with_adaptive_step(seconds(mn), seconds(mx), tol, ctrl);
    }
    static IntegratorOptions with_fixed_step(int64_t step) {
        return {step, step, step, 0.0, 0, true, ErrorControl::RSSCartesianStep};  // options.rs:100-111
    }
    static IntegratorOptions with_fixed_step_s(double s) { return with_fixed_step(seconds(s)); }
    static IntegratorOptions with_tolerance(double tol) { IntegratorOptions o; o.tolerance = tol; return o; }
    void set_max_step(int64_t m) { if (init_step > m) init_step = m; max_step = m; }
    void set_min_step(int64_t m) { if (init_step < m) init_step = m; min_step = m; }
};

// Subset of anise's Frame used on the path + the explicit orientation model of nyxb.h
struct Frame {
    int32_t ephemeris_id = 399;
    double mu_km3_s2 = 398600.435436096;
    double mean_equatorial_radius_km = 6378.14;
    nyxb_rotation rotation{};  // kind 0: inertial axes
    double polar_radius_km = 0.0;  // > 0: ellipsoid for geodetic coordinates (ground stations); 0: sphere
    Frame with_mu_km3_s2(double mu) const { Frame f = *this; f.mu_km3_s2 = mu; return f; }
};
inline Frame EARTH_J2000() { return {}; }
inline Frame IAU_EARTH() {
    Frame f;
    f.rotation = nyxb_rotation{1, 0, 0.0, -0.641, 90.0, -0.557, 190.147, 360.9856235};  // pck00008
    f.polar_radius_km = 6356.75;
    return f;
}

// Spacecraft (cosmic/spacecraft.rs:115-143) without thruster / guidance / STM members
struct Spacecraft {
    double x_km = 0, y_km = 0, z_km = 0, vx_km_s = 0, vy_km_s = 0, vz_km_s = 0;
    int64_t epoch_ns = 0;
    Frame frame;
    double dry_mass_kg = 0, prop_mass_kg = 0, extra_mass_kg = 0;
    double srp_area_m2 = 0, coeff_reflectivity = 1.8, drag_area_m2 = 0, coeff_drag = 2.2;  // anise defaults
    static Spacecraft cartesian(double x, double y, double z, double vx, double vy, double vz, int64_t epoch_ns, const Frame& f) {
        Spacecraft s; s.x_km = x; s.y_km = y; s.z_km = z; s.vx_km_s = vx; s.vy_km_s = vy; s.vz_km_s = vz; s.epoch_ns = epoch_ns; s.frame = f;
        return s;
    }
    int64_t epoch() const { return epoch_ns; }
};

// Ephemeris container standing in for anise's Almanac (see nyxb_body)
struct BodyEphemeris {
    int32_t ephemeris_id; double mu_km3_s2, radius_km; int64_t t0_ns, interval_ns; int32_t n_coeffs;
    std::vector<double> coeffs;  // [n_intervals][3][n_coeffs]
};
struct Almanac { std::vector<BodyEphemeris> bodies; };

struct GravityFieldData {  // io/gravity.rs:90-128
    int32_t degree = 0, order = 0;
    std::vector<double> c_nm, s_nm;  // row-major (degree+1)^2
    Frame frame;
    static GravityFieldData from_j2(double j2, const Frame& frame) {
        GravityFieldData g; g.degree = 2; g.order = 0; g.c_nm.assign(9, 0.0); g.s_nm.assign(9, 0.0); g.c_nm[2 * 3 + 0] = j2; g.frame = frame;
        return g;
    }
};
struct PointMasses { std::vector<int32_t> celestial_objects; };
struct GravityField { GravityFieldData grav_data; };
struct SolarPressure { double phi = 1367.0; int32_t light_source = 10; std::vector<int32_t> shadow_bodies; bool estimate = true; /* solarpressure.rs:47-48, 88-92 */ };
struct Drag { int32_t density = NYXB_DENSITY_EXPONENTIAL; double rho0 = 3.614e-13, r0 = 700000.0, ref_alt_m = 88667.0; Frame frame = IAU_EARTH(); };

struct OrbitalDynamics {
    std::optional<PointMasses> point_masses_;
    std::optional<GravityField> gravity_;
    static OrbitalDynamics two_body() { return {}; }
    static OrbitalDynamics point_masses(std::vector<int32_t> objs) { OrbitalDynamics o; o.point_masses_ = PointMasses{std::move(objs)}; return o; }
    static OrbitalDynamics from_model(GravityField g) { OrbitalDynamics o; o.gravity_ = std::move(g); return o; }
};
struct SpacecraftDynamics {
    OrbitalDynamics orbital_dyn;
    std::optional<SolarPressure> srp;
    std::optional<Drag> drag;
    static SpacecraftDynamics new_(OrbitalDynamics o) { SpacecraftDynamics d; d.orbital_dyn = std::move(o); return d; }
};

struct IntegrationDetails { int64_t step_ns = 0; double error = 0; int32_t attempts = 1; int64_t n_steps = 0, n_rejected = 0, n_rhs = 0; };

namespace detail {
struct EngineDeleter { void operator()(nyxb_engine* e) const { nyxb_engine_destroy(e); } };
using EnginePtr = std::unique_ptr<nyxb_engine, EngineDeleter>;

inline EnginePtr make_engine(const SpacecraftDynamics& dyn, const Frame& frame, const Almanac* almanac, IntegratorMethod method,
                             const IntegratorOptions& o, int32_t mode, int32_t device) {
    nyxb_integ_opts co{(int32_t)method, (int32_t)o.error_ctrl, o.init_step, o.min_step, o.max_step, o.tolerance, o.attempts, o.fixed_step ? 1 : 0};
    nyxb_dynamics d{};
    d.mu_central_km3_s2 = frame.mu_km3_s2;
    d.central_radius_km = frame.mean_equatorial_radius_km;
    std::vector<nyxb_body> bodies;
    auto body_index = [&](int32_t id) -> int32_t {
        if (almanac) for (size_t i = 0; i < almanac->bodies.size(); ++i) if (almanac->bodies[i].ephemeris_id == id) return (int32_t)i;
        throw std::runtime_error("planetary data from third body not loaded");
    };
    if (almanac) for (auto& b : almanac->bodies)
        bodies.push_back(nyxb_body{b.mu_km3_s2, b.radius_km, b.t0_ns, b.interval_ns, (int32_t)(b.coeffs.size() / (3 * b.n_coeffs)), b.n_coeffs, b.coeffs.data()});
    d.n_bodies = (int32_t)bodies.size();
    d.bodies = bodies.data();
    if (dyn.orbital_dyn.point_masses_)
        for (int32_t id : dyn.orbital_dyn.point_masses_->celestial_objects) {   // summation order of orbital.rs:217
            if (id == frame.ephemeris_id) continue;                              // orbital.rs:219-222
            const int32_t j = body_index(id);
            if (!((d.point_mass_mask >> j) & 1u)) d.point_mass_order[d.n_point_masses++] = j;
            d.point_mass_mask |= 1u << j;
        }
    nyxb_gravity_field g{};
    if (dyn.orbital_dyn.gravity_) {
        const auto& gd = dyn.orbital_dyn.gravity_->grav_data;
        // a field of another body than the integration centre is evaluated about that body (gravity_field.rs:149-154)
        const int32_t gbody = gd.frame.ephemeris_id == frame.ephemeris_id ? NYXB_CENTRAL_BODY : body_index(gd.frame.ephemeris_id);
        g = nyxb_gravity_field{gd.degree, gd.order, gd.frame.mu_km3_s2, gd.frame.mean_equatorial_radius_km, gd.c_nm.data(), gd.s_nm.data(), gd.frame.rotation, gbody, 0};
        d.gravity = &g;
        d.n_gravity = 1;
    }
    nyxb_srp s{};
    if (dyn.srp) {
        s.phi_w_m2 = dyn.srp->phi; s.sun_body = body_index(dyn.srp->light_source); s.n_shadow = (int32_t)dyn.srp->shadow_bodies.size(); s.estimate = dyn.srp->estimate ? 1 : 0;
        for (int q = 0; q < s.n_shadow && q < 4; ++q)
            s.shadow_body[q] = dyn.srp->shadow_bodies[q] == frame.ephemeris_id ? NYXB_CENTRAL_BODY : body_index(dyn.srp->shadow_bodies[q]);
        d.srp = &s;
    }
    nyxb_drag dr{};
    if (dyn.drag) {
        dr = nyxb_drag{dyn.drag->density, 0, dyn.drag->rho0, dyn.drag->r0, dyn.drag->ref_alt_m, dyn.drag->frame.mean_equatorial_radius_km, dyn.drag->frame.rotation};
        d.drag = &dr;
    }
    nyxb_engine* e = nyxb_engine_create(&d, &co, mode, device);
    if (!e) throw std::runtime_error(std::string("nyxb_engine_create: ") + nyxb_last_error());
    return EnginePtr(e);
}

struct Soa {
    std::vector<double> state, consts; std::vector<int64_t> epoch;
    explicit Soa(const std::vector<Spacecraft>& v) : state(9 * v.size()), consts(4 * v.size()), epoch(v.size()) {
        const size_t n = v.size();
        for (size_t i = 0; i < n; ++i) {
            const Spacecraft& s = v[i];
            const double y[9] = {s.x_km, s.y_km, s.z_km, s.vx_km_s, s.vy_km_s, s.vz_km_s, s.coeff_reflectivity, s.coeff_drag, s.prop_mass_kg};
            for (int e = 0; e < 9; ++e) state[e * n + i] = y[e];  // cosmic/spacecraft.rs:449-473
            consts[i] = s.dry_mass_kg; consts[n + i] = s.extra_mass_kg; consts[2 * n + i] = s.srp_area_m2; consts[3 * n + i] = s.drag_area_m2;
            epoch[i] = s.epoch_ns;
        }
    }
};
inline Spacecraft unpack(const Spacecraft& tmpl, const std::vector<double>& out, const std::vector<int64_t>& ep, size_t n, size_t i) {
    Spacecraft s = tmpl;
    s.x_km = out[i]; s.y_km = out[n + i]; s.z_km = out[2 * n + i]; s.vx_km_s = out[3 * n + i]; s.vy_km_s = out[4 * n + i]; s.vz_km_s = out[5 * n + i];
    s.coeff_reflectivity = out[6 * n + i]; s.coeff_drag = out[7 * n + i]; s.prop_mass_kg = out[8 * n + i]; s.epoch_ns = ep[i];
    return s;
}
}  // namespace detail

class PropInstance;

// Propagator<SpacecraftDynamics> (propagator.rs:34-118)
class Propagator {
  public:
    SpacecraftDynamics dynamics;
    IntegratorOptions opts;
    IntegratorMethod method = IntegratorMethod::RungeKutta89;
    int32_t mode = NYXB_MODE_STRICT, device = 0;
    int32_t kernel = NYXB_KERNEL_AUTO;   // nyxb_engine_set_kernel: AUTO = the library's dispatch (by mode, field degree, ensemble size)
    static Propagator new_(SpacecraftDynamics d, IntegratorMethod m, IntegratorOptions o) { Propagator p; p.dynamics = std::move(d); p.method = m; p.opts = o; return p; }
    static Propagator rk89(SpacecraftDynamics d, IntegratorOptions o) { return new_(std::move(d), IntegratorMethod::RungeKutta89, o); }
    static Propagator dp78(SpacecraftDynamics d, IntegratorOptions o) { return new_(std::move(d), IntegratorMethod::DormandPrince78, o); }
    static Propagator default_(SpacecraftDynamics d) { return rk89(std::move(d), IntegratorOptions::default_()); }
    Propagator& with_mode(int32_t m) { mode = m; return *this; }
    inline PropInstance with(const Spacecraft& state, const Almanac* almanac = nullptr) const;

    struct BatchResult { std::vector<double> state; std::vector<int64_t> epoch; std::vector<nyxb_details> details; std::vector<int32_t> status; };
    // the rayon fan-out of mc/montecarlo.rs:233-253 as ONE batched call
    BatchResult propagate_batch(const std::vector<Spacecraft>& v, int64_t end_epoch_ns, const Almanac* almanac = nullptr,
                                std::vector<int64_t>* step_io = nullptr) const {
        BatchResult r;
        const size_t n = v.size();
        r.state.resize(9 * n); r.epoch.resize(n); r.details.resize(n); r.status.resize(n);
        if (n == 0) return r;
        auto eng = detail::make_engine(dynamics, v[0].frame, almanac, method, opts, mode, device);
        if (kernel != NYXB_KERNEL_AUTO && nyxb_engine_set_kernel(eng.get(), kernel) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_engine_set_kernel: ") + nyxb_last_error());
        detail::Soa soa(v);
        int32_t rc = nyxb_propagate_batch(eng.get(), n, soa.state.data(), soa.consts.data(), soa.epoch.data(), end_epoch_ns,
                                          step_io ? step_io->data() : nullptr, r.state.data(), r.epoch.data(), r.details.data(), r.status.data());
        if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_propagate_batch: ") + nyxb_last_error());
        return r;
    }
    // the same fan-out over several GPUs of this process: one engine per device, contiguous run-index shards, results copied
    // straight into the caller's arrays (nyxb_propagate_batch_multi; mc/montecarlo.rs:188-203 on G GPUs is ONE call of it)
    BatchResult propagate_batch_multi(const std::vector<Spacecraft>& v, int64_t end_epoch_ns, const std::vector<int32_t>& devices,
                                      const Almanac* almanac = nullptr, std::vector<int64_t>* step_io = nullptr) const {
        BatchResult r;
        const size_t n = v.size();
        r.state.resize(9 * n); r.epoch.resize(n); r.details.resize(n); r.status.resize(n);
        if (n == 0) return r;
        if (devices.empty()) throw std::runtime_error("propagate_batch_multi: no devices");
        std::vector<detail::EnginePtr> engs;
        std::vector<nyxb_engine*> raw;
        for (int32_t d : devices) {
            engs.push_back(detail::make_engine(dynamics, v[0].frame, almanac, method, opts, mode, d));
            if (kernel != NYXB_KERNEL_AUTO && nyxb_engine_set_kernel(engs.back().get(), kernel) != NYXB_RC_OK)
                throw std::runtime_error(std::string("nyxb_engine_set_kernel: ") + nyxb_last_error());
            raw.push_back(engs.back().get());
        }
        detail::Soa soa(v);
        int32_t rc = nyxb_propagate_batch_multi(raw.data(), (int32_t)raw.size(), n, soa.state.data(), soa.consts.data(), soa.epoch.data(),
                                                end_epoch_ns, step_io ? step_io->data() : nullptr, r.state.data(), r.epoch.data(),
                                                r.details.data(), r.status.data());
        if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_propagate_batch_multi: ") + nyxb_last_error());
        return r;
    }
    // Spacecraft::with_stm() + until_epoch for a batch: final states and the 9x9 STMs (column-major per trajectory, [81][n])
    struct StmResult { std::vector<double> state, stm; std::vector<int64_t> epoch; std::vector<nyxb_details> details; std::vector<int32_t> status;
                       double phi(size_t n, size_t i, int r, int c) const { return stm[(size_t)(c * 9 + r) * n + i]; } };
    StmResult propagate_batch_stm(const std::vector<Spacecraft>& v, int64_t end_epoch_ns, const Almanac* almanac = nullptr,
                                  const std::vector<double>* stm_in = nullptr) const {
        StmResult r;
        const size_t n = v.size();
        r.state.resize(9 * n); r.stm.resize(81 * n); r.epoch.resize(n); r.details.resize(n); r.status.resize(n);
        if (n == 0) return r;
        auto eng = detail::make_engine(dynamics, v[0].frame, almanac, method, opts, mode, device);
        detail::Soa soa(v);
        int32_t rc = nyxb_propagate_batch_stm(eng.get(), n, soa.state.data(), soa.consts.data(), soa.epoch.data(), end_epoch_ns, nullptr,
                                              stm_in ? stm_in->data() : nullptr, r.state.data(), r.epoch.data(), r.stm.data(),
                                              r.details.data(), r.status.data());
        if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_propagate_batch_stm: ") + nyxb_last_error());
        return r;
    }
    // until_epoch_with_traj for a batch (instance.rs:297-340): final states + every accepted step of every trajectory in the
    // step-major SoA sink; `every(queries)` = Traj::at (md/trajectory/traj.rs:83-126) for all trajectories and query epochs in
    // one launch on the recording still resident on the device (nyxb_traj_resample).
    struct Resampled {
        size_t m = 0, n = 0; std::vector<double> state; std::vector<int32_t> status;   // [6][m][n], [m][n]
        double at(int c, size_t j, size_t i) const { return state[((size_t)c * m + j) * n + i]; }
        bool ok(size_t j, size_t i) const { return status[j * n + i] == NYXB_TRAJ_OK; }
    };
    struct TrajBatch : BatchResult {
        int64_t capacity = 0; size_t n = 0;
        std::vector<int64_t> t_epoch, t_count; std::vector<double> t_state;   // [cap][n], [n], [6][cap][n]
        std::shared_ptr<nyxb_engine> engine;
        int64_t epoch_at(size_t s, size_t i) const { return t_epoch[s * n + i]; }
        double state_at(int c, size_t s, size_t i) const { return t_state[((size_t)c * capacity + s) * n + i]; }
        Resampled every(const std::vector<int64_t>& query_epoch_ns) const {
            Resampled r; r.m = query_epoch_ns.size(); r.n = n;
            r.state.resize(6 * r.m * n); r.status.resize(r.m * n);
            int32_t rc = nyxb_traj_resample(engine.get(), n, nullptr, r.m, query_epoch_ns.data(), r.state.data(), r.status.data());
            if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_traj_resample: ") + nyxb_last_error());
            return r;
        }
        // the Brent search of until_nth_event (event.rs:186-211) inside every trajectory's last recorded step, one launch
        struct Located { std::vector<int64_t> epoch; std::vector<double> state; std::vector<int32_t> status; };   // [n], [6][n], [n]
        Located locate(int32_t event_kind, double value, int64_t epoch_precision_ns = 1000000) const {
            Located r; r.epoch.resize(n); r.state.resize(6 * n); r.status.resize(n);
            int32_t rc = nyxb_event_locate(engine.get(), n, nullptr, event_kind, value, epoch_precision_ns, status.data(), r.epoch.data(),
                                           r.state.data(), r.status.data());
            if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_event_locate: ") + nyxb_last_error());
            return r;
        }
    };
    // `event` != nullptr: stop every run at the end of the step in which the event scalar crossed zero for the trigger-th time
    TrajBatch propagate_batch_traj(const std::vector<Spacecraft>& v, int64_t end_epoch_ns, int64_t capacity, const Almanac* almanac = nullptr,
                                   nyxb_event* event = nullptr) const {
        TrajBatch r;
        const size_t n = v.size();
        r.n = n; r.capacity = capacity;
        r.state.resize(9 * n); r.epoch.resize(n); r.details.resize(n); r.status.resize(n);
        r.t_epoch.assign((size_t)capacity * n, 0); r.t_state.assign((size_t)6 * capacity * n, 0.0); r.t_count.assign(n, 0);
        if (n == 0) return r;
        r.engine = std::shared_ptr<nyxb_engine>(detail::make_engine(dynamics, v[0].frame, almanac, method, opts, mode, device).release(), nyxb_engine_destroy);
        detail::Soa soa(v);
        nyxb_traj_sink sink{capacity, r.t_epoch.data(), r.t_state.data(), r.t_count.data()};
        int32_t rc = nyxb_propagate_batch_event(r.engine.get(), n, soa.state.data(), soa.consts.data(), soa.epoch.data(), end_epoch_ns, nullptr,
                                                r.state.data(), r.epoch.data(), r.details.data(), r.status.data(), &sink, event);
        if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_propagate_batch_event: ") + nyxb_last_error());
        return r;
    }
    // nyx-py Propagator.many_until_epoch (py_md.rs:224-271): failed runs are dropped
    std::vector<Spacecraft> many_until_epoch(const std::vector<Spacecraft>& v, int64_t end_epoch_ns, const Almanac* almanac = nullptr) const {
        auto r = propagate_batch(v, end_epoch_ns, almanac);
        std::vector<Spacecraft> out;
        for (size_t i = 0; i < v.size(); ++i) if ((r.status[i] & 0xff) == 0) out.push_back(detail::unpack(v[i], r.state, r.epoch, v.size(), i));
        return out;
    }
};

// PropInstance (instance.rs:41-499): keeps the adapted step between calls
class PropInstance {
  public:
    Spacecraft state;
    IntegrationDetails details;
    PropInstance(const Propagator& p, const Spacecraft& s, const Almanac* a) : state(s), prop_(p), almanac_(a), step_{p.opts.init_step} {
        details.step_ns = p.opts.init_step;
    }
    Spacecraft for_duration(int64_t duration_ns) { return until_epoch(state.epoch_ns + duration_ns); }
    Spacecraft until_epoch(int64_t end_ns) {
        auto r = prop_.propagate_batch({state}, end_ns, almanac_, &step_);
        if (r.status[0] & 0xff) throw PropagationError(r.status[0]);
        if (r.details[0].n_steps > 0) details = {r.details[0].step_ns, r.details[0].error, r.details[0].attempts, r.details[0].n_steps, r.details[0].n_rejected, r.details[0].n_rhs};
        state = detail::unpack(state, r.state, r.epoch, 1, 0);
        return state;
    }
    IntegrationDetails latest_details() const { return details; }
  private:
    Propagator prop_;
    const Almanac* almanac_;
    std::vector<int64_t> step_;
};
inline PropInstance Propagator::with(const Spacecraft& state, const Almanac* almanac) const { return PropInstance(*this, state, almanac); }

// MonteCarlo (mc/montecarlo.rs:48-327) with a diagonal Cartesian dispersion (MvnSpacecraft::from_spacecraft_cov with a diagonal covariance)
struct Run { size_t index; Spacecraft dispersed_state; std::variant<Spacecraft, PropagationError> result; };
struct Results { std::vector<Run> runs; std::string scenario; int64_t total_steps = 0; };
class MonteCarlo {
  public:
    Spacecraft nominal_state; double std_dev[9]; std::string scenario; uint64_t seed;
    MonteCarlo(Spacecraft nominal, const double (&sd)[9], std::string name, uint64_t seed_) : nominal_state(nominal), scenario(std::move(name)), seed(seed_) {
        for (int i = 0; i < 9; ++i) std_dev[i] = sd[i];
    }
    // mc/montecarlo.rs:277-296: one serial stream; `skip` discards the first draws
    std::vector<Spacecraft> generate_states(size_t skip, size_t num_runs) const {
        std::mt19937_64 rng(seed);
        std::normal_distribution<double> nrm(0.0, 1.0);
        std::vector<Spacecraft> out;
        for (size_t i = 0; i < skip + num_runs; ++i) {
            double z[9];
            for (double& v : z) v = nrm(rng);
            if (i < skip) continue;
            Spacecraft s = nominal_state;
            s.x_km += std_dev[0] * z[0]; s.y_km += std_dev[1] * z[1]; s.z_km += std_dev[2] * z[2];
            s.vx_km_s += std_dev[3] * z[3]; s.vy_km_s += std_dev[4] * z[4]; s.vz_km_s += std_dev[5] * z[5];
            s.coeff_reflectivity += std_dev[6] * z[6]; s.coeff_drag += std_dev[7] * z[7]; s.prop_mass_kg += std_dev[8] * z[8];
            out.push_back(s);
        }
        return out;
    }
    // the same dispersions drawn on the GPU (nyxb_mvn_sample: counter-based stream keyed by (seed, run index), shard-invariant)
    std::vector<Spacecraft> generate_states_on_device(size_t skip, size_t num_runs, int32_t device = 0) const {
        const Spacecraft& t = nominal_state;
        const double tmpl[9] = {t.x_km, t.y_km, t.z_km, t.vx_km_s, t.vy_km_s, t.vz_km_s, t.coeff_reflectivity, t.coeff_drag, t.prop_mass_kg};
        double L[81] = {0};
        for (int i = 0; i < 9; ++i) L[i * 9 + i] = std_dev[i];
        std::vector<double> st(9 * num_runs);
        if (nyxb_mvn_sample(device, seed, skip, num_runs, tmpl, nullptr, L, st.data(), nullptr) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_mvn_sample: ") + nyxb_last_error());
        std::vector<int64_t> ep(num_runs, t.epoch_ns);
        std::vector<Spacecraft> out;
        for (size_t i = 0; i < num_runs; ++i) out.push_back(detail::unpack(t, st, ep, num_runs, i));
        return out;
    }
    Results run_until_epoch(const Propagator& prop, const Almanac* almanac, int64_t end_epoch_ns, size_t num_runs) const {
        return resume_run_until_epoch(prop, almanac, 0, end_epoch_ns, num_runs);
    }
    Results resume_run_until_epoch(const Propagator& prop, const Almanac* almanac, size_t skip, int64_t end_epoch_ns, size_t num_runs) const {
        auto init = generate_states(skip, num_runs);
        auto r = prop.propagate_batch(init, end_epoch_ns, almanac);
        Results res; res.scenario = scenario;
        for (size_t i = 0; i < num_runs; ++i) {
            res.total_steps += r.details[i].n_steps;
            if (r.status[i] & 0xff) res.runs.push_back(Run{i, init[i], PropagationError(r.status[i])});  // per-run error, never aborts (mc/results.rs:48-59)
            else res.runs.push_back(Run{i, init[i], detail::unpack(init[i], r.state, r.epoch, num_runs, i)});
        }
        return res;
    }
};


// ---------------------------------------------------------------------------------------------------------------------
// Orbit determination (SURVEY.md §8 (f)-2): n sequential Kalman filters over one tracking schedule in ONE launch.
// ---------------------------------------------------------------------------------------------------------------------
enum class MeasurementType : int32_t { Range = NYXB_MSR_RANGE, Doppler = NYXB_MSR_DOPPLER,           // od/msr/types.rs:31-45
                                       Azimuth = NYXB_MSR_AZIMUTH, Elevation = NYXB_MSR_ELEVATION,   // degrees (nyxb_aer_station)
                                       X = NYXB_MSR_X, Y = NYXB_MSR_Y, Z = NYXB_MSR_Z };              // position fixes
enum class KalmanVariant : int32_t { ReferenceUpdate = NYXB_KF_REFERENCE_UPDATE, DeviationTracking = NYXB_KF_DEVIATION_TRACKING };
struct StochasticNoise { double sigma = 0.0, bias_constant = 0.0; double covariance() const { return sigma * sigma; } };
struct SigmaRejection { double num_sigmas = 3.0; };                                                        // process/rejectcrit.rs:35-46

// GroundStation (od/ground_station/mod.rs:47-75; builtin.rs:25-117), instantaneous Range + Doppler, and Azimuth / Elevation added by
// with_msr_type (a station with angles runs through nyxb_od_aer_batch)
struct GroundStation {
    std::string name;
    double latitude_deg = 0, longitude_deg = 0, height_km = 0, elevation_mask_deg = 0;
    Frame frame = IAU_EARTH();
    std::vector<MeasurementType> measurement_types{MeasurementType::Range, MeasurementType::Doppler};
    StochasticNoise range_noise_km{2e-3, 0.0}, doppler_noise_km_s{3e-6, 0.0};
    StochasticNoise azimuth_noise_deg{}, elevation_noise_deg{};
    static GroundStation dss65_madrid(double mask, StochasticNoise r, StochasticNoise d) { return {"Madrid", 40.427222, 4.250556, 0.834939, mask, IAU_EARTH(), {MeasurementType::Range, MeasurementType::Doppler}, r, d}; }
    static GroundStation dss34_canberra(double mask, StochasticNoise r, StochasticNoise d) { return {"Canberra", -35.398333, 148.981944, 0.691750, mask, IAU_EARTH(), {MeasurementType::Range, MeasurementType::Doppler}, r, d}; }
    static GroundStation dss13_goldstone(double mask, StochasticNoise r, StochasticNoise d) { return {"Goldstone", 35.247164, 243.205, 1.07114904, mask, IAU_EARTH(), {MeasurementType::Range, MeasurementType::Doppler}, r, d}; }
    // geodetic -> body-fixed position and local zenith on the frame's ellipsoid (anise Orbit::try_latlongalt)
    void body_fixed(double pos[3], double up[3]) const {
        const double a = frame.mean_equatorial_radius_km, b = frame.polar_radius_km > 0 ? frame.polar_radius_km : a;
        const double e2 = 1.0 - (b * b) / (a * a), d2r = 3.14159265358979323846 / 180.0;
        const double sl = std::sin(latitude_deg * d2r), cl = std::cos(latitude_deg * d2r), so = std::sin(longitude_deg * d2r), co = std::cos(longitude_deg * d2r);
        const double nu = a / std::sqrt(1.0 - e2 * sl * sl);
        pos[0] = (nu + height_km) * cl * co; pos[1] = (nu + height_km) * cl * so; pos[2] = (nu * (1.0 - e2) + height_km) * sl;
        up[0] = cl * co; up[1] = cl * so; up[2] = sl;
    }
    // GroundStation::with_msr_type (ground_station/mod.rs:137-150): sets the type's noise, appends the type unless it is listed
    GroundStation& with_msr_type(MeasurementType t, StochasticNoise nz) {
        noise(t) = nz;
        if (std::find(measurement_types.begin(), measurement_types.end(), t) == measurement_types.end()) measurement_types.push_back(t);
        return *this;
    }
    StochasticNoise& noise(MeasurementType t) {
        switch (t) {
            case MeasurementType::Range: return range_noise_km;
            case MeasurementType::Doppler: return doppler_noise_km_s;
            case MeasurementType::Azimuth: return azimuth_noise_deg;
            case MeasurementType::Elevation: return elevation_noise_deg;
            default: throw std::runtime_error("a ground station measures Range, Doppler, Azimuth or Elevation");
        }
    }
    const StochasticNoise& noise(MeasurementType t) const { return const_cast<GroundStation*>(this)->noise(t); }
    bool has_angles() const {
        for (auto t : measurement_types) if (t == MeasurementType::Azimuth || t == MeasurementType::Elevation) return true;
        return false;
    }
    // the station for nyxb_od_aer_batch: the geometry of to_c plus the body-fixed geodetic north and east
    nyxb_aer_station to_aer_c(const Frame& integration_frame, int32_t body_index, double central_radius_km) const {
        if (measurement_types.empty() || measurement_types.size() > 4) throw std::runtime_error("a ground station carries one to four types");
        nyxb_aer_station g{};
        body_fixed(g.pos_fixed_km, g.up_fixed);
        const double d2r = 3.14159265358979323846 / 180.0;
        const double sl = std::sin(latitude_deg * d2r), cl = std::cos(latitude_deg * d2r), so = std::sin(longitude_deg * d2r), co = std::cos(longitude_deg * d2r);
        g.north_fixed[0] = -sl * co; g.north_fixed[1] = -sl * so; g.north_fixed[2] = cl;
        g.east_fixed[0] = -so; g.east_fixed[1] = co; g.east_fixed[2] = 0.0;
        g.elevation_mask_deg = elevation_mask_deg; g.rot = frame.rotation;
        const bool same = frame.ephemeris_id == integration_frame.ephemeris_id;
        g.body = same ? NYXB_CENTRAL_BODY : body_index;
        g.body_radius_km = same ? -1.0 : central_radius_km;
        g.n_types = (int32_t)measurement_types.size();
        for (int q = 0; q < g.n_types; ++q) {
            g.types[q] = (int32_t)measurement_types[q];
            const StochasticNoise& nz = noise(measurement_types[q]);
            g.noise_var[q] = nz.covariance(); g.bias[q] = nz.bias_constant;
        }
        return g;
    }
    nyxb_ground_station to_c(const Frame& integration_frame, int32_t body_index, double central_radius_km) const {
        nyxb_ground_station g{};
        body_fixed(g.pos_fixed_km, g.up_fixed);
        g.elevation_mask_deg = elevation_mask_deg; g.rot = frame.rotation;
        const bool same = frame.ephemeris_id == integration_frame.ephemeris_id;
        g.body = same ? NYXB_CENTRAL_BODY : body_index;
        g.body_radius_km = same ? -1.0 : central_radius_km;
        g.n_types = (int32_t)measurement_types.size();
        for (int q = 0; q < g.n_types && q < 2; ++q) {
            g.types[q] = (int32_t)measurement_types[q];
            const StochasticNoise& nz = measurement_types[q] == MeasurementType::Range ? range_noise_km : doppler_noise_km_s;
            g.noise_var[q] = nz.covariance(); g.bias[q] = nz.bias_constant;
        }
        return g;
    }
};

struct ProcessNoise3D {   // od/snc.rs:38-56, 118-134, 288-311
    double diag[3] = {0, 0, 0}; int64_t disable_time = 0; bool ric = false;
    static ProcessNoise3D from_diagonal(const double (&v)[3], int64_t disable, bool ric_frame = false) { ProcessNoise3D p; for (int i = 0; i < 3; ++i) p.diag[i] = v[i]; p.disable_time = disable; p.ric = ric_frame; return p; }
    static ProcessNoise3D from_velocity_km_s(const double (&v)[3], int64_t noise_duration, int64_t disable, bool ric_frame = false) {
        ProcessNoise3D p; for (int i = 0; i < 3; ++i) p.diag[i] = v[i] / ((double)noise_duration * 1e-9); p.disable_time = disable; p.ric = ric_frame; return p;
    }
};

struct KfEstimate {   // od/estimate/kfestimate.rs: nominal state + 9x9 covariance (row-major here) + state deviation
    Spacecraft nominal_state; double covar[81] = {0}; double state_deviation[9] = {0};
    static KfEstimate from_diag(const Spacecraft& s, const double (&d)[9]) { KfEstimate e; e.nominal_state = s; for (int i = 0; i < 9; ++i) e.covar[i * 9 + i] = d[i]; return e; }
};

// one tracking schedule, n observation sets: obs[(k*ns + slot)*n + i], NaN = type not in the measurement's data; ns = 2 (slot =
// Range / Doppler) for ground stations, 4 (slot = Range / Doppler / Azimuth / Elevation) for ground stations with angles, 3 (slot =
// type - X) for position fixes
struct TrackingDataArc { std::vector<int64_t> epoch_ns; std::vector<std::string> tracker; std::vector<double> obs; size_t n = 0; size_t ns = 2; };

// PositionDevice (od/position/mod.rs): X / Y / Z fixes of the position in the integration frame; with_noise appends the type to the
// device's list, as the reference builds it (the filter measures the component at the LIST position, H follows the type: nyxb.h)
struct PositionDevice {
    std::string name;
    std::vector<MeasurementType> measurement_types;
    std::vector<StochasticNoise> noises;   // per list position
    PositionDevice& with_noise(MeasurementType t, StochasticNoise nz) {
        for (size_t q = 0; q < measurement_types.size(); ++q) if (measurement_types[q] == t) { noises[q] = nz; return *this; }
        measurement_types.push_back(t); noises.push_back(nz); return *this;
    }
    nyxb_position_device to_c() const {
        if (measurement_types.empty() || measurement_types.size() > 3) throw std::runtime_error("a position device carries one to three types");
        nyxb_position_device d{};
        d.n_types = (int32_t)measurement_types.size();
        for (int q = 0; q < d.n_types; ++q) { d.types[q] = (int32_t)measurement_types[q]; d.noise_var[q] = noises[q].covariance(); d.bias[q] = noises[q].bias_constant; }
        return d;
    }
};

// Traj (md/trajectory/traj.rs) reduced to what the interlink needs: ascending epochs and (x, y, z, vx, vy, vz) per record in `frame`
struct Traj {
    std::optional<std::string> name;
    Frame frame = EARTH_J2000();
    std::vector<int64_t> epoch_ns;   // [k] ascending
    std::vector<double> state;       // [k][6]
    size_t size() const { return epoch_ns.size(); }
};

// InterlinkTxSpacecraft (od/interlink/trk_device.rs:37-260): a transmitter known by its recorded trajectory, measuring the range and
// Doppler of the filtered spacecraft (nyxb_interlink_tx in nyxb.h, with the reference's as-coded quirks).  Instantaneous measurements
// without aberration correction only, with the trajectory in the integration frame; `key` names the device in TrackingDataArc.tracker.
struct InterlinkTxSpacecraft {
    std::string key;
    Traj traj;
    std::vector<MeasurementType> measurement_types;
    std::vector<StochasticNoise> noises;   // per list position
    std::optional<int64_t> integration_time;
    std::optional<std::string> ab_corr;
    std::string name() const { return traj.name ? *traj.name : "unnamed"; }   // trk_device.rs:93-95
    nyxb_interlink_tx to_c(int32_t column, const Frame& integration_frame) const {
        if (integration_time) throw std::runtime_error("interlink: integrated (two-way) measurements are not supported");
        if (ab_corr) throw std::runtime_error("interlink: aberration correction is not supported (ab_corr must be None)");
        if (traj.frame.ephemeris_id != integration_frame.ephemeris_id || traj.frame.rotation.kind != integration_frame.rotation.kind)
            throw std::runtime_error("interlink: the transmitter's trajectory is not in the integration frame");
        if (traj.size() == 0) throw std::runtime_error("interlink: the transmitter's trajectory is empty");
        if (measurement_types.empty() || measurement_types.size() > 2 || noises.size() != measurement_types.size())
            throw std::runtime_error("an interlink carries one or two of {Range, Doppler}, each with its noise");
        nyxb_interlink_tx d{};
        d.tx = column; d.n_types = (int32_t)measurement_types.size();
        for (int q = 0; q < d.n_types; ++q) {
            const MeasurementType t = measurement_types[q];
            if (t != MeasurementType::Range && t != MeasurementType::Doppler) throw std::runtime_error("an interlink carries Range and Doppler only");
            if (q == 1 && t == measurement_types[0]) throw std::runtime_error("an interlink carries distinct types");
            d.types[q] = (int32_t)t; d.noise_var[q] = noises[q].covariance(); d.bias[q] = noises[q].bias_constant;
        }
        d.body_radius_km = integration_frame.mean_equatorial_radius_km;
        return d;
    }
};

class KalmanODProcess;
class PositionKalmanODProcess;
class InterlinkKalmanODProcess;

struct ODSolution {
    size_t n = 0, m = 0, ns = 2;   // ns: observation slots, 2 (ground stations), 4 (ground stations with angles) or 3 (position fixes)
    std::vector<double> state, covar, state_dev, resid_ratio, prefit, postfit;   // [9][n], [81][n] (c*9+r), [9][n], [m][ns][n] x3
    std::vector<int64_t> epoch; std::vector<int32_t> msr_flags, status; std::vector<nyxb_details> details;
    // every estimate (ODSolution.estimates) when process_arcs ran with an estimates capacity (nyxb_od_records): epoch / tag
    // [cap][n], nominal / deviation [cap][9][n], covar / stm [cap][81][n] with (r, c) at [(k*81 + c*9 + r)*n + i], count [n]
    int64_t rec_capacity = 0;
    std::vector<int64_t> rec_epoch, rec_tag, rec_count;
    std::vector<double> rec_nominal, rec_deviation, rec_covar, rec_stm;
    // set by smooth(): smoothed state() / deviation / filter-smoother ratios [cap][9][n], covar [cap][81][n], postfit [cap][ns][n]
    // by estimate position (NaN where the reference has None), and the status of each filter's smoothing
    Frame frame = EARTH_J2000();   // integration frame of the run
    bool smoother_run = false;
    std::vector<double> sm_state, sm_deviation, sm_covar, sm_fs_ratio, sm_postfit;
    std::vector<int32_t> sm_status;
    Spacecraft final_state(const Spacecraft& tmpl, size_t i) const { return detail::unpack(tmpl, state, epoch, n, i); }
    int64_t n_estimates(size_t i) const { return rec_count.empty() ? 0 : std::min(rec_count[i], rec_capacity); }
    bool is_smoother_run() const { return smoother_run; }
    // ODSolution::smooth (od/process/solution/smooth.rs:104-249) of all n filters in one launch; `odp` and `arc` are those of the run
    // (an arc of four slots: nyxb_od_aer_smooth_batch)
    inline ODSolution smooth(const KalmanODProcess& odp, const TrackingDataArc& arc) const;
    // the same for position fixes (nyxb_od_position_smooth_batch; sm_postfit [cap][3][n])
    inline ODSolution smooth(const PositionKalmanODProcess& odp, const TrackingDataArc& arc) const;
    // the same for interlink transmitters (nyxb_od_interlink_smooth_batch; sm_postfit [cap][2][n])
    inline ODSolution smooth(const InterlinkKalmanODProcess& odp, const TrackingDataArc& arc) const;
};

// Covariance mapping of one estimate (KalmanODProcess::predict_until): record k at epoch0 + k * max_step, k < count
struct PredictionSolution {
    int64_t epoch0 = 0, max_step = 0, count = 0;
    std::vector<double> rec_state, rec_covar;   // [count][9] estimate.state(), [count][81] (c*9+r)
    double state[9] = {0}, covar[81] = {0}, state_dev[9] = {0};   // final nominal state, covariance (c*9+r), deviation
    int64_t epoch = 0; int32_t status = 0; nyxb_details details{};
    int64_t record_epoch(int64_t k) const { return epoch0 + k * max_step; }
    double record_covar(int64_t k, int r, int c) const { return rec_covar[(size_t)k * 81 + c * 9 + r]; }
};

namespace detail {
inline nyxb_od_config od_config(KalmanVariant variant, const std::optional<SigmaRejection>& rej, const std::optional<ProcessNoise3D>& snc,
                                int64_t max_step, int64_t epoch_precision, int32_t msr_size) {
    nyxb_od_config cfg{};
    cfg.variant = (int32_t)variant; cfg.msr_size = msr_size; cfg.reject_num_sigmas = rej ? rej->num_sigmas : -1.0;
    cfg.max_step_ns = max_step; cfg.epoch_precision_ns = epoch_precision;
    if (snc) { cfg.snc_enabled = 1; cfg.snc_frame = snc->ric ? 1 : 0; for (int i = 0; i < 3; ++i) cfg.snc_diag[i] = snc->diag[i]; cfg.snc_disable_time_ns = snc->disable_time; }
    return cfg;
}
// the index of the station's body in the almanac, or NYXB_CENTRAL_BODY; a station on another body than the integration centre needs
// its ephemeris
inline int32_t station_body(const GroundStation& d, const Frame& frame, const Almanac* almanac) {
    if (d.frame.ephemeris_id == frame.ephemeris_id) return NYXB_CENTRAL_BODY;
    if (!almanac) throw std::runtime_error("an almanac with the station's body is needed");
    for (size_t j = 0; j < almanac->bodies.size(); ++j) if (almanac->bodies[j].ephemeris_id == d.frame.ephemeris_id) return (int32_t)j;
    throw std::runtime_error("no ephemeris loaded for the station's body");
}
// the devices as nyxb_ground_station, in order
inline std::vector<nyxb_ground_station> pack_stations(const std::vector<GroundStation>& devices, const Frame& frame, const Almanac* almanac) {
    std::vector<nyxb_ground_station> st;
    for (auto& d : devices) st.push_back(d.to_c(frame, station_body(d, frame, almanac), frame.mean_equatorial_radius_km));
    return st;
}
// the devices as nyxb_aer_station, in order (nyxb_od_aer_batch)
inline std::vector<nyxb_aer_station> pack_aer_stations(const std::vector<GroundStation>& devices, const Frame& frame, const Almanac* almanac) {
    std::vector<nyxb_aer_station> st;
    for (auto& d : devices) st.push_back(d.to_aer_c(frame, station_body(d, frame, almanac), frame.mean_equatorial_radius_km));
    return st;
}
// the observation slots of a ground-station arc: 4 runs through nyxb_od_aer_batch, 2 through nyxb_od_ekf_batch, which takes no angles
inline size_t station_slots(const std::vector<GroundStation>& devices, const TrackingDataArc& arc) {
    if (arc.ns == 4) return 4;
    for (auto& d : devices)
        if (d.has_angles()) throw std::runtime_error("stations that measure azimuth or elevation need an arc of four slots (Range, Doppler, Azimuth, Elevation)");
    return 2;
}
// the solution's record arrays for estimates_capacity records of each filter and the nyxb_od_records pointing at them (empty for a
// negative capacity: no records)
inline nyxb_od_records alloc_records(ODSolution& s, int64_t estimates_capacity) {
    if (estimates_capacity < 0) return nyxb_od_records{};
    const size_t cap = (size_t)estimates_capacity, n = s.n;
    s.rec_capacity = estimates_capacity;
    s.rec_epoch.resize(cap * n); s.rec_tag.resize(cap * n); s.rec_count.resize(n);
    s.rec_nominal.resize(cap * 9 * n); s.rec_deviation.resize(cap * 9 * n); s.rec_covar.resize(cap * 81 * n); s.rec_stm.resize(cap * 81 * n);
    return nyxb_od_records{estimates_capacity, s.rec_epoch.data(), s.rec_tag.data(), s.rec_nominal.data(), s.rec_deviation.data(), s.rec_covar.data(),
                           s.rec_stm.data(), s.rec_count.data()};
}
// index of each measurement's tracker in `devices`; -1 for an unknown tracker
inline std::vector<int32_t> tracker_index(const std::vector<GroundStation>& devices, const TrackingDataArc& arc) {
    std::vector<int32_t> trk(arc.epoch_ns.size());
    for (size_t k = 0; k < trk.size(); ++k) { trk[k] = -1; for (size_t j = 0; j < devices.size(); ++j) if (devices[j].name == arc.tracker[k]) trk[k] = (int32_t)j; }
    return trk;
}
}  // namespace detail

// KalmanODProcess (od/process/{initializers.rs:60-113, mod.rs:128-497}); msr_size 2 = SpacecraftKalmanOD, 1 = SpacecraftKalmanScalarOD
class KalmanODProcess {
  public:
    Propagator prop; KalmanVariant variant; std::optional<SigmaRejection> sigma_reject; std::vector<GroundStation> devices;
    const Almanac* almanac = nullptr; std::optional<ProcessNoise3D> process_noise;
    int64_t max_step = 60 * NS_PER_S, epoch_precision = 1000; int32_t msr_size = 2;
    KalmanODProcess(Propagator p, KalmanVariant v, std::optional<SigmaRejection> rej, std::vector<GroundStation> dev, const Almanac* alm = nullptr, int32_t msr = 2)
        : prop(std::move(p)), variant(v), sigma_reject(rej), devices(std::move(dev)), almanac(alm), msr_size(msr) {}
    KalmanODProcess& with_process_noise(ProcessNoise3D snc) { process_noise = snc; return *this; }

    nyxb_od_config config() const { return detail::od_config(variant, sigma_reject, process_noise, max_step, epoch_precision, msr_size); }

    // KalmanODProcess::predict_until / predict_for (od/process/mod.rs:440-496): every record of the time updates
    PredictionSolution predict_until(const KfEstimate& initial, int64_t end_epoch) const {
        const Frame& frame = initial.nominal_state.frame;
        auto eng = detail::make_engine(prop.dynamics, frame, almanac, prop.method, prop.opts, prop.mode, prop.device);
        detail::Soa soa(std::vector<Spacecraft>{initial.nominal_state});
        const nyxb_od_config cfg = config();
        if (cfg.max_step_ns <= 0) throw std::runtime_error("StepSize: max_step must be positive");
        double cov0[81];
        for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) cov0[c * 9 + r] = initial.covar[r * 9 + c];
        const int64_t epoch0 = soa.epoch[0], span = end_epoch - epoch0;
        const int64_t cap = 1 + (span > 0 ? (span + max_step - 1) / max_step : 1);
        PredictionSolution s; s.epoch0 = epoch0; s.max_step = max_step;
        s.rec_state.resize((size_t)cap * 9); s.rec_covar.resize((size_t)cap * 81);
        nyxb_predict_outputs out{s.state, &s.epoch, s.covar, s.state_dev, &s.details, &s.status, cap, s.rec_state.data(), s.rec_covar.data(), &s.count};
        if (nyxb_od_predict_batch(eng.get(), &cfg, 1, soa.state.data(), soa.consts.data(), soa.epoch.data(), &end_epoch, cov0,
                                  initial.state_deviation, &out) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_predict_batch: ") + nyxb_last_error());
        if (s.count > cap) s.count = cap;
        s.rec_state.resize((size_t)s.count * 9); s.rec_covar.resize((size_t)s.count * 81);
        return s;
    }
    PredictionSolution predict_for(const KfEstimate& initial, int64_t duration) const {
        return predict_until(initial, initial.nominal_state.epoch() + duration);
    }

    // estimates_capacity >= 0: also record the first estimates_capacity entries of each filter's ODSolution.estimates
    // (nyxb_od_ekf_record_batch); the filter's outputs are the same bits.  An arc of four slots (arc.ns = 4: Range, Doppler, Azimuth,
    // Elevation) runs through nyxb_od_aer_batch, with record tags NYXB_OD_POS_TAG; stations with angles need one.
    ODSolution process_arcs(const std::vector<KfEstimate>& initial, const TrackingDataArc& arc, int64_t estimates_capacity = -1) const {
        const size_t n = initial.size(), m = arc.epoch_ns.size();
        const size_t ns = detail::station_slots(devices, arc);
        if (arc.n != n || arc.obs.size() != m * ns * n || arc.tracker.size() != m) throw std::runtime_error("arc shape does not match the filters");
        std::vector<Spacecraft> noms; for (auto& e : initial) noms.push_back(e.nominal_state);
        const Frame& frame = noms.at(0).frame;
        auto eng = detail::make_engine(prop.dynamics, frame, almanac, prop.method, prop.opts, prop.mode, prop.device);
        detail::Soa soa(noms);
        std::vector<double> cov0(81 * n);
        for (size_t i = 0; i < n; ++i) for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) cov0[(size_t)(c * 9 + r) * n + i] = initial[i].covar[r * 9 + c];
        std::vector<int32_t> trk = detail::tracker_index(devices, arc);
        const nyxb_od_config cfg = config();
        nyxb_tracking_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
        ODSolution s; s.n = n; s.m = m; s.ns = ns; s.frame = frame;
        s.state.resize(9 * n); s.epoch.resize(n); s.covar.resize(81 * n); s.state_dev.resize(9 * n); s.resid_ratio.resize(m * ns * n); s.prefit.resize(m * ns * n);
        s.postfit.resize(m * ns * n); s.msr_flags.resize(m * n); s.details.resize(n); s.status.resize(n);
        nyxb_od_outputs out{s.state.data(), s.epoch.data(), s.covar.data(), s.state_dev.data(), s.resid_ratio.data(), s.prefit.data(), s.postfit.data(),
                            s.msr_flags.data(), nullptr, nullptr, s.details.data(), s.status.data()};
        if (ns == 4) {
            const std::vector<nyxb_aer_station> ast = detail::pack_aer_stations(devices, frame, almanac);
            nyxb_od_records rec = detail::alloc_records(s, estimates_capacity);
            if (nyxb_od_aer_batch(eng.get(), &cfg, (int32_t)ast.size(), ast.data(), &carc, n, soa.state.data(), soa.consts.data(), soa.epoch.data(),
                                  cov0.data(), &out, estimates_capacity >= 0 ? &rec : nullptr) != NYXB_RC_OK)
                throw std::runtime_error(std::string("nyxb_od_aer_batch: ") + nyxb_last_error());
            return s;
        }
        std::vector<nyxb_ground_station> st = detail::pack_stations(devices, frame, almanac);
        if (estimates_capacity < 0) {
            if (nyxb_od_ekf_batch(eng.get(), &cfg, (int32_t)st.size(), st.data(), &carc, n, soa.state.data(), soa.consts.data(), soa.epoch.data(), cov0.data(), &out) != NYXB_RC_OK)
                throw std::runtime_error(std::string("nyxb_od_ekf_batch: ") + nyxb_last_error());
            return s;
        }
        nyxb_od_records rec = detail::alloc_records(s, estimates_capacity);
        if (nyxb_od_ekf_record_batch(eng.get(), &cfg, (int32_t)st.size(), st.data(), &carc, n, soa.state.data(), soa.consts.data(), soa.epoch.data(),
                                     cov0.data(), &out, &rec) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_ekf_record_batch: ") + nyxb_last_error());
        return s;
    }
};

inline ODSolution ODSolution::smooth(const KalmanODProcess& odp, const TrackingDataArc& arc) const {
    if (rec_count.empty()) throw std::runtime_error("no estimate records: run process_arcs(.., estimates_capacity)");
    if (smoother_run) throw std::runtime_error("already smoothed");
    // the engine of the filter run (its dynamics and integration frame) supplies the stations' ephemerides
    const Frame& integ = frame;
    auto eng = detail::make_engine(odp.prop.dynamics, integ, odp.almanac, odp.prop.method, odp.prop.opts, odp.prop.mode, odp.prop.device);
    const size_t slots = detail::station_slots(odp.devices, arc);
    std::vector<int32_t> trk = detail::tracker_index(odp.devices, arc);
    const nyxb_od_config cfg = odp.config();
    nyxb_tracking_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
    nyxb_od_records rec{rec_capacity, const_cast<int64_t*>(rec_epoch.data()), const_cast<int64_t*>(rec_tag.data()), const_cast<double*>(rec_nominal.data()),
                        const_cast<double*>(rec_deviation.data()), const_cast<double*>(rec_covar.data()), const_cast<double*>(rec_stm.data()),
                        const_cast<int64_t*>(rec_count.data())};
    ODSolution s = *this;
    const size_t cap = (size_t)rec_capacity;
    s.smoother_run = true;
    s.sm_state.resize(cap * 9 * n); s.sm_deviation.resize(cap * 9 * n); s.sm_covar.resize(cap * 81 * n); s.sm_fs_ratio.resize(cap * 9 * n);
    s.sm_postfit.resize(cap * slots * n); s.sm_status.resize(n);
    nyxb_smooth_outputs out{s.sm_state.data(), s.sm_deviation.data(), s.sm_covar.data(), s.sm_fs_ratio.data(), s.sm_postfit.data(), s.sm_status.data()};
    if (slots == 4) {
        const std::vector<nyxb_aer_station> ast = detail::pack_aer_stations(odp.devices, integ, odp.almanac);
        if (nyxb_od_aer_smooth_batch(eng.get(), &cfg, (int32_t)ast.size(), ast.data(), &carc, n, &rec, status.data(), &out) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_aer_smooth_batch: ") + nyxb_last_error());
        return s;
    }
    std::vector<nyxb_ground_station> st = detail::pack_stations(odp.devices, integ, odp.almanac);
    if (nyxb_od_smooth_batch(eng.get(), &cfg, (int32_t)st.size(), st.data(), &carc, n, &rec, status.data(), &out) != NYXB_RC_OK)
        throw std::runtime_error(std::string("nyxb_od_smooth_batch: ") + nyxb_last_error());
    return s;
}

// KalmanODProcess<.., PositionDevice> (od/process/mod.rs:128-497 with od/position): the filter over position fixes, msr_size 1 to 3
class PositionKalmanODProcess {
  public:
    Propagator prop; KalmanVariant variant; std::optional<SigmaRejection> sigma_reject; std::vector<PositionDevice> devices;
    const Almanac* almanac = nullptr; std::optional<ProcessNoise3D> process_noise;
    int64_t max_step = 60 * NS_PER_S, epoch_precision = 1000; int32_t msr_size = 3;
    PositionKalmanODProcess(Propagator p, KalmanVariant v, std::optional<SigmaRejection> rej, std::vector<PositionDevice> dev, int32_t msr = 3)
        : prop(std::move(p)), variant(v), sigma_reject(rej), devices(std::move(dev)), msr_size(msr) {}
    PositionKalmanODProcess& with_process_noise(ProcessNoise3D snc) { process_noise = snc; return *this; }
    nyxb_od_config config() const { return detail::od_config(variant, sigma_reject, process_noise, max_step, epoch_precision, msr_size); }
    std::vector<nyxb_position_device> devices_c() const { std::vector<nyxb_position_device> d; for (auto& x : devices) d.push_back(x.to_c()); return d; }
    std::vector<int32_t> tracker_index(const TrackingDataArc& arc) const {
        std::vector<int32_t> trk(arc.epoch_ns.size());
        for (size_t k = 0; k < trk.size(); ++k) { trk[k] = -1; for (size_t j = 0; j < devices.size(); ++j) if (devices[j].name == arc.tracker[k]) trk[k] = (int32_t)j; }
        return trk;
    }

    // arc.ns must be 3; estimates_capacity >= 0 also records the estimates (tags NYXB_OD_POS_TAG), with the same filter outputs
    ODSolution process_arcs(const std::vector<KfEstimate>& initial, const TrackingDataArc& arc, int64_t estimates_capacity = -1) const {
        const size_t n = initial.size(), m = arc.epoch_ns.size();
        if (arc.ns != 3 || arc.n != n || arc.obs.size() != m * 3 * n || arc.tracker.size() != m) throw std::runtime_error("arc shape does not match the filters");
        std::vector<Spacecraft> noms; for (auto& e : initial) noms.push_back(e.nominal_state);
        const Frame& frame = noms.at(0).frame;
        auto eng = detail::make_engine(prop.dynamics, frame, almanac, prop.method, prop.opts, prop.mode, prop.device);
        detail::Soa soa(noms);
        std::vector<double> cov0(81 * n);
        for (size_t i = 0; i < n; ++i) for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) cov0[(size_t)(c * 9 + r) * n + i] = initial[i].covar[r * 9 + c];
        const std::vector<nyxb_position_device> dev = devices_c();
        std::vector<int32_t> trk = tracker_index(arc);
        const nyxb_od_config cfg = config();
        nyxb_position_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
        ODSolution s; s.n = n; s.m = m; s.ns = 3; s.frame = frame;
        s.state.resize(9 * n); s.epoch.resize(n); s.covar.resize(81 * n); s.state_dev.resize(9 * n); s.resid_ratio.resize(m * 3 * n); s.prefit.resize(m * 3 * n);
        s.postfit.resize(m * 3 * n); s.msr_flags.resize(m * n); s.details.resize(n); s.status.resize(n);
        nyxb_od_outputs out{s.state.data(), s.epoch.data(), s.covar.data(), s.state_dev.data(), s.resid_ratio.data(), s.prefit.data(), s.postfit.data(),
                            s.msr_flags.data(), nullptr, nullptr, s.details.data(), s.status.data()};
        nyxb_od_records rec = detail::alloc_records(s, estimates_capacity);
        if (nyxb_od_position_batch(eng.get(), &cfg, (int32_t)dev.size(), dev.data(), &carc, n, soa.state.data(), soa.consts.data(), soa.epoch.data(),
                                   cov0.data(), &out, estimates_capacity >= 0 ? &rec : nullptr) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_position_batch: ") + nyxb_last_error());
        return s;
    }
};

inline ODSolution ODSolution::smooth(const PositionKalmanODProcess& odp, const TrackingDataArc& arc) const {
    if (rec_count.empty()) throw std::runtime_error("no estimate records: run process_arcs(.., estimates_capacity)");
    if (smoother_run) throw std::runtime_error("already smoothed");
    auto eng = detail::make_engine(odp.prop.dynamics, frame, odp.almanac, odp.prop.method, odp.prop.opts, odp.prop.mode, odp.prop.device);
    const std::vector<nyxb_position_device> dev = odp.devices_c();
    std::vector<int32_t> trk = odp.tracker_index(arc);
    const nyxb_od_config cfg = odp.config();
    nyxb_position_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
    nyxb_od_records rec{rec_capacity, const_cast<int64_t*>(rec_epoch.data()), const_cast<int64_t*>(rec_tag.data()), const_cast<double*>(rec_nominal.data()),
                        const_cast<double*>(rec_deviation.data()), const_cast<double*>(rec_covar.data()), const_cast<double*>(rec_stm.data()),
                        const_cast<int64_t*>(rec_count.data())};
    ODSolution s = *this;
    const size_t cap = (size_t)rec_capacity;
    s.smoother_run = true;
    s.sm_state.resize(cap * 9 * n); s.sm_deviation.resize(cap * 9 * n); s.sm_covar.resize(cap * 81 * n); s.sm_fs_ratio.resize(cap * 9 * n);
    s.sm_postfit.resize(cap * 3 * n); s.sm_status.resize(n);
    nyxb_smooth_outputs out{s.sm_state.data(), s.sm_deviation.data(), s.sm_covar.data(), s.sm_fs_ratio.data(), s.sm_postfit.data(), s.sm_status.data()};
    if (nyxb_od_position_smooth_batch(eng.get(), &cfg, (int32_t)dev.size(), dev.data(), &carc, n, &rec, status.data(), &out) != NYXB_RC_OK)
        throw std::runtime_error(std::string("nyxb_od_position_smooth_batch: ") + nyxb_last_error());
    return s;
}

// KalmanODProcess<.., InterlinkTxSpacecraft> (od/process/mod.rs:128-497 with od/interlink): the filter over interlink transmitters,
// msr_size 1 or 2, on a two-slot arc (slot = Range / Doppler).  Each device's trajectory is one column of the recordings handed to
// nyxb_od_interlink_batch; record tags NYXB_OD_TAG.
class InterlinkKalmanODProcess {
  public:
    Propagator prop; KalmanVariant variant; std::optional<SigmaRejection> sigma_reject; std::vector<InterlinkTxSpacecraft> devices;
    const Almanac* almanac = nullptr; std::optional<ProcessNoise3D> process_noise;
    int64_t max_step = 60 * NS_PER_S, epoch_precision = 1000; int32_t msr_size = 2;
    InterlinkKalmanODProcess(Propagator p, KalmanVariant v, std::optional<SigmaRejection> rej, std::vector<InterlinkTxSpacecraft> dev,
                             const Almanac* alm = nullptr, int32_t msr = 2)
        : prop(std::move(p)), variant(v), sigma_reject(rej), devices(std::move(dev)), almanac(alm), msr_size(msr) {}
    InterlinkKalmanODProcess& with_process_noise(ProcessNoise3D snc) { process_noise = snc; return *this; }
    nyxb_od_config config() const { return detail::od_config(variant, sigma_reject, process_noise, max_step, epoch_precision, msr_size); }
    std::vector<int32_t> tracker_index(const TrackingDataArc& arc) const {
        std::vector<int32_t> trk(arc.epoch_ns.size());
        for (size_t k = 0; k < trk.size(); ++k) { trk[k] = -1; for (size_t j = 0; j < devices.size(); ++j) if (devices[j].key == arc.tracker[k]) trk[k] = (int32_t)j; }
        return trk;
    }
    // the devices (device j reads column j) and their recordings as a host-pointer nyxb_traj_sink over the struct's own arrays
    struct Links {
        std::vector<nyxb_interlink_tx> dev; std::vector<int64_t> epoch, count; std::vector<double> state; nyxb_traj_sink sink{};
    };
    Links links(const Frame& frame) const {
        Links l;
        const size_t ntx = devices.size();
        size_t cap = 0;
        for (auto& d : devices) cap = std::max(cap, d.traj.size());
        l.epoch.assign(cap * ntx, 0); l.state.assign(6 * cap * ntx, 0.0); l.count.assign(ntx, 0);
        for (size_t j = 0; j < ntx; ++j) {
            const Traj& t = devices[j].traj;
            l.dev.push_back(devices[j].to_c((int32_t)j, frame));
            l.count[j] = (int64_t)t.size();
            for (size_t s = 0; s < t.size(); ++s) {
                l.epoch[s * ntx + j] = t.epoch_ns[s];
                for (int c = 0; c < 6; ++c) l.state[((size_t)c * cap + s) * ntx + j] = t.state[s * 6 + c];
            }
        }
        l.sink = nyxb_traj_sink{(int64_t)cap, l.epoch.data(), l.state.data(), l.count.data()};
        return l;
    }

    // arc.ns must be 2; estimates_capacity >= 0 also records the estimates (tags NYXB_OD_TAG), with the same filter outputs
    ODSolution process_arcs(const std::vector<KfEstimate>& initial, const TrackingDataArc& arc, int64_t estimates_capacity = -1) const {
        const size_t n = initial.size(), m = arc.epoch_ns.size();
        if (arc.ns != 2 || arc.n != n || arc.obs.size() != m * 2 * n || arc.tracker.size() != m)
            throw std::runtime_error("interlink devices need a two-slot arc (Range, Doppler) matching the filters");
        std::vector<Spacecraft> noms; for (auto& e : initial) noms.push_back(e.nominal_state);
        const Frame& frame = noms.at(0).frame;
        const Links l = links(frame);
        auto eng = detail::make_engine(prop.dynamics, frame, almanac, prop.method, prop.opts, prop.mode, prop.device);
        detail::Soa soa(noms);
        std::vector<double> cov0(81 * n);
        for (size_t i = 0; i < n; ++i) for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) cov0[(size_t)(c * 9 + r) * n + i] = initial[i].covar[r * 9 + c];
        std::vector<int32_t> trk = tracker_index(arc);
        const nyxb_od_config cfg = config();
        nyxb_tracking_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
        ODSolution s; s.n = n; s.m = m; s.ns = 2; s.frame = frame;
        s.state.resize(9 * n); s.epoch.resize(n); s.covar.resize(81 * n); s.state_dev.resize(9 * n); s.resid_ratio.resize(m * 2 * n); s.prefit.resize(m * 2 * n);
        s.postfit.resize(m * 2 * n); s.msr_flags.resize(m * n); s.details.resize(n); s.status.resize(n);
        nyxb_od_outputs out{s.state.data(), s.epoch.data(), s.covar.data(), s.state_dev.data(), s.resid_ratio.data(), s.prefit.data(), s.postfit.data(),
                            s.msr_flags.data(), nullptr, nullptr, s.details.data(), s.status.data()};
        nyxb_od_records rec = detail::alloc_records(s, estimates_capacity);
        if (nyxb_od_interlink_batch(eng.get(), &cfg, (int32_t)l.dev.size(), l.dev.data(), l.dev.size(), &l.sink, &carc, n, soa.state.data(),
                                    soa.consts.data(), soa.epoch.data(), cov0.data(), &out, estimates_capacity >= 0 ? &rec : nullptr) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_interlink_batch: ") + nyxb_last_error());
        return s;
    }
};

inline ODSolution ODSolution::smooth(const InterlinkKalmanODProcess& odp, const TrackingDataArc& arc) const {
    if (rec_count.empty()) throw std::runtime_error("no estimate records: run process_arcs(.., estimates_capacity)");
    if (smoother_run) throw std::runtime_error("already smoothed");
    auto eng = detail::make_engine(odp.prop.dynamics, frame, odp.almanac, odp.prop.method, odp.prop.opts, odp.prop.mode, odp.prop.device);
    const InterlinkKalmanODProcess::Links l = odp.links(frame);
    std::vector<int32_t> trk = odp.tracker_index(arc);
    const nyxb_od_config cfg = odp.config();
    nyxb_tracking_arc carc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
    nyxb_od_records rec{rec_capacity, const_cast<int64_t*>(rec_epoch.data()), const_cast<int64_t*>(rec_tag.data()), const_cast<double*>(rec_nominal.data()),
                        const_cast<double*>(rec_deviation.data()), const_cast<double*>(rec_covar.data()), const_cast<double*>(rec_stm.data()),
                        const_cast<int64_t*>(rec_count.data())};
    ODSolution s = *this;
    const size_t cap = (size_t)rec_capacity;
    s.smoother_run = true;
    s.sm_state.resize(cap * 9 * n); s.sm_deviation.resize(cap * 9 * n); s.sm_covar.resize(cap * 81 * n); s.sm_fs_ratio.resize(cap * 9 * n);
    s.sm_postfit.resize(cap * 2 * n); s.sm_status.resize(n);
    nyxb_smooth_outputs out{s.sm_state.data(), s.sm_deviation.data(), s.sm_covar.data(), s.sm_fs_ratio.data(), s.sm_postfit.data(), s.sm_status.data()};
    if (nyxb_od_interlink_smooth_batch(eng.get(), &cfg, (int32_t)l.dev.size(), l.dev.data(), l.dev.size(), &l.sink, &carc, n, &rec, status.data(),
                                       &out) != NYXB_RC_OK)
        throw std::runtime_error(std::string("nyxb_od_interlink_smooth_batch: ") + nyxb_last_error());
    return s;
}

// BatchLeastSquares (od/blse/mod.rs:30-541) with the reference's builder defaults; estimate / evaluate of one problem through
// nyxb_od_bls_batch / nyxb_od_bls_evaluate_batch.  A per-problem status is thrown as the reference's ODError.
enum class BLSSolver : int32_t { NormalEquations = NYXB_BLS_NORMAL_EQUATIONS, LevenbergMarquardt = NYXB_BLS_LEVENBERG_MARQUARDT };

struct BLSSolution {   // od/blse/solution.rs
    Spacecraft estimated_state; double covariance[81] = {0};   // row-major
    int32_t num_iterations = 0; double final_rms = 0.0, final_corr_pos_km = 0.0; bool converged = false;
    nyxb_details details{};
    // From<BLSSolution> for KfEstimate (solution.rs:75-93): the Cr, Cd and mass variances zeroed
    KfEstimate to_kf_estimate() const {
        KfEstimate e; e.nominal_state = estimated_state;
        for (int q = 0; q < 81; ++q) e.covar[q] = covariance[q];
        e.covar[60] = e.covar[70] = e.covar[80] = 0.0;
        return e;
    }
};

class BatchLeastSquares {
  public:
    Propagator prop; std::vector<GroundStation> devices; const Almanac* almanac = nullptr;
    BLSSolver solver = BLSSolver::NormalEquations;
    double tolerance_pos_km = 1e-4; int32_t max_iterations = 10;
    int64_t max_step = 30 * NS_PER_S, epoch_precision = 1000;
    double lm_lambda_init = 10.0, lm_lambda_decrease = 10.0, lm_lambda_increase = 10.0, lm_lambda_min = 1e-12, lm_lambda_max = 1e12;
    bool lm_use_diag_scaling = true;
    BatchLeastSquares(Propagator p, std::vector<GroundStation> dev, const Almanac* alm = nullptr) : prop(std::move(p)), devices(std::move(dev)), almanac(alm) {}

    nyxb_bls_config config() const {
        nyxb_bls_config c{};
        c.solver = (int32_t)solver; c.max_iterations = max_iterations; c.tolerance_pos_km = tolerance_pos_km;
        c.max_step_ns = max_step; c.epoch_precision_ns = epoch_precision;
        c.lm_lambda_init = lm_lambda_init; c.lm_lambda_decrease = lm_lambda_decrease; c.lm_lambda_increase = lm_lambda_increase;
        c.lm_lambda_min = lm_lambda_min; c.lm_lambda_max = lm_lambda_max; c.lm_use_diag_scaling = lm_use_diag_scaling ? 1 : 0;
        return c;
    }

    // BatchLeastSquares::estimate (od/blse/mod.rs:146-446); arc with one observation set
    BLSSolution estimate(const Spacecraft& guess, const TrackingDataArc& arc) const {
        Ctx c(*this, guess, arc);
        BLSSolution s; s.estimated_state = guess;
        double state[9], cov[81], rms = 0.0, corr = 0.0; int64_t epoch = 0; int32_t iters = 0, conv = 0, status = 0;
        nyxb_bls_outputs out{state, &epoch, cov, &iters, &rms, &corr, &conv, &s.details, &status};
        if (nyxb_od_bls_batch(c.eng.get(), &c.cfg, (int32_t)c.st.size(), c.st.data(), &c.carc, 1, c.soa.state.data(), c.soa.consts.data(),
                              c.soa.epoch.data(), &out) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_bls_batch: ") + nyxb_last_error());
        throw_status(status);
        s.estimated_state = detail::unpack(guess, std::vector<double>(state, state + 9), std::vector<int64_t>{epoch}, 1, 0);
        for (int r = 0; r < 9; ++r) for (int q = 0; q < 9; ++q) s.covariance[r * 9 + q] = cov[q * 9 + r];
        s.num_iterations = iters; s.final_rms = rms; s.final_corr_pos_km = corr; s.converged = conv != 0;
        return s;
    }

    // BatchLeastSquares::evaluate (od/blse/mod.rs:450-541)
    double evaluate(const Spacecraft& state, const TrackingDataArc& arc) const {
        Ctx c(*this, state, arc);
        double rms = 0.0; int32_t status = 0;
        if (nyxb_od_bls_evaluate_batch(c.eng.get(), &c.cfg, (int32_t)c.st.size(), c.st.data(), &c.carc, 1, c.soa.state.data(), c.soa.consts.data(),
                                       c.soa.epoch.data(), &rms, &status) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_od_bls_evaluate_batch: ") + nyxb_last_error());
        throw_status(status);
        return rms;
    }

  private:
    struct Ctx {
        detail::Soa soa; detail::EnginePtr eng;
        std::vector<nyxb_ground_station> st; std::vector<int32_t> trk; nyxb_bls_config cfg; nyxb_tracking_arc carc;
        Ctx(const BatchLeastSquares& b, const Spacecraft& s, const TrackingDataArc& arc)
            : soa(std::vector<Spacecraft>{s}), eng(detail::make_engine(b.prop.dynamics, s.frame, b.almanac, b.prop.method, b.prop.opts, b.prop.mode, b.prop.device)),
              st(detail::pack_stations(b.devices, s.frame, b.almanac)), trk(detail::tracker_index(b.devices, arc)), cfg(b.config()) {
            const size_t m = arc.epoch_ns.size();
            if (arc.n != 1 || arc.obs.size() != m * 2 || arc.tracker.size() != m) throw std::runtime_error("arc shape: one observation set expected");
            carc = nyxb_tracking_arc{(int64_t)m, arc.epoch_ns.data(), trk.data(), arc.obs.data()};
        }
    };
    static void throw_status(int32_t status) {
        switch (status & 0xFF) {
            case 0: return;
            case NYXB_ERR_TOO_FEW_MEASUREMENTS: throw std::runtime_error("TooFewMeasurements");
            case NYXB_ERR_SINGULAR_INFORMATION: throw std::runtime_error("SingularInformationMatrix");
            case NYXB_ERR_INVALID_MEASUREMENT: throw std::runtime_error("InvalidMeasurement");
            default: throw std::runtime_error("ODPropError: status " + std::to_string(status & 0xFF));
        }
    }
};

// ---- Impulsive targeting: Targeter::try_achieve_from (md/opti/targeter.rs, raphson_finite_diff.rs:41-747) over nyxb_target_batch.
// Only the impulsive components run (PositionX..VelocityZ); objectives are the nyxb_tgt_param elements.
enum class Vary : int32_t { PositionX = NYXB_VARY_POSITION_X, PositionY = NYXB_VARY_POSITION_Y, PositionZ = NYXB_VARY_POSITION_Z,
                            VelocityX = NYXB_VARY_VELOCITY_X, VelocityY = NYXB_VARY_VELOCITY_Y, VelocityZ = NYXB_VARY_VELOCITY_Z };
enum class TargetFrame : int32_t { None = NYXB_TGT_FRAME_NONE, VNC = NYXB_TGT_FRAME_VNC, RIC = NYXB_TGT_FRAME_RIC };

// Variable with the reference's defaults for the impulsive components (target_variable.rs:219-244)
struct Variable {
    Vary component = Vary::VelocityX;
    double perturbation = 0.0001, init_guess = 0.0, max_step = 0.2, max_value = 5.0, min_value = -5.0;
    static Variable from(Vary v) { Variable x; x.component = v; return x; }
};

// Objective (md/objective.rs); `parameter` is an enum nyxb_tgt_param
struct Objective {
    int32_t parameter = NYXB_TGT_SMA;
    double desired_value = 0.0, tolerance = 1e-3, multiplicative_factor = 1.0, additive_factor = 0.0;
    // default_event_precision (md/param.rs:74-89): 0.1 s for the period, 1e-3 otherwise
    static Objective new_(int32_t p, double desired) { return within_tolerance(p, desired, p == NYXB_TGT_PERIOD ? 0.1 : 1e-3); }
    static Objective within_tolerance(int32_t p, double desired, double tol) { Objective o; o.parameter = p; o.desired_value = desired; o.tolerance = tol; return o; }
};

// TargetingError (md/opti/mod.rs): `variant` is the reference's variant name, `status` the nyxb status
struct TargetingError : std::runtime_error {
    std::string variant; int32_t status;
    TargetingError(std::string v, int32_t st, const std::string& msg) : std::runtime_error(v + ": " + msg), variant(std::move(v)), status(st) {}
};

struct TargeterSolution {  // md/opti/solution.rs:33-50
    Spacecraft corrected_state, achieved_state;
    std::vector<double> correction, achieved_errors;
    int32_t iterations = 0;
};

// every problem of one nyxb_target_batch call: [9][n], [n_vars][n], [n_objs][n], [n] (the last iteration's values on failure)
struct TargeterEnsembleSolution {
    std::vector<Spacecraft> states; int64_t correction_epoch_ns = 0, achievement_epoch_ns = 0; size_t n_vars = 0, n_objs = 0;
    std::vector<double> corrected, achieved, correction, errors; std::vector<int32_t> iterations, status;
    size_t size() const { return states.size(); }
    // nullopt when problem i converged, else the variant try_achieve_from throws
    std::optional<std::string> error(size_t i) const {
        switch (status[i] & 0xFF) {
            case 0: return std::nullopt;
            case NYXB_ERR_TGT_TOO_MANY_ITERATIONS: return std::string("TooManyIterations");
            case NYXB_ERR_TGT_CORRECTION_INEFFECTIVE: return std::string("CorrectionIneffective");
            case NYXB_ERR_TGT_SINGULAR_JACOBIAN: return std::string("SingularJacobian");
            case NYXB_ERR_TGT_NON_FINITE: return std::string("NonFinite");
            default: return std::string("PropError");
        }
    }
    TargeterSolution solution(size_t i) const {
        if (auto e = error(i)) {
            if ((status[i] & 0xFF) < NYXB_ERR_TGT_TOO_MANY_ITERATIONS) throw PropagationError(status[i]);
            throw TargetingError(*e, status[i], "problem " + std::to_string(i));
        }
        const size_t n = size();
        TargeterSolution s;
        s.corrected_state = detail::unpack(states[i], corrected, std::vector<int64_t>(n, correction_epoch_ns), n, i);
        s.achieved_state = detail::unpack(states[i], achieved, std::vector<int64_t>(n, achievement_epoch_ns), n, i);
        for (size_t j = 0; j < n_vars; ++j) s.correction.push_back(correction[j * n + i]);
        for (size_t j = 0; j < n_objs; ++j) s.achieved_errors.push_back(errors[j * n + i]);
        s.iterations = iterations[i];
        return s;
    }
};

class Targeter {
  public:
    Propagator prop; std::vector<Variable> variables; std::vector<Objective> objectives;
    int32_t iterations = 100; TargetFrame correction_frame = TargetFrame::None; const Almanac* almanac = nullptr;

    static Targeter new_(Propagator p, std::vector<Variable> v, std::vector<Objective> o) { Targeter t; t.prop = std::move(p); t.variables = std::move(v); t.objectives = std::move(o); return t; }
    static Targeter delta_v(Propagator p, std::vector<Objective> o) { return new_(std::move(p), {Variable::from(Vary::VelocityX), Variable::from(Vary::VelocityY), Variable::from(Vary::VelocityZ)}, std::move(o)); }
    static Targeter delta_r(Propagator p, std::vector<Objective> o) { return new_(std::move(p), {Variable::from(Vary::PositionX), Variable::from(Vary::PositionY), Variable::from(Vary::PositionZ)}, std::move(o)); }
    static Targeter vnc(Propagator p, std::vector<Objective> o) { Targeter t = delta_v(std::move(p), std::move(o)); t.correction_frame = TargetFrame::VNC; return t; }
    static Targeter vnc_with_components(Propagator p, std::vector<Variable> v, std::vector<Objective> o) { Targeter t = new_(std::move(p), std::move(v), std::move(o)); t.correction_frame = TargetFrame::VNC; return t; }

    nyxb_target_config config() const {
        if (variables.size() > 6 || objectives.size() > 6) throw TargetingError("UnsupportedProblem", 0, "at most 6 variables and 6 objectives");
        nyxb_target_config c{};
        c.n_vars = (int32_t)variables.size(); c.n_objs = (int32_t)objectives.size(); c.correction_frame = (int32_t)correction_frame; c.iterations = iterations;
        for (size_t j = 0; j < variables.size(); ++j) {
            const Variable& v = variables[j];
            c.vars[j] = nyxb_tgt_variable{(int32_t)v.component, 0, v.perturbation, v.init_guess, v.max_step, v.max_value, v.min_value};
        }
        for (size_t i = 0; i < objectives.size(); ++i) {
            const Objective& o = objectives[i];
            c.objs[i] = nyxb_tgt_objective{o.parameter, 0, o.desired_value, o.tolerance, o.multiplicative_factor, o.additive_factor};
        }
        return c;
    }

    // every state's problem in one call; the states share a frame, their epochs may differ
    TargeterEnsembleSolution try_achieve_from_many(const std::vector<Spacecraft>& v, int64_t correction_epoch_ns, int64_t achievement_epoch_ns) const {
        return run(config(), v, correction_epoch_ns, achievement_epoch_ns);
    }
    TargeterSolution try_achieve_from(const Spacecraft& s, int64_t correction_epoch_ns, int64_t achievement_epoch_ns) const {
        return try_achieve_from_many({s}, correction_epoch_ns, achievement_epoch_ns).solution(0);
    }

    // Targeter::apply (targeter.rs:257-351): the corrected state propagated to the achievement epoch, every objective's unscaled error
    // within its tolerance, else TargetingError "Verification".  The check is a call with no iteration and unit factors from the
    // corrected state, so the objectives are evaluated by the same code as the targeting.
    Spacecraft apply(const TargeterSolution& sol) const {
        nyxb_target_config c = config();
        c.iterations = 0;
        for (int j = 0; j < c.n_vars; ++j) c.vars[j].init_guess = 0.0;
        for (int i = 0; i < c.n_objs; ++i) { c.objs[i].multiplicative_factor = 1.0; c.objs[i].additive_factor = 0.0; }
        const int64_t t_c = sol.corrected_state.epoch(), t_f = sol.achieved_state.epoch();
        TargeterEnsembleSolution e = run(c, {sol.corrected_state}, t_c, t_f);
        const int32_t st = e.status[0] & 0xFF;
        if (st != 0 && st < NYXB_ERR_TGT_TOO_MANY_ITERATIONS) throw PropagationError(e.status[0]);
        std::string msg;
        for (int i = 0; i < c.n_objs; ++i)
            if (!(std::fabs(e.errors[(size_t)i]) <= c.objs[i].tolerance))
                msg += "objective " + std::to_string(i) + " error " + std::to_string(e.errors[(size_t)i]) + "; ";
        if (!msg.empty()) throw TargetingError("Verification", e.status[0], msg);
        return detail::unpack(sol.corrected_state, e.achieved, std::vector<int64_t>{t_f}, 1, 0);
    }

  private:
    TargeterEnsembleSolution run(const nyxb_target_config& c, const std::vector<Spacecraft>& v, int64_t t_c, int64_t t_f) const {
        if (v.empty()) throw std::runtime_error("no states");
        auto eng = detail::make_engine(prop.dynamics, v[0].frame, almanac, prop.method, prop.opts, prop.mode, prop.device);
        if (prop.kernel != NYXB_KERNEL_AUTO && nyxb_engine_set_kernel(eng.get(), prop.kernel) != NYXB_RC_OK)
            throw std::runtime_error(std::string("nyxb_engine_set_kernel: ") + nyxb_last_error());
        detail::Soa soa(v);
        const size_t n = v.size();
        TargeterEnsembleSolution e;
        e.states = v; e.correction_epoch_ns = t_c; e.achievement_epoch_ns = t_f; e.n_vars = (size_t)c.n_vars; e.n_objs = (size_t)c.n_objs;
        e.corrected.resize(9 * n); e.achieved.resize(9 * n); e.correction.resize(e.n_vars * n); e.errors.resize(e.n_objs * n);
        e.iterations.resize(n); e.status.resize(n);
        const int32_t rc = nyxb_target_batch(eng.get(), &c, n, soa.state.data(), soa.consts.data(), soa.epoch.data(), t_c, t_f, e.corrected.data(),
                                             e.achieved.data(), e.correction.data(), e.errors.data(), e.iterations.data(), e.status.data());
        if (rc != NYXB_RC_OK) throw std::runtime_error(std::string("nyxb_target_batch: ") + nyxb_last_error());
        return e;
    }
};

}  // namespace nyxb
