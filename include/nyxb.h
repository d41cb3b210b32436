/*
 * nyxb.h — C ABI of the H100 batched orbit-propagation engine (libnyxb.so).
 *
 * This is the drop-in boundary for ONE path of nyx-space/nyx (reference paths are
 * relative to /root/reference/nyx-core/src):
 *
 *   MonteCarlo::run_until_epoch            mc/montecarlo.rs:188-273
 *     -> Propagator::with(..)              propagators/propagator.rs:88-108
 *     -> PropInstance::until_epoch         propagators/instance.rs:279-282
 *     -> PropInstance::propagate           propagators/instance.rs:87-262
 *     -> PropInstance::derive              propagators/instance.rs:358-493
 *     -> SpacecraftDynamics::eom           dynamics/spacecraft.rs:191-310
 *
 * plus the "next" rows of SURVEY.md §8(f) that sit on the same path: trajectory recording, event-terminated runs,
 * STM propagation and the sequential Kalman filter of od/process (nyxb_propagate_batch_stm, nyxb_od_ekf_batch), and
 * on-device dispersions (nyxb_mvn_sample).
 *
 * A Rust shim (see INTEGRATION.md) packs `Vec<Spacecraft>` into the SoA arrays
 * below, calls nyxb_propagate_batch through `extern "C"`, and unpacks the final
 * states into `Results` / `Vec<Spacecraft>`.  Nothing here mentions torch or CUDA
 * types: plain pointers, sizes and PODs only.  All pointers are HOST pointers
 * unless the function name ends in `_dev`.
 *
 * Units follow the reference: km, km/s, kg, m^2, seconds; time is integer
 * nanoseconds (hifitime::Duration / Epoch are integer-ns types).
 */
#ifndef NYXB_H
#define NYXB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NYXB_ABI_VERSION 4 /* 4: nyxb_engine_set_kernel / nyxb_engine_last_kernel / nyxb_engine_set_tx_tuning, nyxb_tx_table_dump, nyxb_propagate_batch_multi, nyxb_reference_normals;
                              nyxb_integ_opts.state_center, nyxb_gravity_field.body, nyxb_dynamics.n_gravity / n_point_masses / point_mass_order; nyxb_od_predict_batch
                              and nyxb_predict_outputs, then nyxb_od_bls_batch, nyxb_od_bls_evaluate_batch, nyxb_bls_config, nyxb_bls_outputs and
                              the status codes 6-8, then nyxb_od_records, nyxb_od_ekf_record_batch, nyxb_smooth_outputs, nyxb_od_smooth_batch,
                              then NYXB_MSR_X/Y/Z, nyxb_position_device, nyxb_position_arc, nyxb_od_position_batch, nyxb_od_position_smooth_batch,
                              then NYXB_MSR_AZIMUTH/ELEVATION, nyxb_aer_station, nyxb_od_aer_batch, nyxb_od_aer_smooth_batch,
                              then nyxb_interlink_tx, nyxb_od_interlink_batch, nyxb_od_interlink_smooth_batch
                              and the status codes 9-12 were added later without a bump (a pure addition: no existing type or entry point changed).  Earlier: 2: nyxb_srp gained `estimate`; STM, filter and dispersion entry points.  3: nyxb_traj_resample[_dev], nyxb_event_locate[_dev] */

/* ---- IntegratorMethod — propagators/rk_methods/mod.rs:65-79 (same order) ---- */
enum nyxb_method {
    NYXB_RK89 = 0,        /* RungeKutta89 (default)   rk_methods/rk.rs:89-252   */
    NYXB_DP78 = 1,        /* DormandPrince78          rk_methods/dormand.rs:71-184 */
    NYXB_DP45 = 2,        /* DormandPrince45          rk_methods/dormand.rs:23-69 */
    NYXB_RK4 = 3,         /* RungeKutta4 (fixed)      rk_methods/rk.rs:60-81    */
    NYXB_CK45 = 4,        /* CashKarp45               rk_methods/rk.rs:21-58    */
    NYXB_V56 = 5          /* Verner56                 rk_methods/verner.rs:24-79 */
};

/* ---- ErrorControl — propagators/error_ctrl.rs:30-71 (same order) ---- */
enum nyxb_error_ctrl {
    NYXB_RSS_CARTESIAN_STATE = 0,
    NYXB_RSS_CARTESIAN_STEP = 1, /* default */
    NYXB_RSS_STATE = 2,
    NYXB_RSS_STEP = 3,
    NYXB_LARGEST_ERROR = 4,
    NYXB_LARGEST_STATE = 5,
    NYXB_LARGEST_STEP = 6
};

/* ---- IntegratorOptions — propagators/options.rs:42-60 ----
 * Durations are hifitime integer nanoseconds.  `with_fixed_step` semantics
 * (options.rs:100-111): fixed_step=1, min=max=init=step, tolerance=0, attempts=0. */
typedef struct {
    int32_t method;      /* enum nyxb_method */
    int32_t error_ctrl;  /* enum nyxb_error_ctrl */
    int64_t init_step_ns;
    int64_t min_step_ns;
    int64_t max_step_ns;
    double tolerance;
    int32_t attempts;    /* u8 in the reference */
    int32_t fixed_step;  /* bool */
    /* IntegratorOptions.integration_frame (options.rs:60; instance.rs:117-142, 167-176, 211-220).  The engine's dynamics always
     * describe the INTEGRATION frame.  0: the states handed to nyxb_propagate_batch* are expressed in it (integration_frame = None, or
     * equal to the state's frame).  k + 1: the states are expressed relative to dynamics.bodies[k] (same inertial axes): they are
     * translated into the integration frame before the loop with that body's position and velocity at each trajectory's start
     * epoch (anise `transform_to`), and translated back at the epoch each run ends at.  Recorded trajectories and event scalars are
     * in the integration frame, as in the reference (the channel sends `self.state` from inside the loop). */
    int32_t state_center;
    int32_t _pad;
} nyxb_integ_opts;

/* ---- Body-fixed frame orientation (what anise `Almanac::rotate` supplies to
 * gravity_field.rs:150-154,258-265 and drag.rs:184-189).  anise and its PCK data
 * are absent from the reference tree, so the orientation is an explicit model:
 *   kind 0: body-fixed axes == inertial axes (no rotation)
 *   kind 1: IAU pole/prime-meridian, angles in degrees,
 *           ra = ra0 + ra1*T, dec = dec0 + dec1*T, W = w0 + w1*d,
 *           T = Julian centuries, d = days past the reference epoch (t = 0 ns),
 *           DCM inertial->fixed = R3(W) R1(90deg-dec) R3(90deg+ra). */
typedef struct {
    int32_t kind;
    int32_t _pad;
    double ra0_deg, ra1_deg_cy;
    double dec0_deg, dec1_deg_cy;
    double w0_deg, w1_deg_day;
} nyxb_rotation;

/* ---- GravityField — dynamics/gravity_field.rs:36-48 + io/gravity.rs:90-96 ----
 * c_nm/s_nm: normalised coefficients, row-major [(degree+1) x (degree+1)], entry
 * (n,m) at n*(degree+1)+m.  mu and r_eq are passed explicitly because the reference
 * takes them from the *frame* (gravity_field.rs:195-207), never from the file. */
typedef struct {
    int32_t degree;
    int32_t order;
    double mu_km3_s2;
    double r_eq_km;
    const double* c_nm;
    const double* s_nm;
    nyxb_rotation rot;
    /* The body this field belongs to: NYXB_CENTRAL_BODY (-1) = the integration-frame centre, else an index into
     * nyxb_dynamics.bodies — the state is translated to that body before the harmonic sum and the acceleration vector is rotated
     * back unchanged (gravity_field.rs:149-154, 258-267: "needed for multiple harmonic fields"). */
    int32_t body;
    int32_t _pad;
} nyxb_gravity_field;

/* ---- Ephemeris of one celestial body relative to the integration-frame centre,
 * inertial axes: piecewise Chebyshev position series (what anise evaluates from an
 * SPK for orbital.rs:230-234 / solarpressure.rs:138-143 / eclipse.rs:77).
 * coeffs layout: [n_intervals][3][n_coeffs]; interval i covers
 * [t0_ns + i*interval_ns, t0_ns + (i+1)*interval_ns). */
typedef struct {
    double mu_km3_s2;
    double radius_km;      /* mean equatorial radius (shadow computations) */
    int64_t t0_ns;
    int64_t interval_ns;
    int32_t n_intervals;
    int32_t n_coeffs;
    const double* coeffs;
} nyxb_body;

#define NYXB_MAX_BODIES 8
#define NYXB_CENTRAL_BODY (-1)
#define NYXB_MAX_FIELDS 3      /* harmonic fields per dynamics (OrbitalDynamics holds a Vec of accel models, orbital.rs:44-46) */

/* ---- SolarPressure + ShadowModel — dynamics/solarpressure.rs:43-49,135-165;
 * cosmic/eclipse.rs:35-83.  Body indices refer to nyxb_dynamics.bodies;
 * NYXB_CENTRAL_BODY designates the integration-frame centre. */
typedef struct {
    double phi_w_m2;        /* solar flux at 1 AU, default 1367 (solarpressure.rs:35) */
    int32_t sun_body;       /* index of the light source in bodies[] */
    int32_t n_shadow;
    int32_t shadow_body[4];
    int32_t estimate;       /* SolarPressure.estimate (solarpressure.rs:47-48, 131-133): Cr column of the STM A-matrix */
    int32_t _pad;
} nyxb_srp;

/* ---- Drag — dynamics/drag.rs:36-42,123-130,181-284 ---- */
enum nyxb_density {
    NYXB_DENSITY_CONSTANT = 0,   /* AtmDensity::Constant(rho) */
    NYXB_DENSITY_EXPONENTIAL = 1,/* AtmDensity::Exponential{rho0,r0,ref_alt_m} */
    NYXB_DENSITY_STDATM = 2      /* AtmDensity::StdAtm{max_alt_m} */
};
typedef struct {
    int32_t density;        /* enum nyxb_density */
    int32_t _pad;
    double rho0;            /* Constant: rho ; Exponential: rho0 */
    double r0;              /* Exponential */
    double ref_alt_m;       /* Exponential: ref_alt_m ; StdAtm: max_alt_m */
    double r_eq_km;         /* frame.mean_equatorial_radius_km() */
    nyxb_rotation rot;      /* drag frame orientation (IAU_EARTH in the reference) */
} nyxb_drag;

/* ---- SpacecraftDynamics — closed set of models the GPU path accepts
 * (dynamics/sequence/config.rs:96-169 serialises exactly this set). ---- */
typedef struct {
    double mu_central_km3_s2;     /* osc.frame.mu_km3_s2()  orbital.rs:86-90 */
    double central_radius_km;     /* used when the centre is a shadow body */
    int32_t n_bodies;
    int32_t n_gravity;            /* entries of `gravity` (0 with gravity != NULL is read as 1: ABI <= 3 callers) */
    const nyxb_body* bodies;      /* ephemerides available to the models */
    uint32_t point_mass_mask;     /* bit j set: bodies[j] acts as PointMasses member (orbital.rs:213-247) */
    int32_t n_point_masses;       /* > 0: `point_mass_order` lists the members in `celestial_objects` order (orbital.rs:217), which is
                                     the summation order STRICT mode reproduces; 0: ascending body index of the mask */
    const nyxb_gravity_field* gravity;  /* NULL: none; else n_gravity fields in accel-model order.  gravity[0] is the field the
                                           cooperative kernels split over lanes / warps; the others are summed per trajectory */
    const nyxb_srp* srp;                /* NULL: none */
    const nyxb_drag* drag;              /* NULL: none */
    int32_t point_mass_order[NYXB_MAX_BODIES];
} nyxb_dynamics;

/* ---- IntegrationDetails (propagators/mod.rs:49-56) + counters for the metric ---- */
typedef struct {
    int64_t step_ns;     /* details.step of the last step */
    double error;        /* details.error of the last adaptive step */
    int32_t attempts;    /* details.attempts of the last step */
    int32_t _pad;
    int64_t n_steps;     /* accepted steps incl. the final partial step */
    int64_t n_rejected;  /* rejected attempts */
    int64_t n_rhs;       /* RHS evaluations */
} nyxb_details;

/* ---- per-trajectory status: mirrors the reference's error variants ---- */
enum nyxb_status {
    NYXB_OK = 0,
    NYXB_ERR_PROP_MATH = 1,      /* PropagationError::PropMathError (NaN)  instance.rs:432-439 */
    NYXB_ERR_FUEL_EXHAUSTED = 2, /* DynamicsError::FuelExhausted           spacecraft.rs:163-168 */
    NYXB_ERR_MASSLESS = 3,       /* DynamicsError::MasslessSpacecraft      spacecraft.rs:201-203 */
    NYXB_ERR_EPHEMERIS = 4,      /* almanac error: epoch outside ephemeris coverage */
    NYXB_ERR_EVENT_NOT_FOUND = 5,/* PropagationError::NthEventError: end epoch reached first (event.rs:177-182) */
    NYXB_ERR_TOO_FEW_MEASUREMENTS = 6, /* ODError::TooFewMeasurements (blse/mod.rs:155-161) */
    NYXB_ERR_SINGULAR_INFORMATION = 7, /* ODError::SingularInformationMatrix (blse/mod.rs:312-315) */
    NYXB_ERR_INVALID_MEASUREMENT = 8,  /* ODError::InvalidMeasurement: an observation that is not finite (blse/mod.rs:266-272) */
    NYXB_ERR_SINGULAR_STM = 9,         /* ODError::SingularStateTransitionMatrix (solution/smooth.rs:149-154) */
    NYXB_ERR_RECORDS_TRUNCATED = 10,   /* the estimate records of a filter exceed their capacity: nothing to smooth from */
    NYXB_ERR_TX_NO_DATA = 11,          /* ODError::ODTrajError: the interlink transmitter's recording does not cover the epoch
                                          (interlink/trk_device.rs:180-183, sensitivity.rs:93-101) */
    NYXB_ERR_NO_RANGE = 12,            /* ODError::MeasurementSimError: an interlink Doppler row without an observed range in the same
                                          measurement (interlink/sensitivity.rs:105-110) */
    NYXB_ERR_TGT_TOO_MANY_ITERATIONS = 13,     /* TargetingError::TooManyIterations (raphson_finite_diff.rs:746) */
    NYXB_ERR_TGT_CORRECTION_INEFFECTIVE = 14,  /* TargetingError::CorrectionIneffective: | |err| - previous |err| | < 1e-10 */
    NYXB_ERR_TGT_SINGULAR_JACOBIAN = 15,       /* TargetingError::SingularJacobian: the pseudo-inverse's m x m inverse failed */
    NYXB_ERR_TGT_NON_FINITE = 16,              /* an objective value or Jacobian entry that is not finite (anise's partial_for fails) */
    NYXB_WARN_MAX_ATTEMPTS = 0x100 /* OR-ed flag: instance.rs:440-445 (warn only) */
};

/* ---- execution mode ---- */
enum nyxb_mode {
    NYXB_MODE_STRICT = 0, /* reference operation order, no FMA contraction: bit-parity mode */
    NYXB_MODE_FAST = 1    /* FMA + reordered cooperative harmonics: tolerance-parity mode */
};

/* ---- library-level return codes ---- */
enum nyxb_rc {
    NYXB_RC_OK = 0,
    NYXB_RC_BAD_ARG = -1,
    NYXB_RC_NO_DEVICE = -2,
    NYXB_RC_CUDA = -3,
    NYXB_RC_UNSUPPORTED = -4
};

typedef struct nyxb_engine nyxb_engine; /* opaque: device tables for one (dynamics, opts) pair */

/* Build device-resident tables (tableau, harmonic coefficients, ephemerides) for a
 * propagator setup == `Propagator::new(dynamics, method, opts)` (propagator.rs:55-61).
 * `device` is the CUDA ordinal.  Returns NULL on failure (see nyxb_last_error). */
nyxb_engine* nyxb_engine_create(const nyxb_dynamics* dyn, const nyxb_integ_opts* opts,
                                int32_t mode, int32_t device);
void nyxb_engine_destroy(nyxb_engine* eng);

/* Propagate n independent spacecraft until `end_epoch_ns`
 * == for each i: `prop.with(state_i, almanac).until_epoch(end_epoch)`
 * (mc/montecarlo.rs:233-253; nyx-py many_until_epoch py_md.rs:224-271).
 *
 *  state_soa   [9][n]  x,y,z,vx,vy,vz,Cr,Cd,prop_mass   (cosmic/spacecraft.rs:449-473)
 *  consts_soa  [4][n]  dry_mass_kg, extra_mass_kg, srp_area_m2, drag_area_m2
 *  epoch0_ns   [n]     start epochs (ns past the reference epoch of the ephemerides)
 *  step_ns     [n] or NULL: in/out adapted step of each PropInstance (instance.rs:56);
 *                      NULL => every run starts from opts.init_step_ns
 *  out_*       same layouts; out_epoch_ns [n]; details [n]; status [n]
 * Per-trajectory failures are reported in out_status and never abort the batch
 * (mc/results.rs:48-59).  Thread-safe for distinct engines. */
int32_t nyxb_propagate_batch(nyxb_engine* eng, size_t n,
                             const double* state_soa, const double* consts_soa,
                             const int64_t* epoch0_ns, int64_t end_epoch_ns,
                             int64_t* step_ns,
                             double* out_state_soa, int64_t* out_epoch_ns,
                             nyxb_details* out_details, int32_t* out_status);

/* Same, but every array is a DEVICE pointer on the engine's device and the launch
 * is enqueued on `cuda_stream` (a cudaStream_t passed as void*, NULL = default
 * stream) without synchronising.  Used by bench.py's HBM-resident `value` leg and
 * by the multi-GPU driver (final-state all-gather is stream-ordered after it). */
int32_t nyxb_propagate_batch_dev(nyxb_engine* eng, size_t n,
                                 const double* state_soa, const double* consts_soa,
                                 const int64_t* epoch0_ns, int64_t end_epoch_ns,
                                 int64_t* step_ns,
                                 double* out_state_soa, int64_t* out_epoch_ns,
                                 nyxb_details* out_details, int32_t* out_status,
                                 void* cuda_stream);

/* Multi-GPU fan-out of one ensemble behind the boundary (mc/montecarlo.rs:233-253: runs are independent, shards are contiguous
 * run-index ranges, nothing is exchanged while integrating).  `engines[g]`: one engine per device, all created from the same
 * (dynamics, options, mode); shard g = runs [g n / G, (g+1) n / G).  HOST arrays exactly as nyxb_propagate_batch; every device
 * integrates concurrently and its results land directly in the caller's [9][n] arrays — for a host caller this is the gather of
 * final states (device-resident callers launch nyxb_propagate_batch_dev per rank and all-gather, see nyx_b200/dist.py).
 * `mc.run_until_epoch(prop, almanac, end, num_runs)` on G GPUs is ONE call of this function. */
int32_t nyxb_propagate_batch_multi(nyxb_engine* const* engines, int32_t n_engines, size_t n,
                                   const double* state_soa, const double* consts_soa,
                                   const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                   double* out_state_soa, int64_t* out_epoch_ns,
                                   nyxb_details* out_details, int32_t* out_status);

/* ---- Trajectory recording (next row (f)-1 of SURVEY.md §8): what `for_duration_with_traj` / `until_epoch_with_traj`
 * (propagators/instance.rs:297-340) collect through the mpsc channel (instance.rs:186-193, 255-259): the start state and
 * the state after every accepted step, final partial step included.  Record s of trajectory i lives at
 *   epoch_ns[s*n + i],  state[(c*capacity + s)*n + i]  (c = x,y,z,vx,vy,vz)
 * i.e. step-major SoA: trajectories that advance together write coalesced 56-byte-per-step streams.
 * count[i] = min(n_steps + 1, capacity); records beyond `capacity` are dropped (the final state is still returned).
 * As the transmitters of nyxb_od_interlink_batch / _smooth_batch (HOST pointers, n = n_tx): every column must be complete, with
 * 1 <= count[j] <= capacity (a propagation that dropped records has count > capacity and is refused), epochs in step order. */
typedef struct {
    int64_t capacity;
    int64_t* epoch_ns;   /* [capacity][n] */
    double* state;       /* [6][capacity][n] */
    int64_t* count;      /* [n] */
} nyxb_traj_sink;

/* ---- Event-terminated propagation (next row (f)-3): the stop condition of `PropInstance::until_nth_event`
 * (propagators/event.rs:88-211, used by MonteCarlo::run_until_nth_event mc/montecarlo.rs:93-183).  After every accepted
 * NON-final step the event scalar minus `value` is evaluated; a sign change (y_prev * y_next < 0, event.rs:141-144) counts
 * one crossing; the run stops at the end of the step that brings the count to `trigger` (the state is returned and
 * recorded).  The root search inside that last step (Brent on the Hermite-interpolated trajectory, event.rs:186-196)
 * stays on the host.  Closed set of scalars (the reference's anise `ScalarExpr` is open-ended and not in the tree). */
enum nyxb_event_kind {
    NYXB_EVENT_NONE = 0,
    NYXB_EVENT_RMAG = 1,   /* |r| km            */
    NYXB_EVENT_RDOTV = 2,  /* r . v  km^2/s  (zero at the apsides) */
    NYXB_EVENT_X = 3, NYXB_EVENT_Y = 4, NYXB_EVENT_Z = 5,   /* Cartesian components, km (Z = 0: node crossing) */
    NYXB_EVENT_VMAG = 6    /* |v| km/s          */
};
typedef struct {
    int32_t kind;       /* enum nyxb_event_kind */
    int32_t trigger;    /* 1-based number of crossings to stop at */
    double value;       /* desired value: the monitored function is scalar - value */
    int32_t* crossings; /* [n] out: crossings seen; status NYXB_ERR_EVENT_NOT_FOUND when < trigger at the end epoch */
} nyxb_event;

/* nyxb_propagate_batch_traj + stop condition (HOST arrays; event == NULL: plain until-epoch propagation). */
int32_t nyxb_propagate_batch_event(nyxb_engine* eng, size_t n,
                                   const double* state_soa, const double* consts_soa,
                                   const int64_t* epoch0_ns, int64_t end_epoch_ns,
                                   int64_t* step_ns,
                                   double* out_state_soa, int64_t* out_epoch_ns,
                                   nyxb_details* out_details, int32_t* out_status,
                                   const nyxb_traj_sink* sink, const nyxb_event* event);

/* nyxb_propagate_batch + recording into `sink` (HOST arrays; NULL sink == nyxb_propagate_batch). */
int32_t nyxb_propagate_batch_traj(nyxb_engine* eng, size_t n,
                                  const double* state_soa, const double* consts_soa,
                                  const int64_t* epoch0_ns, int64_t end_epoch_ns,
                                  int64_t* step_ns,
                                  double* out_state_soa, int64_t* out_epoch_ns,
                                  nyxb_details* out_details, int32_t* out_status,
                                  const nyxb_traj_sink* sink);

/* Device-pointer variant: the sink's arrays are DEVICE pointers (the struct itself is read on the host). */
int32_t nyxb_propagate_batch_traj_dev(nyxb_engine* eng, size_t n,
                                      const double* state_soa, const double* consts_soa,
                                      const int64_t* epoch0_ns, int64_t end_epoch_ns,
                                      int64_t* step_ns,
                                      double* out_state_soa, int64_t* out_epoch_ns,
                                      nyxb_details* out_details, int32_t* out_status,
                                      const nyxb_traj_sink* sink, void* cuda_stream);

/* ---- Batched resampling of recorded trajectories on a common epoch grid (row (f)-1): what `Traj::every` /
 * `every_between` (md/trajectory/traj.rs:148-162, traj_it.rs:32-63) yield through `Traj::at` (traj.rs:83-126: exact hit,
 * else a window of 13 records around the query — 12 at the right edge, as coded — Hermite-interpolated in (r, v),
 * md/trajectory/interpolatable.rs:53-108) and what `Results::every_value_of[_between]` (mc/results.rs:88-160) iterate over,
 * for all n trajectories and all m query epochs in ONE launch.
 *  sink            the recording as filled by nyxb_propagate_batch_traj / _event (capacity, epoch_ns, state, count);
 *                  NULL (host variant only): the recording of this engine's last host-pointer propagation, still
 *                  resident in device memory (no upload);
 *  query_epoch_ns  [m];
 *  out_state       [6][m][n]  x,y,z,vx,vy,vz of trajectory i at query j at [(c*m + j)*n + i]; NaN where no data;
 *  out_status      [m][n]     NYXB_TRAJ_OK, or NYXB_TRAJ_NO_DATA when the query lies outside the trajectory's recorded
 *                             span (TrajError::NoInterpolationData) — a per-entry status, the batch never aborts.
 * Seconds are counted from the first record of the window (the reference passes absolute ET seconds to anise's
 * hermite_eval, which is not in the tree: parity unpinned at that boundary, DESIGN.md §9). */
enum nyxb_traj_status { NYXB_TRAJ_OK = 0, NYXB_TRAJ_NO_DATA = 1 };
int32_t nyxb_traj_resample(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink,
                           size_t m, const int64_t* query_epoch_ns, double* out_state, int32_t* out_status);
/* Device-pointer variant: the sink's arrays, the queries and the outputs are DEVICE pointers; stream-ordered. */
int32_t nyxb_traj_resample_dev(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink,
                               size_t m, const int64_t* query_epoch_ns, double* out_state, int32_t* out_status,
                               void* cuda_stream);

/* ---- Event location on the recorded trajectories (row (f)-3): the search `until_nth_event` runs after the propagation
 * stopped (propagators/event.rs:166-211: Brent's method on `event(traj.at(epoch))` between the last state on the channel and
 * the returned state), for all n runs in ONE launch.  The bracket is the last recorded step of each trajectory; the search
 * stops when the bracket is narrower than `epoch_precision_ns`; the state at the event epoch is the Hermite-interpolated one
 * (nyxb_traj_resample's arithmetic).
 *  sink               as for nyxb_traj_resample (NULL: the resident recording of the last host-pointer propagation);
 *  kind, value        the monitored scalar (enum nyxb_event_kind) and its desired value;
 *  run_status         [n] or NULL: out_status of the propagation — runs with an error code are skipped;
 *  out_event_epoch_ns [n], out_event_state [6][n] (NaN where not located),
 *  out_status         [n]: NYXB_TRAJ_OK; NYXB_TRAJ_NO_DATA (skipped run, fewer than two records);
 *                     NYXB_EVENT_NOT_BRACKETED (the scalar has the same sign at both ends of the last step).
 * The search cannot see a truncated recording: it takes the last two records the sink holds.  When the run took more steps
 * than the sink's capacity (count == capacity), those are not the bracketing step and the located event is wrong or
 * NOT_BRACKETED.  Give the propagation a sink with room for every step (PropInstance.until_nth_event refuses a capacity
 * that is too small; MonteCarlo.run_until_nth_event grows its sink and propagates again). */
enum { NYXB_EVENT_NOT_BRACKETED = 2 };
int32_t nyxb_event_locate(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, int32_t kind, double value,
                          int64_t epoch_precision_ns, const int32_t* run_status,
                          int64_t* out_event_epoch_ns, double* out_event_state, int32_t* out_status);
/* Device-pointer variant (sink arrays, run_status and outputs are DEVICE pointers; stream-ordered). */
int32_t nyxb_event_locate_dev(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, int32_t kind, double value,
                              int64_t epoch_precision_ns, const int32_t* run_status,
                              int64_t* out_event_epoch_ns, double* out_event_state, int32_t* out_status, void* cuda_stream);

/* ---- State-transition-matrix propagation (next row (f)-2 of SURVEY.md §8): `Spacecraft::with_stm()` + propagate.
 * The integrated vector is the reference's 90-vector [x,y,z,vx,vy,vz,Cr,Cd,prop_mass, STM 9x9 column-major]
 * (cosmic/spacecraft.rs:449-473).  Stage derivative of the STM block AS CODED in the reference:
 * `ctx.stm * grad` with `ctx` = the state at the START of the step (dynamics/spacecraft.rs:203-227,
 * propagators/instance.rs:363-364), grad = the 9x9 A-matrix of `dual_eom` (spacecraft.rs:312-363;
 * orbital.rs:116-172, 249-307; gravity_field.rs:273-431; solarpressure.rs:167-233; Cr column when the SRP model
 * estimates it; Drag has no partials: `PartialsUndefined`, drag.rs:109-118, 286-295 -> NYXB_RC_UNSUPPORTED).
 * Only the Cartesian error controls (which look at r and v alone, error_ctrl.rs:89-122) and fixed steps are accepted.
 *  stm_in_soa / out_stm_soa  [81][n], entry (row r, col c) of trajectory i at [(c*9 + r)*n + i];
 *  stm_in_soa == NULL: identity (State::with_stm, cosmic/spacecraft.rs:433-440). */
int32_t nyxb_propagate_batch_stm(nyxb_engine* eng, size_t n,
                                 const double* state_soa, const double* consts_soa,
                                 const int64_t* epoch0_ns, int64_t end_epoch_ns,
                                 int64_t* step_ns, const double* stm_in_soa,
                                 double* out_state_soa, int64_t* out_epoch_ns, double* out_stm_soa,
                                 nyxb_details* out_details, int32_t* out_status);

/* ---- Sequential Kalman orbit determination over an ensemble (next row (f)-2; BASELINE configs[4]):
 * n independent `KalmanODProcess::process_arc` runs (od/process/mod.rs:128-497) — propagate the nominal state + STM
 * to each measurement, `KalmanFilter::time_update` / `measurement_update` (od/kalman/filtering.rs:59-316), state
 * replacement (EKF) and STM reset — in ONE kernel launch, one filter per trajectory. */
enum nyxb_msr_type { NYXB_MSR_RANGE = 0, NYXB_MSR_DOPPLER = 1,   /* od/msr/types.rs:31-45 (the two-way capable ones) */
                     NYXB_MSR_AZIMUTH = 2, NYXB_MSR_ELEVATION = 3, /* degrees; ground stations with angles (nyxb_aer_station) */
                     NYXB_MSR_X = 6, NYXB_MSR_Y = 7, NYXB_MSR_Z = 8 }; /* position fixes (nyxb_position_device) */

/* GroundStation (od/ground_station/mod.rs:47-75) reduced to what the filter needs.  The host converts latitude /
 * longitude / height into the body-fixed position and the local zenith (anise `Orbit::try_latlongalt`); the tracker's
 * inertial state is R^T p (+ w x r), translated by the ephemeris of `body` when the station does not sit on the
 * integration centre (trk_device.rs:150-152 `location`).  Instantaneous measurements only
 * (`integration_time: None`, trk_device.rs:154-200); light-time correction off. */
typedef struct {
    double pos_fixed_km[3];
    double up_fixed[3];          /* unit local zenith in the body-fixed frame (elevation = asin(rho_hat . up)) */
    double elevation_mask_deg;
    nyxb_rotation rot;           /* orientation of the station's body-fixed frame */
    int32_t body;                /* NYXB_CENTRAL_BODY or index into dynamics.bodies: the body the station sits on */
    int32_t n_types;             /* 1 or 2 */
    int32_t types[2];            /* enum nyxb_msr_type, in the device's IndexSet order */
    int32_t _pad;
    double noise_var[2];         /* TrackingDevice::measurement_covar per type (trk_device.rs:223-236) */
    double bias[2];              /* TrackingDevice::measurement_bias per type (trk_device.rs:238-253) */
    double body_radius_km;       /* radius of the body the spacecraft orbits when it can obstruct the line of sight
                                    (trk_device.rs:162-166); <= 0: no obstruction test */
} nyxb_ground_station;

enum nyxb_kf_variant { NYXB_KF_REFERENCE_UPDATE = 0 /* EKF */, NYXB_KF_DEVIATION_TRACKING = 1 /* CKF */ }; /* od/kalman/mod.rs */

typedef struct {
    int32_t variant;             /* enum nyxb_kf_variant */
    int32_t msr_size;            /* MsrSize::DIM: 2 = SpacecraftKalmanOD, 1 = SpacecraftKalmanScalarOD (od/mod.rs:77-91) */
    double reject_num_sigmas;    /* SigmaRejection.num_sigmas (process/rejectcrit.rs:35-46); < 0: None */
    int64_t max_step_ns;         /* KalmanODProcess.max_step, default 1 min (process/initializers.rs:66-75) */
    int64_t epoch_precision_ns;  /* default 1 us */
    /* one ProcessNoise3D (od/snc.rs:38-56), no decay / start time */
    int32_t snc_enabled;
    int32_t snc_frame;           /* 0: state frame, 1: LocalFrame::RIC (snc.rs:226-262) */
    double snc_diag[3];          /* km^2/s^4 */
    int64_t snc_disable_time_ns;
} nyxb_od_config;

/* Tracking arc shared by the ensemble (one schedule, n observation sets) and the per-measurement outputs.
 * obs[(k*2 + t)*n + i]: observation of type t (enum nyxb_msr_type) of trajectory i at measurement k; NaN = that
 * type is not in `msr.data` (both NaN: the measurement is not in trajectory i's arc at all). */
typedef struct {
    int64_t n_msr;
    const int64_t* epoch_ns;     /* [n_msr] ascending */
    const int32_t* tracker;      /* [n_msr] index into stations; < 0: unknown tracker (process/mod.rs:400-410) */
    const double* obs;           /* [n_msr][2][n] */
} nyxb_tracking_arc;

enum nyxb_msr_flag {
    NYXB_MSRF_PROCESSED = 1,     /* a measurement update ran (accepted or rejected by the sigma test) */
    NYXB_MSRF_REJECTED = 2,      /* residual ratio above num_sigmas: time update only (filtering.rs:169-184) */
    NYXB_MSRF_NOT_VISIBLE = 4,   /* device.measure() returned None: below the mask / obstructed (process/mod.rs:386-392) */
    NYXB_MSRF_ABSENT = 8         /* no data for this trajectory */
};

typedef struct {
    double* state_soa;           /* [9][n]  final nominal state (EKF: estimate) */
    int64_t* epoch_ns;           /* [n] */
    double* covar_soa;           /* [81][n] final covariance, (r,c) at [(c*9+r)*n + i] */
    double* state_dev_soa;       /* [9][n]  final state deviation (CKF); NULL to skip */
    /* per measurement k and residual window w (msr_size 2: one window holding both types; msr_size 1: one per type) */
    double* resid_ratio;         /* [n_msr][2][n] or NULL */
    double* prefit;              /* [n_msr][2][n] or NULL  (slot = position of the type in the device's list) */
    double* postfit;             /* [n_msr][2][n] or NULL */
    int32_t* msr_flags;          /* [n_msr][n]    or NULL */
    double* est_state;           /* [n_msr][9][n] or NULL: estimated state after measurement k */
    double* est_covar_diag;      /* [n_msr][9][n] or NULL */
    nyxb_details* details;       /* [n] or NULL: n_steps / n_rhs over the whole arc */
    int32_t* status;             /* [n] */
} nyxb_od_outputs;

/* state_soa/consts_soa/epoch0_ns as in nyxb_propagate_batch (initial_estimate.nominal_state);
 * covar0_soa [81][n] initial covariance (KfEstimate.covar); HOST pointers everywhere. */
int32_t nyxb_od_ekf_batch(nyxb_engine* eng, const nyxb_od_config* cfg,
                          int32_t n_stations, const nyxb_ground_station* stations,
                          const nyxb_tracking_arc* arc, size_t n,
                          const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                          const double* covar0_soa, const nyxb_od_outputs* out);

/* ---- Every estimate of a filter run, for the smoother.  nyxb_od_ekf_record_batch runs nyxb_od_ekf_batch (same arguments, same
 * kernel family, bit-identical `out`) and also writes one record per entry the reference pushes to ODSolution.estimates
 * (process/mod.rs:211-426), in push order:
 *   - a time update per propagation chunk that does not land on a measurement (several per gap when the step is below max_step);
 *   - a measurement update per residual window that reaches `measurement_update`, sigma-rejected ones included (their estimate is the
 *     time update made inside it, filtering.rs:186-200).  With msr_size 1 and two types, one epoch gives two records, the second with
 *     STM = I.
 * Nothing is recorded for absent measurements, unknown trackers or windows that are not visible; the STM is not reset there either, so
 * the next record's STM spans back to the previous record.  Per record: nominal_state (for an EKF measurement update, the PRE-update
 * nominal), state_deviation (EKF: x-hat after a measurement update, zero after a time update; CKF: the deviation, Phi x after a time
 * update), covariance, and the STM since the previous record (Phi), as KfEstimate holds them; estimate.state() = nominal + deviation
 * with Cr clamped to [0, 2].  Residuals are not repeated here: the tag leads to prefit / postfit / resid_ratio of nyxb_od_outputs.
 * Records k >= capacity are dropped; count[i] counts all of them (as nyxb_traj_sink).  1 456 bytes per record. */
#define NYXB_OD_TAG_TIME_UPDATE (-1)
/* tag of a measurement-update record: ((k*2 + w)*2 + rejected)*2 + (msr_size - 1), with k the measurement index, w the residual
 * window (the types w*msr_size .. of the tracker) and rejected 1 for a sigma-rejected window */
#define NYXB_OD_TAG(k, w, rejected, msr_size) ((((int64_t)(k) * 2 + (w)) * 2 + (rejected)) * 2 + ((msr_size) - 1))
#define NYXB_OD_TAG_MSR(tag) ((tag) >> 3)
#define NYXB_OD_TAG_WINDOW(tag) (((tag) >> 2) & 1)
#define NYXB_OD_TAG_REJECTED(tag) (((tag) >> 1) & 1)
#define NYXB_OD_TAG_MSR_SIZE(tag) (((tag) & 1) + 1)

typedef struct {
    int64_t capacity;            /* records kept per filter */
    int64_t* epoch_ns;           /* [capacity][n] */
    int64_t* tag;                /* [capacity][n] NYXB_OD_TAG_TIME_UPDATE or NYXB_OD_TAG(..) */
    double* nominal;             /* [capacity][9][n] [(k*9 + r)*n + i] */
    double* deviation;           /* [capacity][9][n] */
    double* covar;               /* [capacity][81][n] (r,c) at [(k*81 + c*9 + r)*n + i] */
    double* stm;                 /* [capacity][81][n] Phi from the previous record, same layout */
    int64_t* count;              /* [n] records produced by filter i (kept or not) */
} nyxb_od_records;

/* Arguments as nyxb_od_ekf_batch, plus the records: every array of *rec non-NULL (the record arrays may be NULL when capacity is 0).
 * Records a filter does not reach are left as NaN (tag and epoch: -1). */
int32_t nyxb_od_ekf_record_batch(nyxb_engine* eng, const nyxb_od_config* cfg,
                                 int32_t n_stations, const nyxb_ground_station* stations,
                                 const nyxb_tracking_arc* arc, size_t n,
                                 const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                                 const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec);

/* ---- ODSolution::smooth (od/process/solution/smooth.rs:104-249) for n filters in ONE launch, from their records.  As coded, each
 * estimate k < l (l the last) is smoothed from the FILTER estimate k+1 (not a smoothed one): x_s = Phi^-1 x_{k+1},
 * P_s = Phi^-1 P_{k+1} Phi^-T, Phi the STM of record k+1, inverted by LU (singular: an exactly zero pivot); the nominal stays record
 * k's.  The last estimate is copied unchanged.  Outputs, [capacity][..][n] like the records, each NULL to skip, NaN where the
 * reference has None or a record is past count:
 *   state     estimate.state() of the smoothed estimate (nominal + deviation, Cr clamped);
 *   deviation, covar (layout of the records);
 *   fs_ratio  filter-smoother ratios (state_f - state_s)_q / sqrt((P_f - P_s)_qq), NaN / +-inf kept; NaN for the last estimate;
 *   postfit   [capacity][2][n]: position k holds the reference's residuals[k+1] recomputed (off by one, as coded): real_obs of
 *             measurement k+1's window (0 for an absent type) minus measure_instantaneous(smoothed state k) at record k's EPOCH minus
 *             the station bias, slot = position of the type in the device's list as nyxb_od_outputs; NaN when record k+1 is a time
 *             update or the smoothed state is not visible.  The last position is the filter's own residual, unchanged: it is
 *             nyxb_od_outputs.postfit at the last record's tag and is left NaN here.
 *   status    [n] required: 0, the filter's status when filter_status[i] != 0 (not smoothed), NYXB_ERR_TOO_FEW_MEASUREMENTS for
 *             fewer than two records (the reference panics), NYXB_ERR_RECORDS_TRUNCATED when count > capacity,
 *             NYXB_ERR_SINGULAR_STM, or NYXB_ERR_EPHEMERIS; the batch is never aborted, and every output of a filter with a nonzero
 *             status is NaN.
 * stations, arc and cfg->msr_size must be those of the filter run (records tagged with another msr_size, or pointing at a measurement
 * or tracker that is not there, are NYXB_RC_BAD_ARG); of cfg only msr_size is read.  HOST pointers everywhere. */
typedef struct {
    double* state;               /* [capacity][9][n] or NULL */
    double* deviation;           /* [capacity][9][n] or NULL */
    double* covar;               /* [capacity][81][n] or NULL */
    double* fs_ratio;            /* [capacity][9][n] or NULL */
    double* postfit;             /* [capacity][2][n] or NULL */
    int32_t* status;             /* [n] */
} nyxb_smooth_outputs;

int32_t nyxb_od_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_ground_station* stations,
                             const nyxb_tracking_arc* arc, size_t n, const nyxb_od_records* rec, const int32_t* filter_status,
                             nyxb_smooth_outputs* out);

/* ---- Position-fix orbit determination (od/position: PositionDevice, GNSS-style X, Y, Z fixes of the spacecraft position in the
 * INTEGRATION frame of the estimate): the filter of nyxb_od_ekf_batch with a position device in place of the ground station.  As coded
 * in the reference:
 *   - the computed observation of the type at list position ii is component ii of the nominal position (trk_device.rs:76-83), the
 *     bias added by measure() and subtracted again (process/mod.rs:324-333): the bias cancels, so a bias in the data stays in the
 *     prefit;
 *   - H puts the type's unit row at its OWN component, X -> 0, Y -> 1, Z -> 2 (position/sensitivity.rs:55-75): a device listed
 *     [Y, X, Z] has an H that disagrees with its computed observation;
 *   - H starts from zeros: a window slot without a type, or with a type absent from the fix, keeps a zero row, its real observation
 *     is 0 and R keeps the type's variance (so its prefit is minus the computed observation);
 *   - windows follow process/mod.rs:270-296: msr_size 3 one window, msr_size 1 one per type (the 2nd and 3rd with Phi = I), msr_size 2
 *     with three types [t0, t1] then [t2] with a zero row and a zero R entry: S is singular and so is R, SingularNoiseRk
 *     (NYXB_ERR_PROP_MATH) at the first fix;
 *   - a zero variance gives SingularNoiseRk; there is no visibility test.
 * msr_size 3: the residual ratio from the Cholesky factor of S (falling back to that of R), the gain from the Cholesky solve
 * S K^T = (P H^T)^T (falling back to the closed-form 3x3 inverse); msr_size 1 and 2 take the ground station's arithmetic. */
typedef struct {
    int32_t n_types;             /* 1 to 3 */
    int32_t types[3];            /* NYXB_MSR_X / _Y / _Z, distinct, in the device's list order */
    double noise_var[3];         /* km^2, per list position */
    double bias[3];              /* km, per list position (cancels in the computed observation) */
} nyxb_position_device;

/* obs[(k*3 + t - NYXB_MSR_X)*n + i]: the fix component of type t of filter i at measurement k; NaN = the type is not in `msr.data`
 * (all three NaN: the measurement is not in filter i's arc). */
typedef struct {
    int64_t n_msr;
    const int64_t* epoch_ns;     /* [n_msr] ascending */
    const int32_t* tracker;      /* [n_msr] index into devices; < 0: unknown tracker */
    const double* obs;           /* [n_msr][3][n] */
} nyxb_position_arc;

/* Record tags of the position filter: window 0..2 and msr_size 1..3 (NYXB_OD_TAG has one bit for each) */
#define NYXB_OD_POS_TAG(k, w, rejected, msr_size) ((((int64_t)(k) * 4 + (w)) * 2 + (rejected)) * 4 + ((msr_size) - 1))
#define NYXB_OD_POS_TAG_MSR(tag) ((tag) >> 5)
#define NYXB_OD_POS_TAG_WINDOW(tag) (((tag) >> 3) & 3)
#define NYXB_OD_POS_TAG_REJECTED(tag) (((tag) >> 2) & 1)
#define NYXB_OD_POS_TAG_MSR_SIZE(tag) (((tag) & 3) + 1)

/* n filters over one schedule of fixes.  cfg as nyxb_od_ekf_batch with msr_size 1, 2 or 3.  out: nyxb_od_outputs whose per-measurement
 * arrays resid_ratio, prefit and postfit are [n_msr][3][n] (slot = position of the type in the device's list; the ratio of msr_size 1
 * in slot w, else slot 0).  rec: NULL, or the estimate records of nyxb_od_ekf_record_batch tagged by NYXB_OD_POS_TAG; `out` is
 * bit-identical either way.  NYXB_RC_BAD_ARG: a type other than X, Y, Z, a duplicate type, n_types outside 1..3, msr_size outside 1..3,
 * a NULL required pointer; NYXB_RC_UNSUPPORTED: the setups nyxb_propagate_batch_stm rejects.  Per-filter failures are statuses.
 * Kernel family as nyxb_od_ekf_batch.  HOST pointers everywhere. */
int32_t nyxb_od_position_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_position_device* devices,
                               const nyxb_position_arc* arc, size_t n, const double* state_soa, const double* consts_soa,
                               const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out,
                               const nyxb_od_records* rec);

/* ODSolution::smooth of position filters: the contract of nyxb_od_smooth_batch, with the records of nyxb_od_position_batch, and
 * out->postfit [capacity][3][n] recomputed through the position device (bias cancelling as in the filter). */
int32_t nyxb_od_position_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_position_device* devices,
                                      const nyxb_position_arc* arc, size_t n, const nyxb_od_records* rec, const int32_t* filter_status,
                                      nyxb_smooth_outputs* out);

/* ---- Angle tracking: a ground station that measures azimuth and elevation (degrees) next to range and Doppler, the filter of
 * nyxb_od_ekf_batch with nyxb_aer_station in place of nyxb_ground_station.  The observation slot of a type is its value, so the arc
 * (nyxb_tracking_arc) carries obs [n_msr][4][n] for these entry points: obs[(k*4 + t)*n + i].  As coded in the reference
 * (ground_station/trk_device.rs:158-208, msr/types.rs:102-117, msr/sensitivity.rs:188-226):
 *   - rho = r_sc - r_station in the integration frame; elevation = asin(rho . up / |rho|), the value the mask test reads; azimuth =
 *     atan2(rho . E, rho . N) mapped into [0, 360), E and N the geodetic east and north rotated like up.  The bias is subtracted as for
 *     range and Doppler; there is no wrap handling (an observed 359.99 deg against a computed 0.01 deg is a prefit of 359.98 deg);
 *   - h_tilde rows from the integration-frame rho (the reference's comment says "rotate back", the code does not), in rad/km while
 *     the observations are in degrees: azimuth [-dy, dx, 0] / (dx^2 + dy^2); elevation [-dx dz, -dy dz, .] / (r^2 sqrt(r^2 - dz^2)) and
 *     sqrt(dx^2 + dy^2) / r^2, r^2 = (sqrt(dx^2 + dy^2 + dz^2))^2.  Identity rows for types absent from the measurement;
 *   - windows as nyxb_od_ekf_batch: types w*msr_size .. of the station's list; [R, D, Az, El] at msr_size 2 gives [R, D] then
 *     [Az, El], at msr_size 1 four windows.  n_types need not be a multiple of msr_size (the last window is short, with an identity
 *     row, a zero R entry and a zero real observation, as the reference).  Range and Doppler are the ground station's arithmetic. */
typedef struct {
    double pos_fixed_km[3];
    double up_fixed[3];          /* unit local zenith in the body-fixed frame */
    double north_fixed[3];       /* unit geodetic north in the body-fixed frame: (-sin lat cos lon, -sin lat sin lon, cos lat) */
    double east_fixed[3];        /* unit geodetic east in the body-fixed frame: (-sin lon, cos lon, 0) */
    double elevation_mask_deg;
    nyxb_rotation rot;           /* as nyxb_ground_station */
    int32_t body;
    int32_t n_types;             /* 1 to 4 */
    int32_t types[4];            /* NYXB_MSR_RANGE / _DOPPLER / _AZIMUTH / _ELEVATION, distinct, in the device's list order */
    double noise_var[4];         /* per list position: km^2, km^2/s^2, deg^2 */
    double bias[4];              /* per list position */
    double body_radius_km;       /* as nyxb_ground_station */
} nyxb_aer_station;

/* n filters over one schedule.  cfg as nyxb_od_ekf_batch with msr_size 1 or 2; arc->obs [n_msr][4][n].  out: nyxb_od_outputs whose
 * per-measurement arrays resid_ratio, prefit and postfit are [n_msr][4][n] (prefit / postfit slot = position of the type in the
 * station's list; the ratio of window w in slot w).  rec: NULL, or the estimate records of nyxb_od_ekf_record_batch tagged by
 * NYXB_OD_POS_TAG; `out` is bit-identical either way.  NYXB_RC_BAD_ARG: a type outside 0..3, a duplicate type, n_types outside 1..4,
 * msr_size outside 1..2, a bad body index, a NULL required pointer; NYXB_RC_UNSUPPORTED: the setups nyxb_propagate_batch_stm rejects.
 * Per-filter failures are statuses.  Kernel family as nyxb_od_ekf_batch.  HOST pointers everywhere. */
int32_t nyxb_od_aer_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_aer_station* stations,
                          const nyxb_tracking_arc* arc, size_t n, const double* state_soa, const double* consts_soa,
                          const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec);

/* ODSolution::smooth of angle-tracking filters: the contract of nyxb_od_smooth_batch, with the records of nyxb_od_aer_batch, arc->obs
 * [n_msr][4][n] and out->postfit [capacity][4][n]. */
int32_t nyxb_od_aer_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_aer_station* stations,
                                 const nyxb_tracking_arc* arc, size_t n, const nyxb_od_records* rec, const int32_t* filter_status,
                                 nyxb_smooth_outputs* out);

/* ---- Spacecraft-to-spacecraft tracking (od/interlink: InterlinkTxSpacecraft): a transmitter spacecraft, known by its recorded
 * trajectory, measures the range and Doppler of the filtered spacecraft.  The filter of nyxb_od_ekf_batch with nyxb_interlink_tx in
 * place of nyxb_ground_station; obs, prefit, postfit and resid_ratio are [n_msr][2][n] with the ground station's slots and record tags
 * (NYXB_OD_TAG).  The transmitter's state is Traj::at of its recording (nyxb_traj_resample's arithmetic), evaluated at every use.
 * As coded in the reference (interlink/trk_device.rs:180-232, interlink/sensitivity.rs:50-172, process/mod.rs:300-330):
 *   - h_tilde runs BEFORE measure, with the transmitter at the nominal state's epoch (the measurement epoch): rho_tx = r_rx - r_tx and
 *     v_rx - v_tx, the range row [dr / rho_obs, 0 ...], the Doppler row [dv / rho_obs - rho_dot_obs dr / rho_obs^2, dr / rho_obs, 0 0 0]
 *     from the OBSERVED range and Doppler.  Identity rows for types absent from the measurement.  A Doppler row needs an observed range
 *     in the same measurement: without one the filter ends with NYXB_ERR_NO_RANGE;
 *   - the computed observation (measure_instantaneous at the propagator's epoch): the transmitter interpolated at that epoch, the line
 *     of sight tested against the body at the centre of the integration frame (Vallado's SIGHT, receiver first as for ground stations), range |rho| and
 *     range rate rho . v_rx / |rho| with v_rx the receiver's velocity in the integration frame: the transmitter's velocity is NOT
 *     subtracted (the reference's comment says otherwise), then minus the bias;
 *   - an epoch outside the transmitter's recording ends the filter with NYXB_ERR_TX_NO_DATA (not "not visible"), also when the line of
 *     sight would be blocked: h_tilde comes first.
 * No integration time, no aberration correction; the recording must be in the integration frame of the estimates.  Batch least squares
 * does not take interlink devices. */
typedef struct {
    int32_t tx;                  /* column of the transmitter's recording in the sink (0 .. n_tx - 1) */
    int32_t n_types;             /* 1 or 2 */
    int32_t types[2];            /* NYXB_MSR_RANGE / _DOPPLER, distinct, in the device's list order */
    double noise_var[2];         /* km^2, km^2/s^2 per list position */
    double bias[2];              /* per list position */
    double body_radius_km;       /* radius of the body at the centre of the integration frame, which can obstruct the link; <= 0: no test */
} nyxb_interlink_tx;

/* n filters over one schedule.  cfg as nyxb_od_ekf_batch with msr_size 1 or 2; n_types need not be a multiple of msr_size (a short last
 * window, as nyxb_od_aer_batch).  tx_sink: the n_tx transmitter recordings as nyxb_traj_sink lays them out for n = n_tx, HOST pointers:
 * record s of column j at epoch_ns[s*n_tx + j], state[(c*capacity + s)*n_tx + j], count[j] records (1 <= count <= capacity; ascending
 * or descending epochs as a propagation writes them).  rec: NULL, or the estimate records (NYXB_OD_TAG); `out` is bit-identical either
 * way.  NYXB_RC_BAD_ARG before any launch: a type other than Range / Doppler, a duplicate type, n_types outside 1..2, a column outside
 * the sink, a recording with count > capacity or count < 1, msr_size outside 1..2, a NULL required pointer; NYXB_RC_UNSUPPORTED: the
 * setups nyxb_propagate_batch_stm rejects.  Per-filter failures are statuses.  Kernel family as nyxb_od_ekf_batch. */
int32_t nyxb_od_interlink_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_interlink_tx* devices,
                                size_t n_tx, const nyxb_traj_sink* tx_sink, const nyxb_tracking_arc* arc, size_t n,
                                const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns, const double* covar0_soa,
                                const nyxb_od_outputs* out, const nyxb_od_records* rec);

/* ODSolution::smooth of interlink filters: the contract of nyxb_od_smooth_batch with the records of nyxb_od_interlink_batch, the
 * residual recomputed with the transmitter at record k's epoch; a record epoch outside the recording gives NYXB_ERR_TX_NO_DATA. */
int32_t nyxb_od_interlink_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_interlink_tx* devices,
                                       size_t n_tx, const nyxb_traj_sink* tx_sink, const nyxb_tracking_arc* arc, size_t n,
                                       const nyxb_od_records* rec, const int32_t* filter_status, nyxb_smooth_outputs* out);

/* ---- Covariance mapping over an ensemble: n independent `KalmanODProcess::predict_until` runs (od/process/mod.rs:440-486) in ONE
 * kernel launch.  Record 0 is the initial estimate; then chunks of cfg->max_step_ns (`for_duration(max_step)`: adaptive steps, the
 * last one cut to land on the chunk end; the adaptive step carries over, and the first chunk starts from opts.init_step: no
 * set_step(max_step) here), each closed by `KalmanFilter::time_update` (P = Phi P Phi^T + SNC; CKF deviation Phi x, EKF zero) and an
 * STM reset, until the first chunk end at or after end_epoch_ns[i].  So record k sits at epoch0_ns[i] + k*max_step_ns exactly, a run
 * has 1 + max(1, ceil((end - epoch0) / max_step)) records, the last may overshoot the end by up to max_step - 1 ns, and an end at
 * or before the start gives two records.
 * Of cfg only variant, max_step_ns and the snc_* fields are read.  max_step_ns <= 0 is rejected with NYXB_RC_BAD_ARG (the reference
 * does not check it and would loop forever).  The setups nyxb_propagate_batch_stm rejects return NYXB_RC_UNSUPPORTED.  A propagation
 * error ends that run with its status; the records written up to then stay valid.  Kernel family as nyxb_od_ekf_batch. */
typedef struct {
    double* state_soa;           /* [9][n]  final nominal state */
    int64_t* epoch_ns;           /* [n]     epoch of the last record */
    double* covar_soa;           /* [81][n] final covariance, (r,c) at [(c*9+r)*n + i] */
    double* state_dev_soa;       /* [9][n]  final state deviation, or NULL */
    nyxb_details* details;       /* [n] or NULL: n_steps / n_rhs over the whole prediction */
    int32_t* status;             /* [n] */
    int64_t capacity;            /* records kept per run; records k >= capacity are dropped (as nyxb_traj_sink) */
    double* rec_state;           /* [capacity][9][n] or NULL: estimate.state() = nominal + deviation (Cr clamped), [(k*9 + r)*n + i] */
    double* rec_covar;           /* [capacity][81][n] or NULL: covariance, (r,c) at [(k*81 + c*9 + r)*n + i] */
    int64_t* rec_count;          /* [n] or NULL: records produced by run i (kept or not) */
} nyxb_predict_outputs;

/* state_soa/consts_soa/epoch0_ns/covar0_soa as in nyxb_od_ekf_batch (initial_estimate.nominal_state, .covar);
 * state_dev0_soa [9][n] initial state deviation (initial_estimate.state_deviation) or NULL = 0; HOST pointers everywhere. */
int32_t nyxb_od_predict_batch(nyxb_engine* eng, const nyxb_od_config* cfg, size_t n,
                              const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                              const int64_t* end_epoch_ns, const double* covar0_soa, const double* state_dev0_soa,
                              const nyxb_predict_outputs* out);

/* ---- Batch least squares over an ensemble: n independent `BatchLeastSquares::estimate` runs (od/blse/mod.rs:146-446) in ONE kernel
 * launch.  The n problems share the schedule and the stations; each has its own initial guess, epoch and observation set (arc->obs,
 * both NaN: the measurement is not in problem i's arc, as `rejected`).  Per iteration, as coded: a new STM propagation from the current
 * estimate at opts.init_step (no set_step(max_step)); the information matrix starts at the IDENTITY; the walk to each measurement takes
 * chunks of min(time left, current step, max_step); after each chunk stm_acc = Phi(t, t0) * stm_acc, where the STM is never reset inside
 * the iteration, so stm_acc is a product of cumulative STMs; each measurement type is its own scalar residual in the station's type
 * order, computed without bias (measure_instantaneous(state, None)), skipped when not visible; rms = sqrt(sum W dy^2 / count) where count
 * is every measurement present in problem i (invisible, unknown-tracker and at-or-before-epoch ones included).  A measurement type the
 * station does not carry is skipped.
 * Per-problem failures are statuses and never abort the batch: NYXB_ERR_TOO_FEW_MEASUREMENTS (count < 2), NYXB_ERR_INVALID_MEASUREMENT,
 * NYXB_ERR_SINGULAR_INFORMATION (normal equations only), or a propagation status.
 * Earlier or stricter than the reference (NYXB_RC_BAD_ARG for the whole call): max_step_ns <= 0 (the reference would loop forever),
 * max_iterations < 0 (a usize there), a station noise variance <= 0 (the reference fails with SingularNoiseRk at the first measurement
 * of that station), and, for Levenberg-Marquardt, a lambda setting <= 0 (unchecked there).  The setups nyxb_propagate_batch_stm rejects
 * return NYXB_RC_UNSUPPORTED.  Kernel family as nyxb_od_ekf_batch. */
enum nyxb_bls_solver { NYXB_BLS_NORMAL_EQUATIONS = 0, NYXB_BLS_LEVENBERG_MARQUARDT = 1 };  /* od/blse/mod.rs BLSSolver */

typedef struct {
    int32_t solver;              /* enum nyxb_bls_solver; default NORMAL_EQUATIONS */
    int32_t max_iterations;      /* default 10 */
    double tolerance_pos_km;     /* convergence: |dx[0..3]| below this; default 1e-4 */
    int64_t max_step_ns;         /* default 30 s */
    int64_t epoch_precision_ns;  /* default 1 us */
    double lm_lambda_init;       /* default 10 */
    double lm_lambda_decrease;   /* default 10 */
    double lm_lambda_increase;   /* default 10 */
    double lm_lambda_min;        /* default 1e-12 */
    double lm_lambda_max;        /* default 1e12 */
    int32_t lm_use_diag_scaling; /* default 1 */
    int32_t _pad;
} nyxb_bls_config;

typedef struct {
    double* state_soa;           /* [9][n] estimated state (the last accepted correction applied; Cr clamped), or NULL */
    int64_t* epoch_ns;           /* [n] its epoch (the guess epoch), or NULL */
    double* covar_soa;           /* [81][n] (r,c) at [(c*9+r)*n + i], or NULL: the inverse of the information matrix of the last
                                    accepted iteration (UDU^T), I when that factorisation fails, zeros when no iteration was accepted */
    int32_t* iterations;         /* [n] or NULL */
    double* final_rms;           /* [n] or NULL: the RMS at the last accepted linearisation point; DBL_MAX when none */
    double* final_corr_pos_km;   /* [n] or NULL: DBL_MAX after a rejected Levenberg-Marquardt step or when none ran */
    int32_t* converged;          /* [n] or NULL: 0 / 1 */
    nyxb_details* details;       /* [n] or NULL: steps / RHS evaluations over all iterations */
    int32_t* status;             /* [n] */
} nyxb_bls_outputs;

/* state_soa/consts_soa/epoch0_ns as in nyxb_od_ekf_batch (the initial guesses); HOST pointers everywhere. */
int32_t nyxb_od_bls_batch(nyxb_engine* eng, const nyxb_bls_config* cfg,
                          int32_t n_stations, const nyxb_ground_station* stations,
                          const nyxb_tracking_arc* arc, size_t n,
                          const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                          const nyxb_bls_outputs* out);

/* `BatchLeastSquares::evaluate` (od/blse/mod.rs:450-541): the RMS of each state over the arc, the same pass without the STM product;
 * NYXB_ERR_TOO_FEW_MEASUREMENTS when problem i has no measurement.  rms [n] may be NULL; status [n] is required.  Of cfg only
 * max_step_ns and epoch_precision_ns are read. */
int32_t nyxb_od_bls_evaluate_batch(nyxb_engine* eng, const nyxb_bls_config* cfg,
                                   int32_t n_stations, const nyxb_ground_station* stations,
                                   const nyxb_tracking_arc* arc, size_t n,
                                   const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                                   double* rms, int32_t* status);

/* ---- On-device Monte Carlo dispersions (next row (f)-4): `MvnSpacecraft::sample` (mc/multivariate.rs:298-331) for the
 * runs [first_index, first_index + n): state_i = template + (sqrt_s_v * z_i + mean), z_i ~ N(0, I_9) drawn from a
 * counter-based stream keyed by (seed, run index) — Philox4x32-10 + Box-Muller, see nyx_b200/csrc/nyxb_mvn.cu — so that a
 * run's draw does not depend on how the ensemble is sharded (the reference's serial Pcg64Mcg + ziggurat stream,
 * mc/montecarlo.rs:277-296, is not reproduced: DESIGN.md §3).
 *  template_state[9], mean[9] (NULL = 0), sqrt_s_v[81] row-major (V * sqrt(S) of the covariance's SVD, multivariate.rs:237-247)
 *  out_state_soa [9][n], out_dispersion_soa [9][n] or NULL (the x_i themselves).
 * `_dev`: ONLY out_state_soa / out_dispersion_soa are device pointers (stream-ordered launch); template_state, mean and sqrt_s_v
 * are HOST pointers in both variants — they are read on the host into the kernel's parameter block. */
int32_t nyxb_mvn_sample(int32_t device, uint64_t seed, uint64_t first_index, size_t n,
                        const double* template_state, const double* mean, const double* sqrt_s_v,
                        double* out_state_soa, double* out_dispersion_soa);
int32_t nyxb_mvn_sample_dev(int32_t device, uint64_t seed, uint64_t first_index, size_t n,
                            const double* template_state, const double* mean, const double* sqrt_s_v,
                            double* out_state_soa, double* out_dispersion_soa, void* cuda_stream);

/* ---- The reference's own dispersion stream (row a2; host code, no device needed): `MonteCarlo::generate_states`
 * (mc/montecarlo.rs:277-296) = one serial `Pcg64Mcg::new(seed)` (seed: u128 = seed_hi * 2^64 + seed_lo) feeding rand_distr's ziggurat
 * `StandardNormal`, nine normals per run, the first `skip` runs dropped.  out_z [n][9] row-major: x_i = sqrt_s_v z_i + mean
 * (multivariate.rs:298-302).  Pcg64Mcg is pinned on the generator's official known-answer vector; the ziggurat tables are regenerated
 * from the published formulas (see nyx_b200/csrc/nyxb_rng.cu). */
int32_t nyxb_reference_normals(uint64_t seed_lo, uint64_t seed_hi, uint64_t skip, size_t n, double* out_z);
int32_t nyxb_pcg64mcg_u64(uint64_t seed_lo, uint64_t seed_hi, size_t n, uint64_t* out);   /* raw generator output (known-answer tests) */
int32_t nyxb_ziggurat_tables(double* x257, double* f257);                                  /* the layer tables (inspection) */

/* ---- Impulsive differential correction: `Targeter::try_achieve_from` / `try_achieve_fd` (md/opti/raphson_finite_diff.rs:41-747)
 * restricted to impulsive variables, for n problems that share the correction and achievement epochs. */
enum nyxb_tgt_vary { NYXB_VARY_POSITION_X = 0, NYXB_VARY_POSITION_Y = 1, NYXB_VARY_POSITION_Z = 2,
                     NYXB_VARY_VELOCITY_X = 3, NYXB_VARY_VELOCITY_Y = 4, NYXB_VARY_VELOCITY_Z = 5 };
/* Objective parameters: the orbital elements, evaluated with mu = nyxb_dynamics.mu_central_km3_s2 (angles in degrees) */
enum nyxb_tgt_param {
    NYXB_TGT_X = 0, NYXB_TGT_Y, NYXB_TGT_Z, NYXB_TGT_VX, NYXB_TGT_VY, NYXB_TGT_VZ, NYXB_TGT_RMAG, NYXB_TGT_VMAG, NYXB_TGT_SMA,
    NYXB_TGT_ECC, NYXB_TGT_INC, NYXB_TGT_RAAN, NYXB_TGT_AOP, NYXB_TGT_TA, NYXB_TGT_AOL, NYXB_TGT_TLONG, NYXB_TGT_PERIOD,
    NYXB_TGT_ENERGY, NYXB_TGT_HMAG, NYXB_TGT_APOAPSIS, NYXB_TGT_PERIAPSIS, NYXB_TGT_C3, NYXB_TGT_DECLINATION,
    NYXB_TGT_N_PARAMS
};
/* Correction frame of the variables: none (inertial, r and v), VNC (columns v^, h^, v^ x h^) or RIC (columns r^, h^ x r^, h^),
 * each the local-to-inertial DCM of the state the correction is applied to. */
enum nyxb_tgt_frame { NYXB_TGT_FRAME_NONE = 0, NYXB_TGT_FRAME_VNC = 1, NYXB_TGT_FRAME_RIC = 2 };

typedef struct {                /* `Variable` (md/opti/target_variable.rs) */
    int32_t component;          /* enum nyxb_tgt_vary */
    int32_t pad;
    double perturbation;        /* finite and nonzero */
    double init_guess;
    double max_step;            /* >= 0 */
    double max_value;           /* >= 0 */
    double min_value;           /* <= max_value */
} nyxb_tgt_variable;            /* 48 bytes */

typedef struct {                /* `Objective` (md/objective.rs) */
    int32_t parameter;          /* enum nyxb_tgt_param */
    int32_t pad;
    double desired;
    double tolerance;
    double multiplicative_factor;
    double additive_factor;
} nyxb_tgt_objective;           /* 40 bytes */

typedef struct {
    int32_t n_vars;             /* 1..6; duplicate components are allowed and add up */
    int32_t n_objs;             /* 1..6 */
    int32_t correction_frame;   /* enum nyxb_tgt_frame; a position variable with a frame is NYXB_RC_BAD_ARG (FrameError) */
    int32_t iterations;         /* >= 0: at most iterations + 1 nominal evaluations */
    nyxb_tgt_variable vars[6];
    nyxb_tgt_objective objs[6];
} nyxb_target_config;           /* 544 bytes */

/* Problem i propagates state i from epoch0_ns[i] to correction_epoch_ns, applies the initial guesses, then iterates: the nominal and
 * one perturbed state per variable are propagated to achievement_epoch_ns (from opts.init_step), the objectives are evaluated and the
 * step J^+ err is clipped and applied, as the reference does.  The reference repeats the perturbed propagations once per objective;
 * they are deterministic, so each runs once per iteration here.
 *   out_corrected_soa [9][n]: the start state at the correction epoch plus the total correction, applied once with the DCM of that
 *                             start state (not the iterated state; the two differ with a frame and several iterations)
 *   out_achieved_soa  [9][n]: the nominal final state of the last iteration, with the start state's mass and coefficients
 *   out_correction [n_vars][n], out_errors [n_objs][n], out_iterations [n]: the last iteration's values, also on failure
 *   out_status [n]: 0 converged, NYXB_ERR_TGT_*, or the status of a failed propagation (the reference panics when a perturbed one
 *                   fails); the warn flag of every propagation of the problem is OR-ed in.  The batch is never aborted.
 * One kernel family and lane count is picked for the whole call, at the size of the first iteration's launch (n (n_vars + 1)), so a
 * problem's result does not depend on how many others still iterate.  Launches: 3 before the loop, then 4 per iteration (staging of
 * the (n_vars + 1) start states, one propagation over every active problem, the update, the stable compaction of the active
 * problems), then 1 to write the outputs; each iteration reads back 4 bytes (the active count).
 * NYXB_RC_BAD_ARG before any launch: counts out of range, an unknown component, parameter or frame, a position variable with a frame,
 * max_step < 0, max_value < 0, min_value > max_value, a zero or non-finite perturbation, iterations < 0, NULL pointers.
 * NYXB_RC_UNSUPPORTED: an integration frame other than the states' own (opts.state_center != 0).  HOST pointers everywhere. */
int32_t nyxb_target_batch(nyxb_engine* eng, const nyxb_target_config* cfg, size_t n,
                          const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                          int64_t correction_epoch_ns, int64_t achievement_epoch_ns,
                          double* out_corrected_soa, double* out_achieved_soa,
                          double* out_correction, double* out_errors,
                          int32_t* out_iterations, int32_t* out_status);

/* Tuning / introspection. */
/* Kernel families behind nyxb_propagate_batch*.  AUTO picks by mode, degree and ensemble size:
 *   THREAD      one thread per trajectory (no or low-degree gravity field; STRICT and FAST)
 *   COOP        8 / 16 / 32 lanes of a warp per trajectory, harmonic sum split by columns over the lanes (STRICT and FAST)
 *   TRANSPOSED  FAST only, degree 8..70: one CTA per set of 32 trajectories, lane = trajectory, warp = column position, persistent
 *               CTAs with (set, time-slice) tickets — the kernel of large harmonics-dominated ensembles (>= 1 024 trajectories, field of degree 8..70; smaller ensembles go to the lane-cooperative kernel) */
enum nyxb_kernel { NYXB_KERNEL_AUTO = 0, NYXB_KERNEL_THREAD = 1, NYXB_KERNEL_COOP = 2, NYXB_KERNEL_TRANSPOSED = 3 };
int32_t nyxb_engine_set_kernel(nyxb_engine* eng, int32_t kernel);          /* enum nyxb_kernel; NYXB_RC_UNSUPPORTED if the setup cannot use it */
int32_t nyxb_engine_last_kernel(const nyxb_engine* eng);                   /* family used by the last propagation launch */
/* nyxb_propagate_batch_stm sets it to THREAD (one thread per trajectory, STRICT and FAST).  nyxb_od_ekf_batch,
 * nyxb_od_predict_batch, nyxb_od_bls_batch and nyxb_od_bls_evaluate_batch set it to COOP when they ran the warp-cooperative kernel (FAST, field of degree >= 8, kernel not forced to
 * THREAD), else to THREAD. */
/* TRANSPOSED kernel: step attempts per time slice (default 64) and an upper bound on the persistent CTAs (0 = SMs x occupancy).
 * Sets are only parked when there are more sets than CTAs. */
int32_t nyxb_engine_set_tx_tuning(nyxb_engine* eng, int32_t slice_attempts, int32_t max_ctas);
int32_t nyxb_engine_set_tx_positions(nyxb_engine* eng, int32_t positions);   /* walker warps per set: 0 = by degree, 8, 10, 16 */
/* 0 = auto, 1, 8, 16, 32.  STRICT mode keeps each trajectory's Legendre triangle in shared memory, which limits the forced lane
 * counts by degree: 8 lanes up to degree 50, 16 up to 75, 32 up to 96.  Above that the call returns NYXB_RC_UNSUPPORTED and the
 * setting is unchanged.  The automatic choice always fits. */
int32_t nyxb_engine_set_lanes(nyxb_engine* eng, int32_t lanes_per_trajectory);
int32_t nyxb_engine_get_lanes(const nyxb_engine* eng);
int64_t nyxb_engine_launch_count(const nyxb_engine* eng); /* kernels launched so far */
double nyxb_engine_last_kernel_ms(const nyxb_engine* eng); /* CUDA-event time of the last launch (host API only) */

/* Register-resident DFMA throughput probe: returns achieved FP64 TFLOP/s (FMA = 2 flop)
 * on `device`; the FP64 roof that bench.py reports against. */
double nyxb_measure_fp64_tflops(int32_t device, int32_t iters);

/* Host-only inspection of the cooperative kernel's coefficient table (no device needed): the column -> lane
 * schedule and the packed records for `lanes` in {8,16,32}.  Two-call pattern: with recs == NULL only the sizes are
 * returned.  Layouts: recs [(L+2)/2 pairs][5 pieces][lanes][2], col_start / col_m [lanes][kmax], colseed [N+2][4]
 * (see nyx_b200/csrc/nyxb_coop.h); col_m = N + 2 marks a stop column (zero seed, no records) that ends a column's recursion
 * before a long idle gap of its lane.  Used by the CPU tests to check the table algebra against a direct evaluation. */
int32_t nyxb_coop_table_dump(const nyxb_gravity_field* field, int32_t lanes, int32_t* out_L, int32_t* out_kmax,
                             double* recs, int32_t* col_start, int32_t* col_m, double* colseed);

/* Same for the transposed kernel (`positions` in {8,10,16}): recA [(n_rec+1)][4], recK [n_rec+2], colseed [N+2][4],
 * sched [positions][2 + 2*kmax] = {first record, columns, (m, entries) per column} (see nyx_b200/csrc/nyxb_tx.h). */
int32_t nyxb_tx_table_dump(const nyxb_gravity_field* field, int32_t positions, int32_t* out_n_rec, int32_t* out_kmax,
                           double* recA, double* recK, double* colseed, int32_t* sched);

int32_t nyxb_abi_version(void);
const char* nyxb_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* NYXB_H */
