// nyxb_od.cuh — device-side data model of the STM / sequential-filter path (SURVEY.md §8 (f)-2), shared by
// nyxb_od.cu (kernels, built STRICT and FAST) and nyxb_api.cu (host packing).
#pragma once
#include "nyxb_device.cuh"
#include "nyxb_hermite.h"

#define ODC_KMAX 4           // columns of the Legendre triangle per lane of a warp kernel (>= the host's deal over 32 lanes: 4 at N = 96)

struct GroundTrk;            // the measurement model of each tracker kind (nyxb_od_device.cuh)
struct PosTrk;
struct AerTrk;
struct LinkTrk;

// NS: the observation slots of one measurement (obs is [m][NS][n])
struct DevStation {
    static constexpr int NS = 2;
    using Trk = GroundTrk;
    double pos[3], up[3];
    double mask_deg;
    DevRotation rot;
    int body, n_types;
    int types[2];
    double noise_var[2], bias[2];
    double body_radius;
};

// GNSS-style position fixes (od/position): X, Y, Z of the spacecraft in the integration frame.  types[] in the device's list order,
// as NYXB_MSR_X.. (the observation slot of a type is type - NYXB_MSR_X); noise_var / bias per list position.
struct DevPosDevice {
    static constexpr int NS = 3;
    using Trk = PosTrk;
    int n_types;
    int types[3];
    double noise_var[3], bias[3];
};

// A ground station that may also measure azimuth and elevation: DevStation's geometry plus the body-fixed geodetic north and east,
// with up to four types (range, Doppler, azimuth, elevation).  The observation slot of a type is its value (obs is [m][4][n]);
// noise_var / bias per list position.
struct DevAerStation {
    static constexpr int NS = 4;
    using Trk = AerTrk;
    double pos[3], up[3], north[3], east[3];
    double mask_deg;
    DevRotation rot;
    int body, n_types;
    int types[4];
    double noise_var[4], bias[4];
    double body_radius;
};

// An interlink transmitter (od/interlink): a spacecraft whose state is Traj::at of column `col` of a recording shared by every device
// of the call (tx, tx_n columns).  Types Range / Doppler in the device's list order; the observation slot of a type is its value, as
// for DevStation (obs is [m][2][n]); noise_var / bias per list position.
struct DevLink {
    static constexpr int NS = 2;
    using Trk = LinkTrk;
    NyxbTrajView tx;
    long long tx_n;
    int col, n_types;
    int types[2];
    double noise_var[2], bias[2];
    double body_radius;            // the body at the integration frame's centre; <= 0: no line-of-sight test
};

// Dev: the tracker kind (DevStation, DevPosDevice for position fixes, whose observations are [m][3][n], or DevAerStation, [m][4][n])
template <class Dev>
struct DevOdT {
    int variant, msr_size;
    double reject;                 // < 0: no sigma rejection
    long long max_step_ns, eps_ns;
    int snc_enabled, snc_frame;
    double snc_diag[3];
    long long snc_disable_ns;
    int n_stations;
    const Dev* stations;
    long long n_msr;
    const long long* msr_epoch;    // [m]
    const int* msr_tracker;        // [m]
    const double* obs;             // [m][Dev::NS][n]
    const double* covar0;          // [81][n]
    // outputs (any of the per-measurement ones may be null)
    double* covar;                 // [81][n]
    double* state_dev;             // [9][n] or null
    double* ratio;                 // [m][Dev::NS][n] (slots: as obs)
    double* prefit;                // [m][Dev::NS][n]
    double* postfit;               // [m][Dev::NS][n]
    int* flags;                    // [m][n]
    double* est_state;             // [m][9][n]
    double* est_cov;               // [m][9][n]
};
struct DevOd : DevOdT<DevStation> {};

// Records of a covariance prediction (KalmanODProcess::predict_until): record k holds estimate.state() (nominal + deviation, Cr
// clamped to [0, 2]: `Spacecraft + OVector<9>`, cosmic/spacecraft.rs:713-728) at [(k*9 + r)*n + i] and the covariance, (r, c) at
// [(k*81 + c*9 + r)*n + i].  Records k >= cap are dropped; either array may be null.
struct OdRecords {
    long long cap;
    double* state;   // [cap][9][n] or null
    double* covar;   // [cap][81][n] or null
};

// Estimate records of a filter run (nyxb_od_records, include/nyxb.h): one record per entry the reference pushes to
// ODSolution.estimates, in push order.  Record k of filter i: epoch [k*n + i], tag [k*n + i] (-1: time update, else the measurement,
// window, rejection and msr_size bits of NYXB_OD_TAG in nyxb.h), nominal state and deviation [(k*9 + r)*n + i], covariance and the STM
// from the previous record, (r, c) at [(k*81 + c*9 + r)*n + i].  Records k >= cap are dropped; count[i] counts all of them.  Every
// array is non-null.
struct OdEstRecords {
    long long cap;
    long long* epoch;    // [cap][n]
    long long* tag;      // [cap][n]
    double* nominal;     // [cap][9][n]
    double* dev;         // [cap][9][n]
    double* covar;       // [cap][81][n]
    double* stm;         // [cap][81][n]
    long long* count;    // [n]
};

// ODSolution::smooth over the records of n filters (nyxb_smooth.cu); Dev as DevOdT
template <class Dev>
struct DevSmoothT {
    int msr_size;
    int n_stations;
    const Dev* stations;
    const int* msr_tracker;        // [m]
    const double* obs;             // [m][Dev::NS][n]
    long long cap;
    const long long* epoch;        // records, layout of OdEstRecords (nyxb_od.cuh)
    const long long* tag;
    const double* nominal;
    const double* dev;
    const double* covar;
    const double* stm;
    const long long* count;        // [n]
    const int* pre_status;         // [n] nonzero: filter i is not smoothed (failed filter, too few or truncated records)
    double* state;                 // [cap][9][n] or null, NaN-filled by the host
    double* sdev;                  // [cap][9][n] or null
    double* scov;                  // [cap][81][n] or null
    double* ratio;                 // [cap][9][n] or null
    double* postfit;               // [cap][Dev::NS][n] or null
    long long* err_key;            // [n] -1, or the largest 2k + (1: singular Phi, 0: ephemeris) among the failing estimates k
};

// Batch least squares (BatchLeastSquares::estimate / evaluate, od/blse/mod.rs:146-541).  The schedule, stations, observations,
// max_step and epoch precision come from DevOd; this holds the solver settings and the per-problem outputs ([n], covar [81][n]).
struct DevBls {
    int evaluate;                  // 1: evaluate() (the RMS of the given state), 0: estimate()
    int solver;                    // enum nyxb_bls_solver
    int max_iter;
    int lm_diag;                   // lm_use_diag_scaling
    double tol_pos_km;
    double lm_init, lm_dec, lm_inc, lm_min, lm_max;
    double* covar;                 // (r, c) at [(c*9 + r)*n + i]
    int* iters;
    double* rms;
    double* corr_pos_km;
    int* converged;
};

// ------------------------------------------------------------------------- OD jobs: what one launch of nyxb_k_od / nyxb_k_od_coop runs
// Each job holds what is specific to it; od_run (nyxb_od_arc.cuh) runs it.  NS: the observation slots of the gain scratch.

// STM propagation to end_epoch (nyxb_propagate_batch_stm); per-thread kernels only
struct OdStmJob {
    static constexpr int NS = 2;   // no filter storage is used
    long long end_epoch;
    long long* step_io;            // [n] initial step in, last step out, or null
    const double* stm_in;          // [81][n] or null (identity)
    double* out_stm;               // [81][n]
};

// the filter (KalmanODProcess::process_arc) over the trackers Dev; REC: every estimate also recorded into er
template <class Dev, bool REC>
struct OdFilterJob {
    static constexpr int NS = Dev::NS;
    DevOdT<Dev> od;
    OdEstRecords er;
};
template <class Dev>
struct OdFilterJob<Dev, false> {
    static constexpr int NS = Dev::NS;
    DevOdT<Dev> od;
};

// covariance prediction (KalmanODProcess::predict_until)
struct OdPredictJob {
    static constexpr int NS = DevStation::NS;
    DevOd od;
    const long long* end_epoch;    // [n]
    const double* dev0;            // [9][n] initial deviation or null
    OdRecords rec;
    long long* rec_count;          // [n] or null
};

// batch least squares (BatchLeastSquares::estimate / evaluate)
struct OdBlsJob {
    static constexpr int NS = DevStation::NS;
    DevOd od;
    DevBls bl;
};

// the per-filter arrays every job reads and writes (device pointers): state [9][n], consts [4][n], epoch0 [n]; out_details may be null
struct OdIo {
    const double* state;
    const double* consts;
    const long long* epoch0;
    double* out_state;
    long long* out_epoch;
    nyxb_details* out_details;
    int* out_status;
};

// Launchers.  The per-thread kernels are built twice (nyxb_od.cu), STRICT and FAST, each in its own namespace so that the two
// builds' instantiations of one kernel template stay distinct symbols; the warp kernels (nyxb_od_coop.cu) are FAST only.
namespace nyxb_od_strict {
template <class Job> cudaError_t launch(const DevSetup& S, const Job& job, size_t n, const OdIo& io, cudaStream_t st);
}
namespace nyxb_od_fast {
template <class Job> cudaError_t launch(const DevSetup& S, const Job& job, size_t n, const OdIo& io, cudaStream_t st);
}
template <class Job> cudaError_t nyxb_od_coop_launch(const DevSetup& S, const Job& job, const int* cols, size_t n, const OdIo& io, cudaStream_t st);
// ODSolution::smooth over the records of the filters of tracker kind Dev (nyxb_smooth.cu)
template <class Dev> cudaError_t nyxb_smooth_launch(const DevSetup& S, const DevSmoothT<Dev>& sm, size_t n, cudaStream_t st);
