// nyxb_od.cuh — device-side data model of the STM / sequential-filter path (SURVEY.md §8 (f)-2), shared by
// nyxb_od.cu (kernels, built STRICT and FAST) and nyxb_api.cu (host packing).
#pragma once
#include "nyxb_device.cuh"

struct DevStation {
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
    int n_types;
    int types[3];
    double noise_var[3], bias[3];
};

// Dev: the tracker kind (DevStation, or DevPosDevice for position fixes, whose observations are [m][3][n])
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
    const double* obs;             // [m][2][n] ([m][3][n] for position fixes)
    const double* covar0;          // [81][n]
    // outputs (any of the per-measurement ones may be null)
    double* covar;                 // [81][n]
    double* state_dev;             // [9][n] or null
    double* ratio;                 // [m][2][n] (slots: as obs)
    double* prefit;                // [m][2][n]
    double* postfit;               // [m][2][n]
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
    const double* obs;             // [m][2][n]
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
    double* postfit;               // [cap][2][n] or null
    long long* err_key;            // [n] -1, or the largest 2k + (1: singular Phi, 0: ephemeris) among the failing estimates k
};
struct DevSmooth : DevSmoothT<DevStation> {};

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

extern "C" cudaError_t nyxb_launch_stm_strict(const DevSetup*, size_t, const double*, const double*, const long long*, long long,
                                              long long*, const double*, double*, long long*, double*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_stm_fast(const DevSetup*, size_t, const double*, const double*, const long long*, long long,
                                            long long*, const double*, double*, long long*, double*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_od_strict(const DevSetup*, const DevOd*, size_t, const double*, const double*, const long long*,
                                             double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_od_fast(const DevSetup*, const DevOd*, size_t, const double*, const double*, const long long*,
                                           double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_pred_strict(const DevSetup*, const DevOd*, size_t, const double*, const double*, const long long*,
                                               const long long*, const double*, const OdRecords*, long long*, double*, long long*,
                                               nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_pred_fast(const DevSetup*, const DevOd*, size_t, const double*, const double*, const long long*,
                                             const long long*, const double*, const OdRecords*, long long*, double*, long long*,
                                             nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_od_rec_strict(const DevSetup*, const DevOd*, const OdEstRecords*, size_t, const double*, const double*,
                                                 const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_od_rec_fast(const DevSetup*, const DevOd*, const OdEstRecords*, size_t, const double*, const double*,
                                               const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_bls_strict(const DevSetup*, const DevOd*, const DevBls*, size_t, const double*, const double*,
                                              const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_bls_fast(const DevSetup*, const DevOd*, const DevBls*, size_t, const double*, const double*,
                                            const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_smooth(const DevSetup*, const DevSmooth*, size_t, cudaStream_t);

// position fixes (DevOdT<DevPosDevice>): the same filter and smoother, three observation slots
struct DevOdPos : DevOdT<DevPosDevice> {};
struct DevSmoothPos : DevSmoothT<DevPosDevice> {};
extern "C" cudaError_t nyxb_launch_odpos_strict(const DevSetup*, const DevOdPos*, const OdEstRecords*, size_t, const double*, const double*,
                                                const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_odpos_fast(const DevSetup*, const DevOdPos*, const OdEstRecords*, size_t, const double*, const double*,
                                              const long long*, double*, long long*, nyxb_details*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_smooth_pos(const DevSetup*, const DevSmoothPos*, size_t, cudaStream_t);
