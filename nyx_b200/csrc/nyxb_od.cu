// nyxb_od.cu — state-transition-matrix propagation and the sequential Kalman filter, one CUDA thread per trajectory
// (SURVEY.md §8 (f)-2; BASELINE configs[4]).  The whole arc of a filter — propagation of the nominal state and the STM
// between measurements, time updates, measurement updates, state replacement — runs inside ONE kernel launch; state,
// STM, covariance and stage data stay in registers / L1-resident local memory, HBM sees the inputs once and the
// per-measurement residual records as coalesced [m][..][n] stores.  The propagation and the filter loop are the templates of
// nyxb_od_arc.cuh; this file gives them the per-thread backend (ThreadB) and holds the kernels and their launchers.
//
// Built twice like nyxb_kernels.cu: -DNYXB_STRICT=1 -fmad=false (same operation order as oracle/nyx_oracle_od.c for
// the dynamics) and -DNYXB_STRICT=0 -fmad=true.
//
// Reference behaviour (paths relative to /root/reference/nyx-core/src):
//   SpacecraftDynamics::eom `Some(stm)` branch / dual_eom      dynamics/spacecraft.rs:203-227, 312-363
//   OrbitalDynamics::dual_eom, PointMasses::gradient           dynamics/orbital.rs:116-172, 249-307
//   GravityField::gradient                                     dynamics/gravity_field.rs:273-431
//   SolarPressure::gradient                                    dynamics/solarpressure.rs:167-233
//   PropInstance::{propagate, single_step, derive}             propagators/instance.rs:87-262, 343-493
//   KalmanODProcess::process_arc                               od/process/mod.rs:128-497
//   KalmanFilter::{time_update, measurement_update}            od/kalman/filtering.rs:59-316
//   BatchLeastSquares::{estimate, evaluate}                    od/blse/mod.rs:146-541
//   ProcessNoise::propagate                                    od/snc.rs:175-286
//   GroundStation::measure_instantaneous, ScalarSensitivity    od/ground_station/trk_device.rs:154-200, od/msr/sensitivity.rs:118-239
// The reference gets the partials from forward-mode dual numbers (hyperdual 1.5.0); so does this file, with a 3-partial
// dual type (only d/d(position) is ever read).
#include "nyxb_od_arc.cuh"

#ifndef NYXB_STRICT
#error "NYXB_STRICT must be defined to 0 or 1"
#endif
#if NYXB_STRICT
#define NYXB_KSTM nyxb_k_stm_strict
#define NYXB_KOD nyxb_k_od_strict
#define NYXB_KPRED nyxb_k_pred_strict
#define NYXB_LAUNCH_STM nyxb_launch_stm_strict
#define NYXB_LAUNCH_OD nyxb_launch_od_strict
#define NYXB_LAUNCH_PRED nyxb_launch_pred_strict
#define NYXB_KBLS nyxb_k_bls_strict
#define NYXB_LAUNCH_BLS nyxb_launch_bls_strict
#define NYXB_KODREC nyxb_k_od_rec_strict
#define NYXB_LAUNCH_ODREC nyxb_launch_od_rec_strict
#define NYXB_KODPOS nyxb_k_odpos_strict
#define NYXB_KODPOSREC nyxb_k_odpos_rec_strict
#define NYXB_LAUNCH_ODPOS nyxb_launch_odpos_strict
#else
#define NYXB_KSTM nyxb_k_stm_fast
#define NYXB_KOD nyxb_k_od_fast
#define NYXB_KPRED nyxb_k_pred_fast
#define NYXB_LAUNCH_STM nyxb_launch_stm_fast
#define NYXB_LAUNCH_OD nyxb_launch_od_fast
#define NYXB_LAUNCH_PRED nyxb_launch_pred_fast
#define NYXB_KBLS nyxb_k_bls_fast
#define NYXB_LAUNCH_BLS nyxb_launch_bls_fast
#define NYXB_KODREC nyxb_k_od_rec_fast
#define NYXB_LAUNCH_ODREC nyxb_launch_od_rec_fast
#define NYXB_KODPOS nyxb_k_odpos_fast
#define NYXB_KODPOSREC nyxb_k_odpos_rec_fast
#define NYXB_LAUNCH_ODPOS nyxb_launch_odpos_fast
#endif

// ------------------------------------------------------------------------- per-thread backend of nyxb_od_arc.cuh
// one RHS evaluation: k[6] = (v, a), A-parts G[9], gcr[3]
__device__ static int eom_stm(const DevSetup& S, OdInst& in, double delta_t_s, const double ys[9], double k[6], double G[9], double gcr[3]) {
    long long t_ns = in.epoch_ns + dur_from_seconds(delta_t_s);
    double yy[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) yy[e] = ys[e];
    yy[6] = yy[6] < 0.0 ? 0.0 : (yy[6] > 2.0 ? 2.0 : yy[6]);
    double mass = in.dry_mass + yy[8] + in.extra_mass;
    if (S.has_srp && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3];
    int rc = dual_eom_dev<true>(S, t_ns, yy, mass, in.srp_area, acc, G, gcr);
    in.n_rhs++;
    if (rc) return rc;
    k[0] = yy[3]; k[1] = yy[4]; k[2] = yy[5];
    k[3] = acc[0]; k[4] = acc[1]; k[5] = acc[2];
    return 0;
}

// One thread runs the whole trajectory or filter: every loop is serial and its arrays are local.  NS: the tracker kind's observation
// slots (the gain scratch PHt and K is 9 x NS).
template <int NS>
struct ThreadBT {
    static constexpr int stride = 1;
    const DevSetup& S;
    double phi[81];
    struct Step {
        double nphi[81], k[NYXB_MAX_STAGES][6], Ai[NYXB_MAX_STAGES][12];
        __device__ explicit Step(ThreadBT&) {}
    };
    struct Filt {
        double P[81], xdev[9], Pb[81], T[81], F[81], PHt[9 * NS], K[9 * NS];
        __device__ explicit Filt(ThreadBT&) {}
    };
    __device__ explicit ThreadBT(const DevSetup& s) : S(s) {}
    __device__ int first() const { return 0; }
    __device__ bool lead() const { return true; }
    __device__ void sync() const {}
    __device__ bool any(bool v) const { return v; }
    __device__ int rhs(OdInst& in, double delta_t_s, const double ys[9], Step& st, int slot) const {
        return eom_stm(S, in, delta_t_s, ys, st.k[slot], st.Ai[slot], st.Ai[slot] + 9);
    }
};
using ThreadB = ThreadBT<2>;

__global__ void __launch_bounds__(64)
NYXB_KSTM(const __grid_constant__ DevSetup S, size_t n, const double* __restrict__ state, const double* __restrict__ consts,
          const long long* __restrict__ epoch0, long long end_epoch, long long* __restrict__ step_io,
          const double* __restrict__ stm_in, double* __restrict__ out_state, long long* __restrict__ out_epoch,
          double* __restrict__ out_stm, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadB b(S);
    OdInst in;
    od_load(S, in, i, n, state, consts, epoch0, step_io);
    if (stm_in) { for (int e = 0; e < 81; ++e) b.phi[e] = stm_in[(size_t)e * n + i]; }
    else od_reset_stm(b);
    int rc = od_propagate(b, in, end_epoch - in.epoch_ns);
    for (int e = 0; e < 81; ++e) out_stm[(size_t)e * n + i] = b.phi[e];
    if (step_io) step_io[i] = in.step_ns;
    od_store(b, in, rc, i, n, out_state, out_epoch, out_details, out_status);
}

__global__ void __launch_bounds__(64)
NYXB_KOD(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, size_t n, const double* __restrict__ state,
         const double* __restrict__ consts, const long long* __restrict__ epoch0, double* __restrict__ out_state,
         long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadB b(S);
    od_process_arc(od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}

// the filter with every estimate recorded (ODSolution.estimates, for ODSolution::smooth)
__global__ void __launch_bounds__(64)
NYXB_KODREC(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, const OdEstRecords er, size_t n,
            const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
            double* __restrict__ out_state, long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details,
            int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadB b(S);
    od_process_arc<ThreadB, true>(od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status, &er);
}

__global__ void __launch_bounds__(64)
NYXB_KPRED(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, size_t n, const double* __restrict__ state,
           const double* __restrict__ consts, const long long* __restrict__ epoch0, const long long* __restrict__ end_epoch,
           const double* __restrict__ dev0, const OdRecords rec, long long* __restrict__ rec_count, double* __restrict__ out_state,
           long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadB b(S);
    od_predict(od, b, i, n, state, consts, epoch0, end_epoch, dev0, rec, rec_count, out_state, out_epoch, out_details, out_status);
}

__global__ void __launch_bounds__(64)
NYXB_KBLS(const __grid_constant__ DevSetup S, const __grid_constant__ DevOd od, const __grid_constant__ DevBls bl, size_t n,
          const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
          double* __restrict__ out_state, long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details,
          int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadB b(S);
    od_bls(od, bl, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}

// the filter over position fixes (PositionDevice), without and with the estimate records
__global__ void __launch_bounds__(64)
NYXB_KODPOS(const __grid_constant__ DevSetup S, const __grid_constant__ DevOdPos od, size_t n, const double* __restrict__ state,
            const double* __restrict__ consts, const long long* __restrict__ epoch0, double* __restrict__ out_state,
            long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadBT<3> b(S);
    od_process_arc<ThreadBT<3>, false, PosTrk>(od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}

__global__ void __launch_bounds__(64)
NYXB_KODPOSREC(const __grid_constant__ DevSetup S, const __grid_constant__ DevOdPos od, const OdEstRecords er, size_t n,
               const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
               double* __restrict__ out_state, long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details,
               int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadBT<3> b(S);
    od_process_arc<ThreadBT<3>, true, PosTrk>(od, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status, &er);
}

extern "C" cudaError_t NYXB_LAUNCH_STM(const DevSetup* S, size_t n, const double* state, const double* consts, const long long* epoch0,
                                       long long end_epoch, long long* step_io, const double* stm_in, double* out_state,
                                       long long* out_epoch, double* out_stm, nyxb_details* out_details, int* out_status,
                                       cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KSTM<<<grid, block, 0, stream>>>(*S, n, state, consts, epoch0, end_epoch, step_io, stm_in, out_state, out_epoch, out_stm,
                                          out_details, out_status);
    return cudaGetLastError();
}

extern "C" cudaError_t NYXB_LAUNCH_OD(const DevSetup* S, const DevOd* od, size_t n, const double* state, const double* consts,
                                      const long long* epoch0, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                      int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // few, long-running threads: spread them over as many SMs as possible
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KOD<<<grid, block, 0, stream>>>(*S, *od, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    return cudaGetLastError();
}

extern "C" cudaError_t NYXB_LAUNCH_ODREC(const DevSetup* S, const DevOd* od, const OdEstRecords* er, size_t n, const double* state,
                                         const double* consts, const long long* epoch0, double* out_state, long long* out_epoch,
                                         nyxb_details* out_details, int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // as the filter kernel
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KODREC<<<grid, block, 0, stream>>>(*S, *od, *er, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    return cudaGetLastError();
}

extern "C" cudaError_t NYXB_LAUNCH_PRED(const DevSetup* S, const DevOd* od, size_t n, const double* state, const double* consts,
                                        const long long* epoch0, const long long* end_epoch, const double* dev0, const OdRecords* rec,
                                        long long* rec_count, double* out_state, long long* out_epoch, nyxb_details* out_details,
                                        int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // as the filter kernel
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KPRED<<<grid, block, 0, stream>>>(*S, *od, n, state, consts, epoch0, end_epoch, dev0, *rec, rec_count, out_state, out_epoch,
                                           out_details, out_status);
    return cudaGetLastError();
}

extern "C" cudaError_t NYXB_LAUNCH_BLS(const DevSetup* S, const DevOd* od, const DevBls* bl, size_t n, const double* state,
                                       const double* consts, const long long* epoch0, double* out_state, long long* out_epoch,
                                       nyxb_details* out_details, int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // as the filter kernel
    unsigned grid = (unsigned)((n + block - 1) / block);
    NYXB_KBLS<<<grid, block, 0, stream>>>(*S, *od, *bl, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    return cudaGetLastError();
}

// er: null for the filter alone
extern "C" cudaError_t NYXB_LAUNCH_ODPOS(const DevSetup* S, const DevOdPos* od, const OdEstRecords* er, size_t n, const double* state,
                                         const double* consts, const long long* epoch0, double* out_state, long long* out_epoch,
                                         nyxb_details* out_details, int* out_status, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // as the filter kernel
    unsigned grid = (unsigned)((n + block - 1) / block);
    if (er)
        NYXB_KODPOSREC<<<grid, block, 0, stream>>>(*S, *od, *er, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    else
        NYXB_KODPOS<<<grid, block, 0, stream>>>(*S, *od, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
    return cudaGetLastError();
}
