// nyxb_od.cu — state-transition-matrix propagation and the sequential Kalman filter, one CUDA thread per trajectory
// (SURVEY.md §8 (f)-2; BASELINE configs[4]).  The whole arc of a filter — propagation of the nominal state and the STM
// between measurements, time updates, measurement updates, state replacement — runs inside ONE kernel launch; state,
// STM, covariance and stage data stay in registers / L1-resident local memory, HBM sees the inputs once and the
// per-measurement residual records as coalesced [m][..][n] stores.  The propagation and the filter loop are the templates of
// nyxb_od_arc.cuh; this file gives them the per-thread backend (ThreadBT) and holds one kernel template, nyxb_k_od<Job>, and its
// launcher, instantiated for every OD job of nyxb_od.cuh.
//
// Built twice like nyxb_kernels.cu: -DNYXB_STRICT=1 -fmad=false (same operation order as oracle/nyx_oracle_od.c for
// the dynamics) and -DNYXB_STRICT=0 -fmad=true, in the namespaces nyxb_od_strict and nyxb_od_fast.
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
//   GroundStation::measure_instantaneous, ScalarSensitivity    od/ground_station/trk_device.rs:154-208, od/msr/sensitivity.rs:118-239
// The reference gets the partials from forward-mode dual numbers (hyperdual 1.5.0); so does this file, with a 3-partial
// dual type (only d/d(position) is ever read).
#include "nyxb_od_arc.cuh"

#ifndef NYXB_STRICT
#error "NYXB_STRICT must be defined to 0 or 1"
#endif
#if NYXB_STRICT
#define NYXB_OD_NS nyxb_od_strict
#else
#define NYXB_OD_NS nyxb_od_fast
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
namespace NYXB_OD_NS {

template <class Job>
__global__ void __launch_bounds__(64)
nyxb_k_od(const __grid_constant__ DevSetup S, const __grid_constant__ Job job, size_t n, const double* __restrict__ state,
          const double* __restrict__ consts, const long long* __restrict__ epoch0, double* __restrict__ out_state,
          long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details, int* __restrict__ out_status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ThreadBT<Job::NS> b(S);
    od_run(job, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}

template <class Job>
cudaError_t launch(const DevSetup& S, const Job& job, size_t n, const OdIo& io, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int block = 32;  // few, long-running threads: spread them over as many SMs as possible
    unsigned grid = (unsigned)((n + block - 1) / block);
    nyxb_k_od<Job><<<grid, block, 0, st>>>(S, job, n, io.state, io.consts, io.epoch0, io.out_state, io.out_epoch, io.out_details,
                                           io.out_status);
    return cudaGetLastError();
}

template cudaError_t launch(const DevSetup&, const OdStmJob&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevStation, false>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevStation, true>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevPosDevice, false>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevPosDevice, true>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevAerStation, false>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevAerStation, true>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevLink, false>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdFilterJob<DevLink, true>&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdPredictJob&, size_t, const OdIo&, cudaStream_t);
template cudaError_t launch(const DevSetup&, const OdBlsJob&, size_t, const OdIo&, cudaStream_t);

}  // namespace NYXB_OD_NS
