// nyxb_smooth.cu — ODSolution::smooth (od/process/solution/smooth.rs:104-249) for n filters in one launch.
//
// As coded, the reference smooths estimate k from the FILTER estimate k+1 alone (x_s = Phi^-1 x_{k+1}, P_s = Phi^-1 P_{k+1} Phi^-T,
// Phi the STM stored with estimate k+1), not from the smoothed k+1 of a backward sweep.  Every k is therefore independent: one thread
// per (estimate k, filter i), the filter index fastest so that every record row ([k][..][n]) is read and written coalesced.  The
// kernel is bandwidth-bound by design (about 1.6 KB read and up to 0.9 KB written per estimate against about 5 kflop); the 9x9 work
// is nyxb_smooth.h, shared with a host build.  The postfit is recomputed through the filter's own window geometry (od_window_setup,
// bias subtracted) at estimate k's epoch with the measurement of record k+1.
//
// Built once, STRICT and without FMA contraction, like the host API: the 9x9 part is then bit-identical to its host build.  The same
// kernel template serves the ground station's records (nyxb_k_smooth<GroundTrk>), those of position fixes (nyxb_k_smooth<PosTrk>) and
// those of stations with angles (nyxb_k_smooth<AerTrk>) and those of interlink transmitters (nyxb_k_smooth<LinkTrk>, whose transmitter is
// interpolated at estimate k's epoch; a recording that does not cover it is the ephemeris error's key, reported as NYXB_ERR_TX_NO_DATA).
#include "nyxb_od_device.cuh"
#include "nyxb_smooth.h"
#include <type_traits>

// TRK: the tracker kind of the filter that wrote the records (GroundTrk, PosTrk, AerTrk, LinkTrk; nyxb_od_device.cuh)
template <class TRK>
__device__ __forceinline__ void smooth_one(const DevSetup& S, const DevSmoothT<typename TRK::Dev>& sm, size_t n) {
    constexpr int NS = TRK::NS;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)sm.cap * n) return;
    const size_t i = t % n;
    const long long k = (long long)(t / n);
    if (sm.pre_status[i]) return;
    const long long l = sm.count[i] - 1;                 // the host guarantees 1 <= l < cap here
    if (k > l) return;
    double nom[9], dk[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) { nom[r] = sm.nominal[((size_t)k * 9 + r) * n + i]; dk[r] = sm.dev[((size_t)k * 9 + r) * n + i]; }
    if (k == l) {                                        // the last estimate is copied unchanged (smooth.rs:120-127)
        double y[9];
        nyxb_est_state(nom, dk, y);
        for (int r = 0; r < 9; ++r) {
            if (sm.state) sm.state[((size_t)k * 9 + r) * n + i] = y[r];
            if (sm.sdev) sm.sdev[((size_t)k * 9 + r) * n + i] = dk[r];
        }
        if (sm.scov)
            for (int e = 0; e < 81; ++e) sm.scov[((size_t)k * 81 + e) * n + i] = sm.covar[((size_t)k * 81 + e) * n + i];
        return;
    }
    const size_t k1 = (size_t)k + 1;
    double phi[81], P[81], x1[9], Pi[81], T[81], xs[9];
    double* Ps = phi;                                    // phi is dead once inverted
    for (int e = 0; e < 81; ++e) {                       // column-major records -> row-major
        const int c = e / 9, r = e - 9 * c;
        phi[r * 9 + c] = sm.stm[(k1 * 81 + e) * n + i];
        P[r * 9 + c] = sm.covar[(k1 * 81 + e) * n + i];
    }
#pragma unroll
    for (int r = 0; r < 9; ++r) x1[r] = sm.dev[(k1 * 9 + r) * n + i];
    if (!nyxb_smooth_core(phi, P, x1, Pi, T, Ps, xs)) {  // ODError::SingularStateTransitionMatrix
        atomicMax(&sm.err_key[i], 2 * k + 1);
        return;
    }
    double ys[9], yf[9], pf[9], ps[9], rat[9];
    nyxb_est_state(nom, xs, ys);
    nyxb_est_state(nom, dk, yf);
#pragma unroll
    for (int q = 0; q < 9; ++q) { pf[q] = sm.covar[((size_t)k * 81 + q * 10) * n + i]; ps[q] = Ps[q * 10]; }
    nyxb_fs_ratios(yf, ys, pf, ps, rat);
    // residual k+1 recomputed at estimate k (smooth.rs:171-210): measure_instantaneous(smoothed state k) minus the bias
    const long long tg = sm.tag[k1 * n + i];
    if (tg >= 0 && sm.postfit) {
        const long long mk = TRK::tag_msr(tg);
        const int wno = TRK::tag_window(tg);
        const typename TRK::Dev& gs = sm.stations[sm.msr_tracker[mk]];
        double o[NS];
#pragma unroll
        for (int s = 0; s < NS; ++s) o[s] = sm.obs[((size_t)mk * NS + s) * n + i];
        typename TRK::Win w;
        const long long ek = sm.epoch[(size_t)k * n + i];
        const int wrc = TRK::setup(S, gs, sm.msr_size, wno, o, ek, ek, ys, w);
        if (wrc == OD_WIN_EPHEMERIS || (std::is_same<TRK, LinkTrk>::value && wrc == OD_WIN_TX_NO_DATA)) { atomicMax(&sm.err_key[i], 2 * k); return; }
        if (wrc == OD_WIN_OK)
            for (int q = 0; q < w.ncur; ++q) sm.postfit[((size_t)k * NS + wno * sm.msr_size + q) * n + i] = w.real_obs[q] - w.comp[q];
    }
    for (int r = 0; r < 9; ++r) {
        if (sm.state) sm.state[((size_t)k * 9 + r) * n + i] = ys[r];
        if (sm.sdev) sm.sdev[((size_t)k * 9 + r) * n + i] = xs[r];
        if (sm.ratio) sm.ratio[((size_t)k * 9 + r) * n + i] = rat[r];
    }
    if (sm.scov)
        for (int e = 0; e < 81; ++e) {
            const int c = e / 9, r = e - 9 * c;
            sm.scov[((size_t)k * 81 + e) * n + i] = Ps[r * 9 + c];
        }
}

template <class TRK>
__global__ void __launch_bounds__(128)
nyxb_k_smooth(const __grid_constant__ DevSetup S, const __grid_constant__ DevSmoothT<typename TRK::Dev> sm, size_t n) {
    smooth_one<TRK>(S, sm, n);
}

// A filter whose smoothing failed (err_key >= 0) has no solution in the reference: every output of it becomes NaN, also those that
// threads of its other estimates wrote.  Runs after nyxb_k_smooth on the same grid.
template <class TRK>
__global__ void __launch_bounds__(128)
nyxb_k_smooth_fail(const __grid_constant__ DevSmoothT<typename TRK::Dev> sm, size_t n) {
    constexpr int NS = TRK::NS;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)sm.cap * n) return;
    const size_t i = t % n, k = t / n;
    if (sm.err_key[i] < 0) return;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int r = 0; r < 9; ++r) {
        if (sm.state) sm.state[(k * 9 + r) * n + i] = nan;
        if (sm.sdev) sm.sdev[(k * 9 + r) * n + i] = nan;
        if (sm.ratio) sm.ratio[(k * 9 + r) * n + i] = nan;
    }
    if (sm.scov) for (int e = 0; e < 81; ++e) sm.scov[(k * 81 + e) * n + i] = nan;
    if (sm.postfit) for (int q = 0; q < NS; ++q) sm.postfit[(k * NS + q) * n + i] = nan;
}

template <class Dev>
cudaError_t nyxb_smooth_launch(const DevSetup& S, const DevSmoothT<Dev>& sm, size_t n, cudaStream_t st) {
    const size_t total = (size_t)sm.cap * n;
    if (total == 0) return cudaSuccess;
    const int block = 128;
    const unsigned grid = (unsigned)((total + block - 1) / block);
    nyxb_k_smooth<typename Dev::Trk><<<grid, block, 0, st>>>(S, sm, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    nyxb_k_smooth_fail<typename Dev::Trk><<<grid, block, 0, st>>>(sm, n);
    return cudaGetLastError();
}

template cudaError_t nyxb_smooth_launch(const DevSetup&, const DevSmoothT<DevStation>&, size_t, cudaStream_t);
template cudaError_t nyxb_smooth_launch(const DevSetup&, const DevSmoothT<DevPosDevice>&, size_t, cudaStream_t);
template cudaError_t nyxb_smooth_launch(const DevSetup&, const DevSmoothT<DevAerStation>&, size_t, cudaStream_t);
template cudaError_t nyxb_smooth_launch(const DevSetup&, const DevSmoothT<DevLink>&, size_t, cudaStream_t);
