// nyxb_od_coop.cu — warp-cooperative sequential Kalman filter (FAST mode): the 32 lanes of a warp run ONE filter.
//
// Why: an orbit-determination ensemble is small (BASELINE configs[4]: 1 000 filters) and every right-hand side carries
// the dual-number spherical-harmonic gradient (GravityField::gradient, gravity_field.rs:273-431: ~2 600 (n, m) entries for
// 70x70, each ~100 FP64 instructions).  One thread per filter leaves the GPU at 32 warps; one WARP per filter gives 1 000
// warps and splits the double sum by COLUMNS of the Legendre triangle:
//   * a lane owns a few columns m (longest-processing-time assignment from the host) and runs the column recursion of
//     A[n][m] and A[n+1][m+1] in dual numbers in registers;
//   * the four partial sums of the reference are regrouped so that everything that depends on n is accumulated first
//     (X_C = sum_n rr_n A[n][m] C_nm, ...) and the per-column constants (cos/sin(m lambda) duals) are applied once per
//     column; one xor-butterfly over the warp adds the lanes (every lane ends with bit-identical sums, so all lanes take
//     the same accept/reject/step decisions without a broadcast);
//   * STM, covariance, stage derivatives and stage A-matrices live in shared memory (one slab per warp); the 9x9
//     algebra of the filter (Phi P Phi^T, Joseph update) is spread over the lanes entry by entry.
// The propagation and the filter loop are the templates of nyxb_od_arc.cuh, shared with the per-thread kernels (nyxb_od.cu),
// which remain the STRICT (oracle-order) path; this file gives them the warp backend (WarpBT) and holds one kernel template,
// nyxb_k_od_coop<Job>, and its launcher, instantiated for the filter, prediction and BLS jobs of nyxb_od.cuh.  Its right-hand side sums in
// another order than the per-thread one (tolerance parity, tests/test_gpu_stm_od.py).
#include "nyxb_od_arc.cuh"

#define ODC_WPB 4            // warps (filters) per block
#define FULL 0xffffffffu

// the warp's slab in shared memory; NS: the tracker kind's observation slots (the gain scratch PHt and K is 9 x NS)
template <int NS>
struct WarpST {
    double phi[81], nphi[81];          // STM (column-major like the ABI) and its candidate
    double P[81], T[81], Pb[81], F[81];
    double k[NYXB_MAX_STAGES][6];
    double Ai[NYXB_MAX_STAGES][12];
    double PHt[9 * NS], K[9 * NS], xdev[9];
};

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ D3 wsum(D3 a) { return D3{wsum(a.v), wsum(a.x), wsum(a.y), wsum(a.z)}; }
__device__ __forceinline__ D3 dfma(D3 acc, D3 t, double c) { return D3{fma(t.v, c, acc.v), fma(t.x, c, acc.x), fma(t.y, c, acc.y), fma(t.z, c, acc.z)}; }

__device__ __forceinline__ D3 dsel(bool c, D3 a, D3 b) { return c ? a : b; }
// complex dual product (ar + i ai)(br + i bi)
__device__ __forceinline__ void cmul(const D3& ar, const D3& ai, const D3& br, const D3& bi, D3& rr, D3& ri) {
    rr = ar * br - ai * bi;
    ri = ar * bi + ai * br;
}

// GravityField::gradient split by columns over the lanes of a warp.  pw: per-warp D3 tables RM/IM/RP of N+2 entries each.
__device__ static void grav_gradient_coop(const DevGrav& g, const int* __restrict__ mycols, long long t_ns, const double r_in[3],
                                          D3* __restrict__ pw, int lane, double acc[3], double Gm[9]) {
    const int N = g.N;
    D3* RM = pw;
    D3* IM = pw + (N + 2);
    D3* RP = pw + 2 * (N + 2);
    double R[9];
    rotation_dcm(g.rot, t_ns, R);
    double rb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) rb[i] = (R[3 * i] * r_in[0] + R[3 * i + 1] * r_in[1]) + R[3 * i + 2] * r_in[2];
    const D3 rx = dvar(rb[0], 0), ry = dvar(rb[1], 1), rz = dvar(rb[2], 2);
    const D3 r_ = dnorm(rx, ry, rz);
    const D3 s_ = rx / r_, t_ = ry / r_, u_ = rz / r_;
    const D3 rho = dc(g.r_eq) / r_;
    {   // powers z^j = (s + i t)^j and (mu / r) rho^(j+1), j = 0..N, in log depth: lane l forms z^l from the binary digits of l
        // (the squarings z, z^2, .., z^16 are uniform), then z^(l+32), z^(l+64), .. by the uniform factor z^32.
        D3 zr = s_, zi = t_, pr = dc(1.0), pi = dc(0.0), qr = rho, qp = dc(1.0);
#pragma unroll 1
        for (int b = 0; b < 5; ++b) {
            D3 nr, ni;
            cmul(pr, pi, zr, zi, nr, ni);
            const bool on = (lane >> b) & 1;
            pr = dsel(on, nr, pr); pi = dsel(on, ni, pi);
            qp = dsel(on, qp * qr, qp);
            cmul(zr, zi, zr, zi, nr, ni);
            zr = nr; zi = ni;
            qr = qr * qr;
        }
        const D3 c0 = (dc(g.mu) / r_) * rho;   // (mu / r) rho^(0+1)
        __syncwarp();
        for (int j = lane; j <= N; j += 32) {
            RM[j] = pr; IM[j] = pi; RP[j] = c0 * qp;
            D3 nr, ni;
            cmul(pr, pi, zr, zi, nr, ni);
            pr = nr; pi = ni;
            qp = qp * qr;
        }
        __syncwarp();
    }
    D3 p0 = dc(0.0), p1 = dc(0.0), p2 = dc(0.0), p3 = dc(0.0);
    const double sq2 = sqrt(2.0);
    for (int kc = 0; kc < ODC_KMAX; ++kc) {
        const int m = mycols[kc];
        if (m < 0) break;
        const int n0 = m > 0 ? m : 1;
        D3 a, am1, b0, b1;
        if (m == 0) {
            am1 = dc(1.0);
            a = dscale(u_, sqrt(3.0));
            b0 = dc(__ldg(g.a_diag + 1));
            b1 = (dc(__ldg(g.offdiag + 1)) * u_) * b0;
        } else {
            am1 = dc(0.0);
            a = dc(__ldg(g.a_diag + m));
            b0 = dc(0.0);
            b1 = dc(__ldg(g.a_diag + m + 1));
        }
        D3 rhop = RP[n0];
        D3 XC = dc(0.0), XS = dc(0.0), YC = dc(0.0), YS = dc(0.0), ZC = dc(0.0), ZS = dc(0.0);
        const DevHarm* rec = g.tab + tri(n0, m);
        for (int n = n0; n <= N; ++n) {
            const double C = __ldg(&rec->cbar), Sv = __ldg(&rec->sbar), v01 = __ldg(&rec->vr01), v11 = __ldg(&rec->vr11);
            const D3 rr = dscale(rhop, g.inv_r_eq);
            const D3 t1 = rr * a;
            XC = dfma(XC, t1, C); XS = dfma(XS, t1, Sv);
            const D3 t2 = dscale(rr * b0, v01);
            YC = dfma(YC, t2, C); YS = dfma(YS, t2, Sv);
            const D3 t3 = dscale(rr * b1, v11);
            ZC = dfma(ZC, t3, C); ZS = dfma(ZS, t3, Sv);
            if (n < N) {
                const DevHarm* rec1 = g.tab + tri(n + 1, m);        // row n+1, column m
                const DevHarm* rec2 = g.tab + tri(n + 2, m + 1);    // row n+2, column m+1
                D3 an, bn;
                if (n == m) {
                    an = (dc(__ldg(g.offdiag + m)) * u_) * a;                                // A[m+1][m]
                    bn = (dc(__ldg(g.offdiag + m + 1)) * u_) * b1;                           // A[m+2][m+1]
                } else {
                    an = dscale(u_, __ldg(&rec1->b)) * a - dscale(am1, __ldg(&rec1->c));
                    bn = dscale(u_, __ldg(&rec2->b)) * b1 - dscale(b0, __ldg(&rec2->c));
                }
                am1 = a; a = an;
                b0 = b1; b1 = bn;
                rhop = rhop * rho;
                rec = rec1;
            }
        }
        const D3 rmm = RM[m], imm = IM[m];
        p2 = p2 + dscale(YC * rmm + YS * imm, sq2);
        p3 = p3 + dscale(ZC * rmm + ZS * imm, sq2);
        if (m > 0) {
            const D3 r1 = RM[m - 1], i1 = IM[m - 1];
            const double mf = (double)m * sq2;
            p0 = p0 + dscale(XC * r1 + XS * i1, mf);
            p1 = p1 + dscale(XS * r1 - XC * i1, mf);
        }
    }
    const D3 a0 = wsum(p0), a1 = wsum(p1), a2 = wsum(p2), a3n = wsum(p3);
    const D3 a3 = D3{-a3n.v, -a3n.x, -a3n.y, -a3n.z};
    const D3 al[3] = { a0 + a3 * s_, a1 + a3 * t_, a2 + a3 * u_ };
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[i] = (R[i] * al[0].v + R[3 + i] * al[1].v) + R[6 + i] * al[2].v;
    double tmp9[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            tmp9[3 * i + j] = (R[i] * dpart(al[0], j) + R[3 + i] * dpart(al[1], j)) + R[6 + i] * dpart(al[2], j);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            Gm[3 * i + j] = (tmp9[3 * i] * R[j] + tmp9[3 * i + 1] * R[3 + j]) + tmp9[3 * i + 2] * R[6 + j];
}

// ------------------------------------------------------------------------- warp backend of nyxb_od_arc.cuh
// what the right-hand side reads
template <int NS>
struct Ctx {
    const DevSetup* S;
    const int* mycols;   // this lane's columns of the Legendre triangle
    D3* pw;              // the warp's power tables
    WarpST<NS>* W;
    int lane;
};

// one RHS: stage slot `slot` of the shared k / Ai arrays receives (v, a) and the A-matrix parts
// __noinline__: called from two places in od_derive; one copy keeps the kernel's instruction footprint (and the
// instruction-cache misses ncu shows as `no_inst` stalls) down
template <int NS>
__device__ __noinline__ static int eom_coop(const Ctx<NS>& cx, OdInst& in, double delta_t_s, const double ys[9], int slot) {
    const DevSetup& S = *cx.S;
    long long t_ns = in.epoch_ns + dur_from_seconds(delta_t_s);
    double yy[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) yy[e] = ys[e];
    yy[6] = yy[6] < 0.0 ? 0.0 : (yy[6] > 2.0 ? 2.0 : yy[6]);
    double mass = in.dry_mass + yy[8] + in.extra_mass;
    if (S.has_srp && !(mass > 0.0)) return NYXB_ERR_MASSLESS;
    double acc[3], Gm[9], gcr[3];
    int rc = dual_eom_dev<false>(S, t_ns, yy, mass, in.srp_area, acc, Gm, gcr);
    in.n_rhs++;
    if (rc) return rc;
    if (S.has_grav) {
        double ga[3], gg[9];
        grav_gradient_coop(S.grav, cx.mycols, t_ns, yy, cx.pw, cx.lane, ga, gg);
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i] += ga[i];
#pragma unroll
        for (int q = 0; q < 9; ++q) Gm[q] += gg[q];
    }
    if (cx.lane == 0) {
        double* k = cx.W->k[slot];
        double* A = cx.W->Ai[slot];
        k[0] = yy[3]; k[1] = yy[4]; k[2] = yy[5]; k[3] = acc[0]; k[4] = acc[1]; k[5] = acc[2];
#pragma unroll
        for (int q = 0; q < 9; ++q) A[q] = Gm[q];
        A[9] = gcr[0]; A[10] = gcr[1]; A[11] = gcr[2];
    }
    __syncwarp();
    return 0;
}

// Every lane holds the same OdInst; the arrays live in the warp's slab and an 81-entry loop gives entry e to lane e % 32.
template <int NS>
struct WarpBT {
    static constexpr int stride = 32;
    const Ctx<NS>& cx;
    const DevSetup& S;
    WarpST<NS>& W;
    double (&phi)[81];
    struct Step {
        double (&nphi)[81];
        double (&k)[NYXB_MAX_STAGES][6];
        double (&Ai)[NYXB_MAX_STAGES][12];
        __device__ explicit Step(WarpBT& b) : nphi(b.W.nphi), k(b.W.k), Ai(b.W.Ai) {}
    };
    struct Filt {
        double (&P)[81], (&xdev)[9], (&Pb)[81], (&T)[81], (&F)[81], (&PHt)[9 * NS], (&K)[9 * NS];
        __device__ explicit Filt(WarpBT& b) : P(b.W.P), xdev(b.W.xdev), Pb(b.W.Pb), T(b.W.T), F(b.W.F), PHt(b.W.PHt), K(b.W.K) {}
    };
    __device__ explicit WarpBT(const Ctx<NS>& c) : cx(c), S(*c.S), W(*c.W), phi(c.W->phi) {}
    __device__ int first() const { return cx.lane; }
    __device__ bool lead() const { return cx.lane == 0; }
    __device__ void sync() const { __syncwarp(); }
    __device__ bool any(bool v) const { return __any_sync(FULL, v); }
    __device__ int rhs(OdInst& in, double delta_t_s, const double ys[9], Step&, int slot) const {
        return eom_coop(cx, in, delta_t_s, ys, slot);
    }
};

// bytes of one warp's slab: WarpST, then the D3 power tables RM / IM / RP of grav_gradient_coop, N + 2 entries each (the launcher
// and the kernel both size it here)
template <int NS>
__host__ __device__ __forceinline__ size_t od_coop_slab(int has_grav, int N) {
    const int npw = has_grav ? 3 * (N + 2) : 0;
    return (sizeof(WarpST<NS>) + sizeof(D3) * (size_t)npw + 15) & ~(size_t)15;
}

// one warp per filter, run, or problem; the host's column deal gives lane l the columns cols[l * ODC_KMAX ..] (-1 ends them)
template <class Job>
__global__ void __launch_bounds__(32 * ODC_WPB)
nyxb_k_od_coop(const __grid_constant__ DevSetup S, const __grid_constant__ Job job, const int* __restrict__ cols, size_t n,
               const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
               double* __restrict__ out_state, long long* __restrict__ out_epoch, nyxb_details* __restrict__ out_details,
               int* __restrict__ out_status) {
    constexpr int NS = Job::NS;
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const size_t i = (size_t)blockIdx.x * ODC_WPB + wib;
    if (i >= n) return;   // whole warps leave together
    const size_t slab = od_coop_slab<NS>(S.has_grav, S.grav.N);
    WarpST<NS>& W = *reinterpret_cast<WarpST<NS>*>(smem + slab * wib);
    Ctx<NS> cx;
    cx.S = &S; cx.mycols = cols + lane * ODC_KMAX; cx.W = &W; cx.lane = lane;
    cx.pw = reinterpret_cast<D3*>(smem + slab * wib + sizeof(WarpST<NS>));
    WarpBT<NS> b(cx);
    od_run(job, b, i, n, state, consts, epoch0, out_state, out_epoch, out_details, out_status);
}

template <class Job>
cudaError_t nyxb_od_coop_launch(const DevSetup& S, const Job& job, const int* cols, size_t n, const OdIo& io, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const size_t smem = od_coop_slab<Job::NS>(S.has_grav, S.grav.N) * ODC_WPB;
    cudaError_t e = cudaFuncSetAttribute(nyxb_k_od_coop<Job>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    unsigned grid = (unsigned)((n + ODC_WPB - 1) / ODC_WPB);
    nyxb_k_od_coop<Job><<<grid, 32 * ODC_WPB, smem, st>>>(S, job, cols, n, io.state, io.consts, io.epoch0, io.out_state, io.out_epoch,
                                                            io.out_details, io.out_status);
    return cudaGetLastError();
}

template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevStation, false>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevStation, true>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevPosDevice, false>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevPosDevice, true>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevAerStation, false>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevAerStation, true>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevLink, false>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdFilterJob<DevLink, true>&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdPredictJob&, const int*, size_t, const OdIo&, cudaStream_t);
template cudaError_t nyxb_od_coop_launch(const DevSetup&, const OdBlsJob&, const int*, size_t, const OdIo&, cudaStream_t);
