// nyxb_tx.cu — TRANSPOSED, warp-specialised propagation kernel (FAST mode): lane = trajectory, walker warp = column position,
// helper warps = everything else, two sets of trajectories in flight per CTA.
//
//   * A SET is 32 trajectories (lane l of every warp = trajectory l of the set).  The harmonic double sum (gravity_field.rs:217-249)
//     is split by COLUMNS of the derived-Legendre triangle over P WALKER warps; all 32 lanes of a walker walk the same entries, so
//     the 40-byte coefficient record of an entry is ONE warp-uniform shared-memory read (2 x LDS.128 + LDS.64 with a single address:
//     half the shared-memory wavefronts of the lane-varying reads of nyxb_k_coop), column boundaries are uniform branches, and no
//     lane idles.
//   * The column walk is software-pipelined by one entry: the six accumulations of entry n use Q[n], which was produced one
//     iteration earlier, while the only dependent FP64 chain is the one DFMA that advances the recursion
//     Q[n+1] = (2n+1) u Q[n] - (n+m)(n-m) r^2 Q[n-1].
//     13 FP64 instructions per entry.
//   * Everything that is serial per right-hand side — reduction of the partial sums, acceleration assembly, RK stage algebra,
//     body-fixed DCM, 1/r, the (cos, sin)(m lambda) cos^m(phi) and rho^m tables, and per step the error norm, the step-size controller,
//     recording and the stop condition — runs on two HELPER warps per set, concurrently with the walkers, which meanwhile walk the
//     OTHER set of the CTA: two sets alternate through the walkers (named barriers READY[set] / DONE[set]), so the FP64 pipe sees
//     the walk of one set while the latency-bound chain of the other is hidden.  Helper 0 (the lead) owns the position side (the
//     candidate and error sums of the positions, the stage DCMs, the controller, the set queue), helper 1 the acceleration side
//     (reduction of the partial sums, acceleration, V_{i+1}, P_{i+2}, the velocity sums).  8 walkers + 2 x 2 helpers = 12 warps:
//     every scheduler hosts two walkers and one helper, and the register cap is 168 per thread.
//     The first version of this kernel ran these phases on the walker warps themselves, between CTA-wide barriers, and spent much
//     of the warp-time in barrier stalls with the FP64 pipe half idle.
//   * Persistent CTAs, one per SM; every set context pulls (set, time-slice) tickets from a global counter: with fewer contexts than
//     sets every SM stays busy to the end (10 000 trajectories = 313 sets on 264 contexts of a 132-SM H100).  A parked set keeps its state in the
//     output arrays plus a small workspace; a finished trajectory inside a set keeps stepping on its own scratch without committing.
//   * HBM: initial state in, final state out, ~200 B per trajectory and slice of parking traffic.
//
// Reference behaviour: instance.rs:87-262, 343-352, 358-493 (propagate / single_step / derive), spacecraft.rs:191-310 (eom),
// gravity_field.rs:148-268.  FMA contraction and the regrouped summation make this a tolerance-parity path (same class as
// nyxb_k_coop: < 1e-6 km over the benchmark span, tests/test_gpu_baseline_spans.py).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>

#include "nyxb_tx.h"

#ifndef TX_MINB
#define TX_MINB 2   /* resident CTAs per SM the kernel is compiled for (register cap 65536 / (256 * TX_MINB)) */
#endif

namespace {
constexpr int NL = 32;   // trajectories per set, one per lane: stride of every per-trajectory shared-memory array
constexpr int HW = 2;    // helper warps per set context: 0 = lead (position side), 1 = acceleration side
constexpr unsigned FULL = 0xffffffffu;

// ---- per-trajectory controller state kept in shared memory ([field][lane])
enum { TXF_H = 0, TXF_ERR, TXF_CR, TXF_CD, TXF_PM, TXF_DRY, TXF_EXTRA, TXF_SRPA, TXF_DRAGA, TXF_EVPREV, TXF_COUNT };
enum { TXI_EPOCH = 0, TXI_STEP, TXI_PREV_STEP, TXI_DET_STEP, TXI_NSTEPS, TXI_NREJ, TXI_NRHS, TXI_COUNT };
enum { TXW_FLAGS = 0, TXW_STATUS, TXW_RC, TXW_ATT, TXW_EVCNT, TXW_ACC, TXW_RCST, TXW_COUNT };
enum { F_FIXED = 1, F_PREVFIXED = 2, F_RETRY = 4, F_LAST = 8, F_DONE = 16, F_BACK = 32, F_VALID = 64 };

// dynamic shared memory: [table blob | NCTX set contexts]; one context (buffers of consecutive stages alternate by parity):
//   wk   [2][WK][32]     walker inputs of a stage: ub, r2, and the powers of z = (cos, sin)(lambda) cos(phi) and rho it starts its
//                        columns from — P = 8, 10: every z^e, e = 0..2P, and rho^e, e = 1..2P (WK = 6P + 4; the walkers only load);
//                        P = 16: z^(2^k), rho^(2^k), k = 0..5 (WK = 20; the walkers multiply them together)   (helpers -> walkers)
//   rn   [2][9][32]      DCM of the stage being prepared (lead helper -> both helpers)
//   part [2][P][4][32]   partial sums of a stage                                                   (walkers -> helpers)
//   as   [2][18][32]     what the helpers need to assemble that stage's acceleration later (DCM, unit vector, K0, K1, two-body factor, position)
//   ysp  [2][3][32]      position of a coming stage (acceleration helper -> both helpers)
//   helper-private: kst [16][6][32] (k_i = (V_i, A_i)), nxt / er / ycur [6][32], controller fields
struct TxLayout {
    unsigned blob, ctx0, ctx_stride;                                  // bytes
    unsigned wk, part, as, ysp, kst, nxt, er, ycur, rot, rn, f64, i64, i32;   // offsets inside a context
    unsigned total;
};
__host__ __device__ inline TxLayout tx_layout(unsigned blob_bytes, int P, int N, int nctx) {
    (void)N;
    TxLayout L;
    L.blob = 0;
    L.ctx0 = (blob_bytes + 127u) & ~127u;
    unsigned o = 0;
    L.wk = o; o += 2u * (P == 16 ? 20u : 6u * (unsigned)P + 4u) * NL * 8;
    L.part = o; o += 2u * (unsigned)P * 4 * NL * 8;
    L.as = o; o += 2u * 18u * NL * 8;
    L.ysp = o; o += 2u * 3u * NL * 8;
    L.kst = o; o += NYXB_MAX_STAGES * 6 * NL * 8;
    L.nxt = o; o += 6 * NL * 8;
    L.er = o; o += 6 * NL * 8;
    L.ycur = o; o += 6 * NL * 8;
    L.rot = o; o += 6 * NL * 8;
    L.rn = o; o += 2u * 9u * NL * 8;
    L.f64 = o; o += TXF_COUNT * NL * 8;
    L.i64 = o; o += TXI_COUNT * NL * 8;
    L.i32 = o; o += TXW_COUNT * NL * 4;
    L.ctx_stride = (o + 127u) & ~127u;
    L.total = L.ctx0 + (unsigned)nctx * L.ctx_stride;
    return L;
}

struct TxSm {   // typed views of one set context
    double *wk, *part, *as, *ysp, *kst, *nxt, *er, *ycur, *rot, *rn, *f64;
    long long* i64;
    int* i32;
};
__device__ __forceinline__ TxSm tx_views(unsigned char* smem, const TxLayout& L, int ctx, int N) {
    (void)N;
    unsigned char* b = smem + L.ctx0 + (unsigned)ctx * L.ctx_stride;
    TxSm sm;
    sm.wk = reinterpret_cast<double*>(b + L.wk); sm.part = reinterpret_cast<double*>(b + L.part);
    sm.as = reinterpret_cast<double*>(b + L.as); sm.ysp = reinterpret_cast<double*>(b + L.ysp);
    sm.kst = reinterpret_cast<double*>(b + L.kst); sm.nxt = reinterpret_cast<double*>(b + L.nxt);
    sm.er = reinterpret_cast<double*>(b + L.er); sm.ycur = reinterpret_cast<double*>(b + L.ycur);
    sm.rot = reinterpret_cast<double*>(b + L.rot); sm.rn = reinterpret_cast<double*>(b + L.rn);
    sm.f64 = reinterpret_cast<double*>(b + L.f64); sm.i64 = reinterpret_cast<long long*>(b + L.i64);
    sm.i32 = reinterpret_cast<int*>(b + L.i32);
    return sm;
}

// named barriers (id 0 is __syncthreads): helpers of a context among themselves, helpers -> walkers, walkers -> helpers
__device__ __forceinline__ void nb_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void nb_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

__device__ __forceinline__ void tx_mbar_arrive(unsigned long long* bar) {   // release.cta: the thread's earlier shared stores are published
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool tx_mbar_test(unsigned bar_smem, unsigned parity) {   // non-blocking; acquire.cta when it succeeds
    unsigned ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(bar_smem), "r"(parity) : "memory");
    return ok != 0;
}

// Diagnostic timeline of CTA 0 (built with -DNYXB_TX_TRACE only; scripts/tx_trace.py reads it): lane 0 of every warp appends
// (clock << 20 | code << 12 | context << 8 | stage) records to its own strip.
enum { TR_POLL = 1, TR_WALK = 2, TR_WALK_END = 3, TR_DONE_WAIT = 4, TR_DONE_SEEN = 5, TR_READY = 6, TR_STAGES_END = 7, TR_CTRL_END = 8, TR_TOP = 9,
       TR_PRE_DONE = 10, TR_DCM_DONE = 11, TR_REDUCED = 12, TR_ACC_DONE = 13, TR_HB_PASSED = 14, TR_CTRL_IN = 15, TR_CTRL_OUT = 16,
       TR_PICKED = 17, TR_COMMITTED = 18, TR_PRIMED = 19, TR_DCM01 = 20 };
#ifdef NYXB_TX_TRACE
#define TX_TRACE(code, ctx, stg)                                                                                              \
    do {                                                                                                                      \
        if (q.trace && blockIdx.x == 0 && (threadIdx.x & 31) == 0 && tr_n < NYXB_TX_TRACE_CAP)                                   \
            q.trace[(size_t)(threadIdx.x >> 5) * NYXB_TX_TRACE_CAP + tr_n++] =                                                  \
                ((unsigned long long)clock64() << 20) | ((unsigned long long)(code) << 12) | ((unsigned long long)(ctx) << 8) | (unsigned long long)(stg); \
    } while (0)
#else
#define TX_TRACE(code, ctx, stg) do { } while (0)
#endif

// ---- one column of the walk.  (a01, a23, kk) hold the column's first record (prefetched); A / K point at it; on return they hold
// the first record of the next column.
// Entry n of column m (record p1..p4, kappa; Q = Q[n], Qn = Q[n+1]):
//     S1..S4 += Q p1..p4          W-term: S5, S6 += (kappa Qn) (p3, p4)
//     Qn = c1 Q - m2              c1 = (2n+1) u rho,  m2 = (n+m)(n-m) rho^2 Q[n-1]
// The loop-carried FP64 dependency is ONE DFMA per entry: c1 and m2 are formed one entry ahead and advanced by additions
// (c1 += 2 u rho; d += g, g += 2 rho^2 with d = (n+m)(n-m) rho^2), everything else in an entry is off the chain, so two walker
// warps per scheduler keep the FP64 pipe fed.  12 FP64 instructions per entry.  The loop is unrolled by hand over two register
// sets for the prefetched record so that no register-to-register moves are left in it (the compiler's own rotation cost 14
// IMAD.MOV per two entries and made the loop issue-bound).
// registers of a walker lane (its trajectory)
struct TxLaneState {
    double ub, r2, dc, dg;                  // u rho, rho^2 and their doubles
    double zar, zai, pa, zbr, zbi, pb;      // current powers of the two exponent sequences
    double qr, qi, qp;                      // common ratio z^(2P), rho^(2P)
    double X, Y, Z, W;                      // partial sums of this position
    double cQ, cc1, cg, cS5, cS6;           // set-up of the column about to be walked
};
#define NYXB_TX_ENTRY(P01, P23, PK)                             \
    {                                                           \
        const double Qn = fma(c1, Q, -m2);                      \
        c1 += t.dc; d += g; g += t.dg;                          \
        m2 = d * Q;                                             \
        S1 = fma(Q, (P01).x, S1);                               \
        S2 = fma(Q, (P01).y, S2);                               \
        S3 = fma(Q, (P23).x, S3);                               \
        S4 = fma(Q, (P23).y, S4);                               \
        const double wv = (PK) * Qn;                            \
        S5 = fma(wv, (P23).x, S5);                              \
        S6 = fma(wv, (P23).y, S6);                              \
        Q = Qn;                                                 \
    }
// t.(cQ, cc1, cg, cS5, cS6) arrive set up for this column — Q = rho^m x seed, c1 = (2m+1) u rho, g = (2m+1) rho^2, S5 / S6 the
// column's seed W term — because the caller sets the NEXT column up right behind the close of this one, in the same basic block, so
// the two short dependent chains overlap.
template <bool SEQ_B>
__device__ __forceinline__ void tx_column(const double2*& A, const double*& K, double2& a01, double2& a23, double& kk, int len,
                                          TxLaneState& t) {
    double Q = t.cQ, c1 = t.cc1, g = t.cg, S5 = t.cS5, S6 = t.cS6;
    double m2 = 0.0, d = 0.0;   // entry n = m: (n+m)(n-m) = 0
    double S1 = 0.0, S2 = 0.0, S3 = 0.0, S4 = 0.0;
    double2 b01, b23;
    double bk;
#pragma unroll 2
    for (int e = len; e > 0; e -= 2) {   // columns are padded to an even number of entries (null records)
        b01 = A[2]; b23 = A[3]; bk = K[1];
        NYXB_TX_ENTRY(a01, a23, kk)
        a01 = A[4]; a23 = A[5]; kk = K[2];   // the table ends with null records
        NYXB_TX_ENTRY(b01, b23, bk)
        A += 4; K += 2;
    }
    // close the column: apply its (cos, sin)((m-1) lambda) cos^(m-1)(phi)
    const double rr = SEQ_B ? t.zbr : t.zar, ii = SEQ_B ? t.zbi : t.zai;
    t.X = fma(rr, S1, fma(ii, S2, t.X));
    t.Y = fma(rr, S2, fma(-ii, S1, t.Y));
    t.Z = fma(rr, S3, fma(ii, S4, t.Z));
    t.W = fma(rr, S5, fma(ii, S6, t.W));
}

// ---- instance.rs:149-196: choose the step of the next attempt (regular, or the final fixed step to the stop time)
__device__ __forceinline__ void tx_pick_step(const TxSm& sm, int lane, long long stop) {
    int fl = sm.i32[TXW_FLAGS * NL + lane];
    if (!(fl & (F_DONE | F_RETRY))) {
        const long long epoch = sm.i64[TXI_EPOCH * NL + lane];
        long long step_ns = sm.i64[TXI_STEP * NL + lane];
        const bool back = fl & F_BACK;
        fl &= ~(F_LAST | F_PREVFIXED);
        if (fl & F_FIXED) fl |= F_PREVFIXED;
        sm.i64[TXI_PREV_STEP * NL + lane] = step_ns;
        if (ctl_past_stop(epoch, step_ns, stop, back)) {
            if (stop == epoch) {
                fl |= F_DONE;
            } else {
                step_ns = stop - epoch;
                fl |= F_FIXED | F_LAST;
                sm.i64[TXI_STEP * NL + lane] = step_ns;
            }
        }
        if (!(fl & F_DONE)) {
            sm.i32[TXW_ATT * NL + lane] = 1;
            sm.f64[TXF_H * NL + lane] = dur_to_seconds(step_ns);
        }
        sm.i32[TXW_FLAGS * NL + lane] = fl;
    }
}

// x^(1/n), n = 2..9, for the step-size controller of this tolerance-parity kernel: a single-precision seed (MUFU lg2 / ex2) and two
// Newton steps on q^n = x in double (relative error ~1e-6 -> 4e-12 -> rounding level).  The correctly rounded pow_inv_int of the
// STRICT kernels (CUDA pow + a double-double Newton step + log) is a ~600-instruction dependent chain; it sat on the serial path
// between two attempts of a set, where it took most of the clocks between the last DONE of an attempt and READY(0) of the next,
// while the error norm that feeds it already differs from the reference's by ~1e-4 relative in FAST mode (DESIGN.md section 3).
__device__ __forceinline__ double tx_pow_inv_int(double x, int n) {
    if (!(x > 1e-30) || !(x < 1e30) || n < 2 || n > 9) return pow_inv_int(x, n);
    const double inv_n = 1.0 / (double)n;
    const double inv_x = 1.0 / x;
    double q = (double)exp2f(log2f((float)x) * (float)inv_n);
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const double q2 = q * q, q4 = q2 * q2, q8 = q4 * q4;
        double qn;   // q^n
        switch (n) {
        case 2: qn = q2; break;
        case 3: qn = q2 * q; break;
        case 4: qn = q4; break;
        case 5: qn = q4 * q; break;
        case 6: qn = q4 * q2; break;
        case 7: qn = q4 * (q2 * q); break;
        case 8: qn = q8; break;
        default: qn = q8 * q; break;
        }
        const double r = fma(qn, inv_x, -1.0);   // q^n / x - 1
        q = fma(-(r * inv_n), q, q);             // Newton: q (1 - r / n)
    }
    return q;
}

// ---- error norm, accept / reject, next step (instance.rs:416-490), single_step bookkeeping (instance.rs:343-352), recording
// and stop condition; executed by the controller warp for its 32 trajectories
__device__ __noinline__ void tx_controller(const DevSetup& S, const DevSink& sink, TxSm sm, int lane, size_t n, size_t tr, int stages) {
    int fl = sm.i32[TXW_FLAGS * NL + lane];
    sm.i32[TXW_ACC * NL + lane] = 0;
    if (fl & F_DONE) return;
    const int rcst = sm.i32[TXW_RCST * NL + lane];   // failure of a right-hand side: code | (stage + 1) << 8
    if (rcst) {
        sm.i64[TXI_NRHS * NL + lane] += (rcst >> 8);
        sm.i32[TXW_RC * NL + lane] = rcst & 0xff;
        sm.i32[TXW_FLAGS * NL + lane] = fl | F_DONE;
        return;
    }
    sm.i64[TXI_NRHS * NL + lane] += stages;
    const double h = sm.f64[TXF_H * NL + lane];
    double cr = sm.f64[TXF_CR * NL + lane];
    const double cd = sm.f64[TXF_CD * NL + lane], pm = sm.f64[TXF_PM * NL + lane];
    long long step_ns = sm.i64[TXI_STEP * NL + lane];
    long long dt_ns = 0;
    bool accept;
    if (fl & F_FIXED) {
        sm.i64[TXI_DET_STEP * NL + lane] = step_ns;
        dt_ns = step_ns;
        accept = true;
    } else {
        // the stage states of y[6..8] are y + h * 0 (instance.rs:394): h = NaN poisons them as in the reference
        const double hz = h * 0.0;
        double e9[9], c9[9], y9[9];
#pragma unroll
        for (int e = 0; e < 6; ++e) { e9[e] = sm.er[e * NL + lane]; c9[e] = sm.nxt[e * NL + lane]; y9[e] = sm.ycur[e * NL + lane]; }
        e9[6] = e9[7] = e9[8] = 0.0;
        y9[6] = cr; y9[7] = cd; y9[8] = pm;
        c9[6] = cr + hz; c9[7] = cd + hz; c9[8] = pm + hz;
        const double err = error_estimate(S.error_ctrl, e9, c9, y9);
        sm.f64[TXF_ERR * NL + lane] = err;
        const int att = sm.i32[TXW_ATT * NL + lane];
        accept = ctl_accept(S, err, h, att);
        if (accept) {
            bool bad = false;
#pragma unroll
            for (int e = 0; e < 9; ++e) bad |= (c9[e] != c9[e]);
            if (bad) {
                sm.i32[TXW_RC * NL + lane] = NYXB_ERR_PROP_MATH;
                sm.i32[TXW_FLAGS * NL + lane] = fl | F_DONE;
                return;
            }
            long long det_step;
            step_ns = ctl_accepted<tx_pow_inv_int>(S, err, h, att, sm.i32[TXW_STATUS * NL + lane], det_step);
            sm.i64[TXI_DET_STEP * NL + lane] = det_step;
            dt_ns = det_step;
        } else {
            sm.i32[TXW_ATT * NL + lane] = att + 1;
            sm.i64[TXI_NREJ * NL + lane] += 1;
            sm.f64[TXF_H * NL + lane] = ctl_retry<tx_pow_inv_int>(S, err, h);
            sm.i32[TXW_FLAGS * NL + lane] = fl | F_RETRY;
            return;
        }
    }
    // ---- single_step(): instance.rs:343-352
    fl &= ~F_RETRY;
    const long long epoch = sm.i64[TXI_EPOCH * NL + lane] + dt_ns;
    sm.i64[TXI_EPOCH * NL + lane] = epoch;
    sm.i32[TXW_ACC * NL + lane] = 1;
    cr = cr < 0.0 ? 0.0 : (cr > 2.0 ? 2.0 : cr);   // cosmic/spacecraft.rs:494
    sm.f64[TXF_CR * NL + lane] = cr;
    const long long ns = sm.i64[TXI_NSTEPS * NL + lane] + 1;
    sm.i64[TXI_NSTEPS * NL + lane] = ns;
    if ((fl & F_VALID) && ns < sink.cap) sink.epoch[(size_t)ns * n + tr] = epoch;   // the state is stored by the component warps
    if (pm < 0.0) { sm.i32[TXW_RC * NL + lane] = NYXB_ERR_FUEL_EXHAUSTED; fl |= F_DONE; }
    if (sink.ev_kind && !(fl & F_LAST)) {   // stop condition on non-final steps (instance.rs:243-252, event.rs:120-150)
        const double yn = event_eval(sink.ev_kind, sink.ev_value, sm.nxt[lane], sm.nxt[NL + lane], sm.nxt[2 * NL + lane],
                                     sm.nxt[3 * NL + lane], sm.nxt[4 * NL + lane], sm.nxt[5 * NL + lane]);
        const int cnt = sm.i32[TXW_EVCNT * NL + lane] + ((sm.f64[TXF_EVPREV * NL + lane] * yn < 0.0) ? 1 : 0);
        sm.f64[TXF_EVPREV * NL + lane] = yn;
        sm.i32[TXW_EVCNT * NL + lane] = cnt;
        if (cnt >= sink.ev_trigger) fl |= F_DONE;
    }
    if (fl & F_LAST) {   // restore the adapted step (instance.rs:194-196)
        step_ns = sm.i64[TXI_PREV_STEP * NL + lane];
        fl = (fl & ~F_FIXED) | ((fl & F_PREVFIXED) ? F_FIXED : 0);
        if (fl & F_BACK) step_ns = -step_ns;
        fl |= F_DONE;
    }
    sm.i64[TXI_STEP * NL + lane] = step_ns;
    sm.i32[TXW_FLAGS * NL + lane] = fl;
}

// ---- controller state of a set: initial (round 0, instance.rs:96-115) or from the parking area
__device__ __noinline__ void tx_load_ctl(const DevSetup& S, const DevSink& sink, const DevTxQueue& q, TxSm sm, int lane, size_t n,
                                         size_t tr, bool valid, int round, const double* __restrict__ state,
                                         const double* __restrict__ consts, const long long* __restrict__ epoch0, long long end_epoch,
                                         const long long* step_io, const double* out_state, const long long* out_epoch) {
    sm.f64[TXF_DRY * NL + lane] = consts[tr];
    sm.f64[TXF_EXTRA * NL + lane] = consts[n + tr];
    sm.f64[TXF_SRPA * NL + lane] = consts[2 * n + tr];
    sm.f64[TXF_DRAGA * NL + lane] = consts[3 * n + tr];
    sm.i32[TXW_ACC * NL + lane] = 0;
    sm.i32[TXW_RCST * NL + lane] = 0;
    const long long ep0 = epoch0[tr];
    const long long duration = end_epoch - ep0;
    if (round == 0) {
        const double pm = state[8 * n + tr];
        sm.f64[TXF_CR * NL + lane] = state[6 * n + tr];
        sm.f64[TXF_CD * NL + lane] = state[7 * n + tr];
        sm.f64[TXF_PM * NL + lane] = pm;
        sm.f64[TXF_H * NL + lane] = 0.0;
        sm.f64[TXF_ERR * NL + lane] = 0.0;
        long long step_ns = step_io ? step_io[tr] : S.init_step_ns;
        int fl = (S.fixed_step ? F_FIXED : 0) | (valid ? F_VALID : 0) | (duration < 0 ? F_BACK : 0);
        int rc = 0;
        if (!valid || duration == 0) fl |= F_DONE;
        if (!(fl & F_DONE) && pm < 0.0) { rc = NYXB_ERR_FUEL_EXHAUSTED; fl |= F_DONE; }
        if (!(fl & F_DONE) && duration < 0) step_ns = -step_ns;
        sm.i64[TXI_EPOCH * NL + lane] = ep0;
        sm.i64[TXI_STEP * NL + lane] = step_ns;
        sm.i64[TXI_PREV_STEP * NL + lane] = step_ns;
        sm.i64[TXI_DET_STEP * NL + lane] = S.init_step_ns;
        sm.i64[TXI_NSTEPS * NL + lane] = 0;
        sm.i64[TXI_NREJ * NL + lane] = 0;
        sm.i64[TXI_NRHS * NL + lane] = 0;
        sm.i32[TXW_FLAGS * NL + lane] = fl;
        sm.i32[TXW_STATUS * NL + lane] = 0;
        sm.i32[TXW_RC * NL + lane] = rc;
        sm.i32[TXW_ATT * NL + lane] = 1;
        sm.i32[TXW_EVCNT * NL + lane] = 0;
        sm.f64[TXF_EVPREV * NL + lane] = 0.0;
        if (sink.ev_kind)
            sm.f64[TXF_EVPREV * NL + lane] = event_eval(sink.ev_kind, sink.ev_value, state[tr], state[n + tr], state[2 * n + tr],
                                                        state[3 * n + tr], state[4 * n + tr], state[5 * n + tr]);
        if (valid && sink.cap > 0) sink.epoch[tr] = ep0;   // start state (instance.rs:307, 321)
    } else {
        const int pf = __ldcg(q.ws_flags + tr);
        const nyxb_details* dp = q.details + tr;
        sm.f64[TXF_CR * NL + lane] = __ldcg(out_state + 6 * n + tr);
        sm.f64[TXF_CD * NL + lane] = __ldcg(out_state + 7 * n + tr);
        sm.f64[TXF_PM * NL + lane] = __ldcg(out_state + 8 * n + tr);
        sm.f64[TXF_H * NL + lane] = __ldcg(q.ws_f64 + tr);
        sm.f64[TXF_EVPREV * NL + lane] = __ldcg(q.ws_f64 + n + tr);
        sm.f64[TXF_ERR * NL + lane] = __ldcg(&dp->error);
        sm.i64[TXI_EPOCH * NL + lane] = __ldcg(out_epoch + tr);
        const long long step_ns = __ldcg(q.ws_step + tr);
        sm.i64[TXI_STEP * NL + lane] = step_ns;
        sm.i64[TXI_PREV_STEP * NL + lane] = step_ns;
        sm.i64[TXI_DET_STEP * NL + lane] = __ldcg((const long long*)&dp->step_ns);
        sm.i64[TXI_NSTEPS * NL + lane] = __ldcg((const long long*)&dp->n_steps);
        sm.i64[TXI_NREJ * NL + lane] = __ldcg((const long long*)&dp->n_rejected);
        sm.i64[TXI_NRHS * NL + lane] = __ldcg((const long long*)&dp->n_rhs);
        sm.i32[TXW_ATT * NL + lane] = __ldcg(&dp->attempts);
        int fl = (pf & (F_FIXED | F_RETRY | F_DONE)) | (valid ? F_VALID : 0) | (duration < 0 ? F_BACK : 0);
        if (!valid) fl |= F_DONE;
        sm.i32[TXW_FLAGS * NL + lane] = fl;
        sm.i32[TXW_STATUS * NL + lane] = (pf & 8) ? NYXB_WARN_MAX_ATTEMPTS : 0;
        sm.i32[TXW_RC * NL + lane] = (pf >> 8) & 0xff;
        sm.i32[TXW_EVCNT * NL + lane] = sink.ev_kind ? __ldcg(sink.ev_crossings + tr) : 0;
    }
}

// ---- park the controller state of a set (== the final outputs once the trajectory is done)
__device__ __noinline__ void tx_park_ctl(const DevSink& sink, const DevTxQueue& q, TxSm sm, int lane, size_t n, size_t tr,
                                         long long* step_io, double* out_state, long long* out_epoch, int* out_status) {
    const int fl = sm.i32[TXW_FLAGS * NL + lane];
    if (!(fl & F_VALID)) return;
    const int rc = sm.i32[TXW_RC * NL + lane], st = sm.i32[TXW_STATUS * NL + lane];
    out_state[6 * n + tr] = sm.f64[TXF_CR * NL + lane];
    out_state[7 * n + tr] = sm.f64[TXF_CD * NL + lane];
    out_state[8 * n + tr] = sm.f64[TXF_PM * NL + lane];
    out_epoch[tr] = sm.i64[TXI_EPOCH * NL + lane];
    const long long step_ns = sm.i64[TXI_STEP * NL + lane];
    q.ws_step[tr] = step_ns;
    q.ws_f64[tr] = sm.f64[TXF_H * NL + lane];
    q.ws_f64[n + tr] = sm.f64[TXF_EVPREV * NL + lane];
    q.ws_flags[tr] = (fl & (F_FIXED | F_RETRY | F_DONE)) | ((st & NYXB_WARN_MAX_ATTEMPTS) ? 8 : 0) | (rc << 8);
    nyxb_details d;
    d.step_ns = sm.i64[TXI_DET_STEP * NL + lane];
    d.error = sm.f64[TXF_ERR * NL + lane];
    d.attempts = sm.i32[TXW_ATT * NL + lane];
    d._pad = 0;
    d.n_steps = sm.i64[TXI_NSTEPS * NL + lane];
    d.n_rejected = sm.i64[TXI_NREJ * NL + lane];
    d.n_rhs = sm.i64[TXI_NRHS * NL + lane];
    q.details[tr] = d;
    out_status[tr] = ctl_finish(sink, tr, st, rc, sm.i32[TXW_EVCNT * NL + lane], d.n_steps);   // final once the run is done
    if (step_io) step_io[tr] = step_ns;
}

// ---- prologue of stage q for the 32 trajectories of a set, run by both helpers of the set: body-fixed position, 1/r, the recursion
// scalars the walkers need, and everything the helpers need to assemble the acceleration of that stage later
enum { AS_R = 0, AS_S = 9, AS_T, AS_U, AS_K0, AS_K1, AS_FAC, AS_P0, AS_P1, AS_P2, AS_COUNT };
// walker inputs.  P = 8, 10 (E = 2P): WK_POW + e = Re z^e, WK_POW + E + 1 + e = Im z^e (e = 0..E), WK_POW + 2E + 1 + e = rho^e (e = 1..E);
// P = 16: WK_POW + 3k = Re z^(2^k), + 1 = Im, + 2 = rho^(2^k)
enum { WK_UB = 0, WK_R2, WK_POW };
template <int P> struct TxWk {
    static constexpr bool ALL = (P != 16);   // every starting power is published
    static constexpr int E = 2 * P;
    static constexpr int COUNT = ALL ? WK_POW + 3 * E + 2 : WK_POW + 18;
    static constexpr int ZR = WK_POW, ZI = WK_POW + E + 1, RH = WK_POW + 2 * E + 1;   // RH + e = rho^e
};

// Stage prologue, run by the two helpers of the context once the position of the stage (ysp) and its DCM (rn) are in shared
// memory: each helper derives (s, t, u, rho) itself, then helper 0 publishes the scalars of the acceleration assembly (as), ub, r2
// and the powers of rho; helper 1 publishes the powers of z the walkers start their columns from (P = 16: the z^(2^k), rho^(2^k)).
template <int P, bool COLD>
__device__ __forceinline__ void tx_prologue(const DevSetup& S, const TxSm& sm, int lane, int par, int j, const double* ysp, long long t_ns) {
    const DevGrav& gv = S.grav;
    const double* rn = sm.rn + par * 9 * NL + lane;
    const double p0 = ysp[lane], p1 = ysp[NL + lane], p2 = ysp[2 * NL + lane];
    double y0 = p0, y1 = p1, y2 = p2;
    double ir_c = 0.0;   // 1/|r| about the integration centre (two-body term)
    if (COLD && S.grav_body >= 0) {   // field of another body: the state is translated to it first (gravity_field.rs:149-154)
        ir_c = rsqrt(fma(y2, y2, fma(y1, y1, y0 * y0)));
        field_offset(S, t_ns, y0, y1, y2);
    }
    const double rb0 = fma(rn[2 * NL], y2, fma(rn[1 * NL], y1, rn[0] * y0));
    const double rb1 = fma(rn[5 * NL], y2, fma(rn[4 * NL], y1, rn[3 * NL] * y0));
    const double rb2 = fma(rn[8 * NL], y2, fma(rn[7 * NL], y1, rn[6 * NL] * y0));
    const double inv_r = rsqrt(fma(rb2, rb2, fma(rb1, rb1, rb0 * rb0)));
    if (S.grav_body < 0) ir_c = inv_r;
    const double rho = gv.r_eq * inv_r;
    const double s_ = rb0 * inv_r, t_ = rb1 * inv_r, u_ = rb2 * inv_r;
    double* wk = sm.wk + par * TxWk<P>::COUNT * NL + lane;
    if (j == 0) {
        wk[WK_UB * NL] = u_ * rho; wk[WK_R2 * NL] = rho * rho;
        double* as = sm.as + par * AS_COUNT * NL + lane;
#pragma unroll
        for (int k = 0; k < 9; ++k) as[(AS_R + k) * NL] = rn[k * NL];
        as[AS_S * NL] = s_; as[AS_T * NL] = t_; as[AS_U * NL] = u_;
        // rr_n A[n][m] = K0 rho (rho^n A),  rr_{n-1} A[n][m] = K0 (rho^n A),  K0 = mu / (r R_eq)
        const double K0 = (gv.mu * gv.inv_r_eq) * inv_r;
        as[AS_K0 * NL] = K0; as[AS_K1 * NL] = K0 * rho;
        as[AS_FAC * NL] = -S.mu_central * ir_c * ir_c * ir_c;   // two-body (orbital.rs:86-92), from the same 1/r when the field is the centre's
        as[AS_P0 * NL] = p0; as[AS_P1 * NL] = p1; as[AS_P2 * NL] = p2;
        if constexpr (TxWk<P>::ALL) {   // rho^1..rho^8 by doubling, then rho^(8+k) = rho^8 rho^k, rho^(16+k) = rho^16 rho^k
            constexpr int E = TxWk<P>::E;
            double rp[9];
            rp[1] = rho;
#pragma unroll
            for (int lo = 1; lo < 8; lo *= 2) {
#pragma unroll
                for (int k = 1; k <= lo; ++k) rp[lo + k] = rp[lo] * rp[k];
            }
            double* wp = wk + TxWk<P>::RH * NL;
            const double r16 = rp[8] * rp[8];
#pragma unroll
            for (int k = 1; k <= 8; ++k) {
                wp[k * NL] = rp[k];
                if (8 + k <= E) wp[(8 + k) * NL] = (k == 8) ? r16 : rp[8] * rp[k];
                if (16 + k <= E) wp[(16 + k) * NL] = r16 * rp[k];
            }
        }
    } else if constexpr (TxWk<P>::ALL) {
        // z^1..z^8 by doubling (z^2; z^3, z^4; z^5..z^8), then z^(8+k) = z^8 z^k, z^(16+k) = z^16 z^k
        constexpr int E = TxWk<P>::E;
        static_assert(E > 8 && E <= 24, "published powers");
        double* wr = wk + TxWk<P>::ZR * NL;
        double* wi = wk + TxWk<P>::ZI * NL;
        double zr[9], zi[9];
        zr[1] = s_; zi[1] = t_;
#pragma unroll
        for (int lo = 1; lo < 8; lo *= 2) {
#pragma unroll
            for (int k = 1; k <= lo; ++k) {
                zr[lo + k] = fma(zr[lo], zr[k], -(zi[lo] * zi[k]));
                zi[lo + k] = fma(zr[lo], zi[k], zi[lo] * zr[k]);
            }
        }
        wr[0] = 1.0; wi[0] = 0.0;
#pragma unroll
        for (int k = 1; k <= 8; ++k) { wr[k * NL] = zr[k]; wi[k * NL] = zi[k]; }
        const double z16r = fma(zr[8], zr[8], -(zi[8] * zi[8])), z16i = 2.0 * zr[8] * zi[8];
#pragma unroll
        for (int k = 1; k <= 8; ++k) {
            if (8 + k <= E) {
                wr[(8 + k) * NL] = (k == 8) ? z16r : fma(zr[8], zr[k], -(zi[8] * zi[k]));
                wi[(8 + k) * NL] = (k == 8) ? z16i : fma(zr[8], zi[k], zi[8] * zr[k]);
            }
            if (16 + k <= E) {
                wr[(16 + k) * NL] = fma(z16r, zr[k], -(z16i * zi[k]));
                wi[(16 + k) * NL] = fma(z16r, zi[k], z16i * zr[k]);
            }
        }
    } else {   // z^(2^k), rho^(2^k): the walkers assemble z^e, rho^(e+1) of their columns from these
        double zr = s_, zi = t_, rp = rho;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            wk[(WK_POW + 3 * k) * NL] = zr; wk[(WK_POW + 3 * k + 1) * NL] = zi; wk[(WK_POW + 3 * k + 2) * NL] = rp;
            const double nr = fma(zr, zr, -(zi * zi));
            zi = 2.0 * zr * zi; zr = nr; rp *= rp;
        }
    }
}

// inertial -> body-fixed DCM at the stage time: first-order update of the (slow) pole angles, exact angle addition for the
// prime-meridian angle (the stage epoch is ns-truncated, cosmic/mod.rs:102)
struct TxRotBase { double sa, ca, sd, cd, sw, cw; };
__device__ __forceinline__ void tx_dcm(const DevRotation& rot, const TxRotBase& b, long long off_ns, double (&R)[9]) {
    if (rot.kind == 0) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        return;
    }
    const double dt_s = (double)off_ns * 1e-9;
    const double da = rot.ra_dot * dt_s, dd = rot.dec_dot * dt_s, dw = rot.wdot * dt_s;
    const double sa = fma(b.ca, da, b.sa), ca = fma(-b.sa, da, b.ca);
    const double sd = fma(b.cd, dd, b.sd), cd = fma(-b.sd, dd, b.cd);
    double sdl, cdl;
    if (fabs(dw) < 0.02) {
        const double z = dw * dw;
        sdl = dw * fma(z, fma(z, 1.0 / 120.0, -1.0 / 6.0), 1.0);
        cdl = fma(z, fma(z, fma(z, -1.0 / 720.0, 1.0 / 24.0), -0.5), 1.0);
    } else {
        det_sincos(dw, sdl, cdl);
    }
    const double sw = fma(b.sw, cdl, b.cw * sdl), cw = fma(b.cw, cdl, -(b.sw * sdl));
    const double b00 = -sa, b01 = ca;
    const double b10 = -(sd * ca), b11 = -(sd * sa), b12 = cd;
    R[0] = fma(cw, b00, sw * b10); R[1] = fma(cw, b01, sw * b11); R[2] = sw * b12;
    R[3] = fma(cw, b10, -(sw * b00)); R[4] = fma(cw, b11, -(sw * b01)); R[5] = cw * b12;
    R[6] = cd * ca; R[7] = cd * sa; R[8] = sd;
}

// orientation angles of the field's body-fixed frame at `epoch` (deterministic sin / cos: the per-step evaluation of the oracle)
__device__ __forceinline__ TxRotBase tx_rot_base(const DevRotation& rot, long long epoch) {
    TxRotBase b;
    const double t_s = dur_to_seconds(epoch);
    const double d = t_s / 86400.0;
    const double Tc = d / 36525.0;
    det_sincos((rot.ra0 + rot.ra1 * Tc) * NYXB_DEG2RAD, b.sa, b.ca);
    det_sincos((rot.dec0 + rot.dec1 * Tc) * NYXB_DEG2RAD, b.sd, b.cd);
    det_sincos(fmod(rot.w0 + rot.w1 * d, 360.0) * NYXB_DEG2RAD, b.sw, b.cw);
    return b;
}
__device__ __forceinline__ void tx_rot_store(double* rot, int lane, const TxRotBase& b) {
    rot[lane] = b.sa; rot[NL + lane] = b.ca; rot[2 * NL + lane] = b.sd; rot[3 * NL + lane] = b.cd; rot[4 * NL + lane] = b.sw;
    rot[5 * NL + lane] = b.cw;
}

// the right-hand side has terms beyond the harmonic field (accel_cold)
__host__ __device__ inline bool tx_cold(const DevSetup& S) { return S.n_bodies > 0 || S.has_srp || S.has_drag || S.n_xgrav > 0; }

// z^W, rho^(W+1) (sequence a) and z^(2^NB - 1 - W), rho^(2^NB - W) (sequence b) from the published z^(2^k), rho^(2^k): W and its
// complement split the NB powers between them; the first factor of each product is a copy
template <int W, int NB>
__device__ __forceinline__ void tx_start_powers(const double* wk, double& zar, double& zai, double& pa, double& zbr, double& zbi, double& pb) {
    const double rho = wk[(WK_POW + 2) * NL];
    bool fa = true, fb = true;
    zar = 1.0; zai = 0.0; zbr = 1.0; zbi = 0.0; pa = rho; pb = rho;
#pragma unroll
    for (int k = 0; k < NB; ++k) {
        const double br = wk[(WK_POW + 3 * k) * NL], bi = wk[(WK_POW + 3 * k + 1) * NL], bp = wk[(WK_POW + 3 * k + 2) * NL];
        if ((W >> k) & 1) {
            if (fa) { zar = br; zai = bi; fa = false; }
            else { const double nr = fma(zar, br, -(zai * bi)); zai = fma(zar, bi, zai * br); zar = nr; }
            pa *= bp;
        } else {
            if (fb) { zbr = br; zbi = bi; fb = false; }
            else { const double nr = fma(zbr, br, -(zbi * bi)); zbi = fma(zbr, bi, zbi * br); zbr = nr; }
            pb *= bp;
        }
    }
}

// COLD: the setup has third bodies, SRP, drag, further fields or a field about another body (accel_cold / field_offset).  Without
// it the helpers' stage loop has no call in it: the values live across those calls were what spilled to local memory.
template <int P, int NCTX, bool COLD>
__global__ void __launch_bounds__((P + HW * NCTX) * 32, 1)
nyxb_k_tx(const __grid_constant__ DevSetup S, const __grid_constant__ DevTx Tx, const __grid_constant__ DevTxQueue q, size_t n,
          const double* __restrict__ state, const double* __restrict__ consts, const long long* __restrict__ epoch0,
          long long end_epoch, long long* step_io, double* out_state, long long* out_epoch, int* out_status, const DevSink sink,
          unsigned blob_bytes, unsigned off_recK, unsigned off_seed, unsigned off_sched) {
    static_assert(P <= NYXB_TX_MAXP && NCTX >= 1 && NCTX <= 2, "walker positions / set contexts");
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long tma_bar;
    // READY[context][parity]: "the walker inputs of the next stage with this parity are published" — an mbarrier (64 arrivals: the
    // two helpers of the context) rather than a named barrier, because the walkers POLL it: a walker warp takes whichever
    // context has a stage ready, so the serial stretch between two step attempts of one set (error norm, controller, commit,
    // first prologue) is covered by the other set's stages instead of stalling the walkers.
    __shared__ __align__(8) unsigned long long ready_bar[NCTX][2];
    __shared__ int s_set[NCTX], s_fresh[NCTX], s_exit[NCTX], s_done[NCTX], s_slice_end[NCTX];
    __shared__ __align__(8) unsigned long long kick_bar;   // context 0 arrives half-way through its first attempt: context 1 starts then
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
#ifdef NYXB_TX_TRACE
    int tr_n = 0;
#endif
    constexpr int NPOW = 6;   // P = 16: z^(2^k), k < NPOW: bits of the exponents below 2P, and the common ratio z^(2P)
    static_assert(P == 8 || P == 10 || P == 16, "walker positions");
    constexpr int NT_RW = (P + HW) * 32;   // threads on a DONE barrier: the walkers + the helpers of the context
    constexpr int NT_HB = HW * 32;         // threads on the helpers' own barrier and arrivals on READY
    // named barriers of context c: HB (helpers among themselves), READY[parity], DONE[parity]
    constexpr int BAR_PER_CTX = 5;
    const int N = S.grav.N;
    const int stages = S.tb.stages;
    const TxLayout L = tx_layout(blob_bytes, P, N, NCTX);
    const double2* recA = reinterpret_cast<const double2*>(smem + L.blob);
    const double* recK = reinterpret_cast<const double*>(smem + L.blob + off_recK);
    const double* colseed = reinterpret_cast<const double*>(smem + L.blob + off_seed);
    const int* sched = reinterpret_cast<const int*>(smem + L.blob + off_sched);

    // ---- CTA-shared tables (records, column seeds, schedule): ONE TMA bulk copy
    if (tid == 0) {
        mbar_init(&tma_bar, 1);
#pragma unroll
        mbar_init(&kick_bar, 1);
#pragma unroll
        for (int c = 0; c < NCTX; ++c) {
            s_exit[c] = 0;
            mbar_init(&ready_bar[c][0], NT_HB);
            mbar_init(&ready_bar[c][1], NT_HB);
        }
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&tma_bar, blob_bytes);
        tma_bulk_g2s(smem + L.blob, Tx.recA, blob_bytes, &tma_bar);
    }
    mbar_wait(&tma_bar, 0);
    __syncthreads();   // the last CTA-wide barrier: from here on walkers and helpers meet on named barriers only

    if (w < P) {
        // =============================================================================================== WALKER
        // Walks its columns for stage 0, 1, 2, ... of whichever set each context holds; the inputs of stage i live in the
        // parity-(i & 1) buffers.  The harmonic sum of stage i+1 needs only the POSITION of that stage, which depends on the
        // accelerations up to stage i-1 (second-order system): the helpers publish it one walk ahead, so the walkers never wait for
        // the stage they have just finished — only, once per step, for the controller.
        // column position of this warp.  A warp's scheduler is warp id mod 4; with P = 8 every scheduler hosts walkers w and w + 4
        // and one helper (warps 8..11).  The zigzag gives the low positions a third column and a few more padded entries
        // (N = 21: 34 32 32 30 30 30 28 28), so position k shares its scheduler with position 7 - k: 34+28, 32+28, 32+30, 30+30.
        const int pos = (P == 8 && w >= 4) ? 11 - w : w;   // warp 0..7 -> 0 1 2 3 7 6 5 4
        const int* my = sched + pos * (2 + 2 * Tx.kmax);
        const int rec_off = my[0], ncol = my[1];
        unsigned active = (1u << NCTX) - 1u;
        unsigned phases = 0;   // bit 2c + par: parity of the READY[c][par] phase this warp waits for next
        const unsigned ready0 = smem_u32(&ready_bar[0][0]);   // READY[c][par] lives at ready0 + 8 (2 c + par)
        int stage0 = 0, stage1 = 0, pref = 0;
        while (active) {
            {
                // pick a context whose next stage is published: the one not served last first
                int c = -1, par = 0;
                TX_TRACE(TR_POLL, 0, 0);
                for (;;) {
#pragma unroll
                    for (int k = 0; k < NCTX; ++k) {
                        const int cc = (pref + k) % NCTX;
                        if (c >= 0 || !((active >> cc) & 1u)) continue;
                        const int pp = (cc == 0 ? stage0 : stage1) & 1;
                        const bool ok = tx_mbar_test(ready0 + 8u * (unsigned)(2 * cc + pp), (phases >> (2 * cc + pp)) & 1u);
                        if (__all_sync(FULL, ok)) { c = cc; par = pp; }
                    }
                    if (c >= 0) break;
                    __nanosleep(20);
                }
                phases ^= 1u << (2 * c + par);
                const int st = (c == 0) ? stage0 : stage1;
                if (st == 0 && *(volatile int*)&s_exit[c]) { active &= ~(1u << c); continue; }
                const int stn = (st + 1 == stages) ? 0 : st + 1;
                if (c == 0) stage0 = stn; else stage1 = stn;
                pref = (c + 1) % NCTX;
                TX_TRACE(TR_WALK, c, st);
                const TxSm sm = tx_views(smem, L, c, N);
                // z^e = (cos, sin)(e lambda) cos^e(phi) and rho^(e+1) for the two interleaved exponent sequences of this position:
                // e = pos + 2P j (za, pa) and e = 2P-1-pos + 2P j (zb, pb)
                TxLaneState t;
                const double* wk = sm.wk + par * TxWk<P>::COUNT * NL + lane;
                t.ub = wk[WK_UB * NL]; t.r2 = wk[WK_R2 * NL];
                t.dc = t.ub + t.ub; t.dg = t.r2 + t.r2;
                if constexpr (TxWk<P>::ALL) {   // published: z^pos, z^(2P-1-pos), z^(2P), rho^(pos+1), rho^(2P-pos), rho^(2P)
                    constexpr int E = TxWk<P>::E;
                    t.zar = wk[(TxWk<P>::ZR + pos) * NL]; t.zai = wk[(TxWk<P>::ZI + pos) * NL];
                    t.pa = wk[(TxWk<P>::RH + pos + 1) * NL];
                    t.zbr = wk[(TxWk<P>::ZR + E - 1 - pos) * NL]; t.zbi = wk[(TxWk<P>::ZI + E - 1 - pos) * NL];
                    t.pb = wk[(TxWk<P>::RH + E - pos) * NL];
                    t.qr = wk[(TxWk<P>::ZR + E) * NL]; t.qi = wk[(TxWk<P>::ZI + E) * NL]; t.qp = wk[(TxWk<P>::RH + E) * NL];
                } else {
                    switch (pos) {   // one specialised copy per position: the choices below are compile-time there
#define NYXB_TX_CASE(WW) case WW: tx_start_powers<WW, NPOW - 1>(wk, t.zar, t.zai, t.pa, t.zbr, t.zbi, t.pb); break;
                        NYXB_TX_CASE(0) NYXB_TX_CASE(1) NYXB_TX_CASE(2) NYXB_TX_CASE(3) NYXB_TX_CASE(4) NYXB_TX_CASE(5) NYXB_TX_CASE(6) NYXB_TX_CASE(7)
                        NYXB_TX_CASE(8) NYXB_TX_CASE(9) NYXB_TX_CASE(10) NYXB_TX_CASE(11) NYXB_TX_CASE(12) NYXB_TX_CASE(13) NYXB_TX_CASE(14)
                        default: tx_start_powers<15, NPOW - 1>(wk, t.zar, t.zai, t.pa, t.zbr, t.zbi, t.pb); break;
#undef NYXB_TX_CASE
                    }
                    t.qr = wk[(WK_POW + 3 * (NPOW - 1)) * NL]; t.qi = wk[(WK_POW + 3 * (NPOW - 1) + 1) * NL];   // z^(2P)
                    t.qp = wk[(WK_POW + 3 * (NPOW - 1) + 2) * NL];                                             // rho^(2P)
                }
                t.X = 0.0; t.Y = 0.0; t.Z = 0.0; t.W = 0.0;
                const double2* A = recA + 2 * rec_off;
                const double* K = recK + rec_off;
                double2 a01 = A[0], a23 = A[1];
                double kk = K[0];
                // one loop over the columns; the roles of the two sequences are swapped after every column.  The seeds of the next
                // column are fetched before the current one is walked.
                int len = my[3];
                {
                    const double4 sd = *reinterpret_cast<const double4*>(colseed + 4 * my[2]);
                    t.cQ = t.pa * sd.x; t.cc1 = sd.w * t.ub; t.cg = sd.w * t.r2;
                    t.cS5 = t.cQ * sd.y; t.cS6 = t.cQ * sd.z;
                }
                // two columns per trip: the first belongs to sequence a, the second to sequence b (no exchange of the two register
                // sets); the set-up of the next column needs only the OTHER sequence's rho power, which is already there, and the
                // advance of the sequence just used (one complex product) is off every dependent path until two columns later
                for (int k = 0; k < ncol; k += 2) {
                    {
                        const int len_n = my[5 + 2 * k];   // the schedule rows end with a null column (all-zero seeds)
                        const double4 sd_n = *reinterpret_cast<const double4*>(colseed + 4 * my[4 + 2 * k]);
                        tx_column<false>(A, K, a01, a23, kk, len, t);
                        t.cQ = t.pb * sd_n.x; t.cc1 = sd_n.w * t.ub; t.cg = sd_n.w * t.r2;
                        t.cS5 = t.cQ * sd_n.y; t.cS6 = t.cQ * sd_n.z;
                        const double nr = fma(t.zar, t.qr, -(t.zai * t.qi));
                        t.zai = fma(t.zar, t.qi, t.zai * t.qr); t.zar = nr; t.pa *= t.qp;
                        len = len_n;
                    }
                    if (k + 1 >= ncol) break;
                    {
                        const int len_n = my[7 + 2 * k];
                        const double4 sd_n = *reinterpret_cast<const double4*>(colseed + 4 * my[6 + 2 * k]);
                        tx_column<true>(A, K, a01, a23, kk, len, t);
                        t.cQ = t.pa * sd_n.x; t.cc1 = sd_n.w * t.ub; t.cg = sd_n.w * t.r2;
                        t.cS5 = t.cQ * sd_n.y; t.cS6 = t.cQ * sd_n.z;
                        const double nr = fma(t.zbr, t.qr, -(t.zbi * t.qi));
                        t.zbi = fma(t.zbr, t.qi, t.zbi * t.qr); t.zbr = nr; t.pb *= t.qp;
                        len = len_n;
                    }
                }
                double* pt = sm.part + ((par * P + pos) * 4) * NL + lane;
                pt[0] = t.X; pt[NL] = t.Y; pt[2 * NL] = t.Z; pt[3 * NL] = t.W;
                nb_arrive(1 + c * BAR_PER_CTX + 3 + par, NT_RW);   // DONE[par]: the partial sums of this position are in shared memory
                TX_TRACE(TR_WALK_END, c, st);
            }
        }
        return;
    }

    // =================================================================================================== HELPER
    // set context; two helpers per set, lane = trajectory of the set:
    //   helper 0 (lead): candidate state and error estimate of the positions, the DCMs of stage 0 and of every stage i+2, the
    //                    controller, the set queue, loading and parking the controller state;
    //   helper 1:        the state vector (load, stage-0 and stage-1 inputs, commit, park), reduction of the partial sums, the acceleration (with accel_cold) of all three components, V_{i+1} and
    //                    P_{i+2} (both need the acceleration just assembled, so they stay on the warp that has it), candidate state
    //                    and error estimate of the velocities, the DCM of stage 1 and the orientation angles of the next step.
    // Both derive the stage prologue (tx_prologue) and split what it publishes.
    const int c = (w - P) / HW, j = (w - P) % HW;
    const TxSm sm = tx_views(smem, L, c, N);
    const int BAR_HB = 1 + c * BAR_PER_CTX, BAR_DONE = BAR_HB + 3;
    const DevGrav& gv = S.grav;
    const bool has_extra = COLD && tx_cold(S);
    const bool lead = (j == 0);
    const double* ta = S.tb.a;    // a_{q,m} (stage q >= 1, m < q) = ta[(q - 1) * NYXB_MAX_STAGES + m]

    // The two sets of a CTA must not reach the serial stretch between two attempts (error norm, controller, commit, first
    // prologues: ~11 000 clocks without work for the walkers) at the same time, and nothing pulls them apart once they run in
    // phase (measured: both contexts started together stayed within 1 % of an attempt of each other, and the walkers idled through
    // every such stretch).  Context 1 therefore starts when context 0 is half-way through its first attempt.
    bool kick_pending = (NCTX > 1 && c == 0 && lead);
    if (NCTX > 1 && c == 1) {
        if (lead && lane == 0) mbar_wait(&kick_bar, 0);
        nb_sync(BAR_HB, NT_HB);
    }

    for (;;) {
        // ---------------------------------------------------------------- acquire a set: a fresh one, else a parked one
        if (lead && lane == 0) {
            int set = -1, fresh = 0;
            if (atomicAdd(q.ctl + TXQ_FRESH, 0) < q.n_sets) {
                const int f = atomicAdd(q.ctl + TXQ_FRESH, 1);
                if (f < q.n_sets) { set = f; fresh = 1; }
            }
            if (set < 0 && q.slice > 0) {
                while (atomicCAS(q.ctl + TXQ_LOCK, 0, 1) != 0) __nanosleep(64);
                __threadfence();
                volatile int* vc = q.ctl;
                const int head = vc[TXQ_HEAD], tail = vc[TXQ_TAIL];
                if (head < tail) {
                    set = ((volatile int*)q.ring)[head % q.n_sets];
                    vc[TXQ_HEAD] = head + 1;
                }
                __threadfence();
                atomicExch(q.ctl + TXQ_LOCK, 0);
            }
            s_set[c] = set; s_fresh[c] = fresh;
            s_exit[c] = set < 0;   // nothing fresh, nothing parked: every unfinished set is in progress in another context
        }
        nb_sync(BAR_HB, NT_HB);
        if (s_exit[c] && kick_pending && lane == 0) tx_mbar_arrive(&kick_bar);
        if (s_exit[c]) {
            tx_mbar_arrive(&ready_bar[c][0]);   // releases the walkers (they expect stage 0), which read s_exit and drop this context
            return;
        }
        const int set = s_set[c];
        const int round = s_fresh[c] ? 0 : 1;   // 0: initial state from the inputs; otherwise from the parking area
        const size_t traj_raw = (size_t)set * NL + lane;
        const bool valid = traj_raw < n;
        const size_t tr = valid ? traj_raw : (size_t)set * NL;   // an absent lane shadows the set's first trajectory, never committed

        // ---------------------------------------------------------------- load the set
        if (!lead) {
#pragma unroll
            for (int cc = 0; cc < 6; ++cc) {
                const double yc = (round == 0) ? state[(size_t)cc * n + tr] : __ldcg(out_state + (size_t)cc * n + tr);
                sm.ycur[cc * NL + lane] = yc;
                if (round == 0 && valid && sink.cap > 0) sink.state[((size_t)cc * sink.cap) * n + tr] = yc;
            }
        } else {
            tx_load_ctl(S, sink, q, sm, lane, n, tr, valid, round, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch);
            tx_pick_step(sm, lane, end_epoch);
            const bool done = sm.i32[TXW_FLAGS * NL + lane] & F_DONE;
            const bool all = __all_sync(FULL, done);
            if (lane == 0) { s_done[c] = all; s_slice_end[c] = 0; }
            if (gv.rot.kind != 0) tx_rot_store(sm.rot, lane, tx_rot_base(gv.rot, sm.i64[TXI_EPOCH * NL + lane]));
        }
        nb_sync(BAR_HB, NT_HB);

        // ---------------------------------------------------------------- step attempts of this slice
        for (int it = 0; !s_done[c]; ++it) {
            TX_TRACE(TR_TOP, c, 0);
            const double h = sm.f64[TXF_H * NL + lane];
            const long long epoch = sm.i64[TXI_EPOCH * NL + lane];
            // orientation angles at the step epoch (the lead evaluates every DCM of the attempt but that of stage 1).  They are NOT
            // evaluated here, on the serial path between two attempts: helper 1 evaluates them for the epoch this attempt leads to
            // while the walkers are busy, and commits them to sm.rot when the controller accepts the step (a rejected step keeps its
            // epoch).
            TxRotBase rb_;
            rb_.sa = 0.0; rb_.ca = 1.0; rb_.sd = 1.0; rb_.cd = 0.0; rb_.sw = 0.0; rb_.cw = 1.0;
            const bool fixed = sm.i32[TXW_FLAGS * NL + lane] & F_FIXED;
            double Rn[9];
            // ---- prime the pipeline: stage 0 (the state itself) and stage 1 (needs only V_0 = v): instance.rs:369-394
            const long long off1 = (stages > 1) ? dur_from_seconds(S.tb.c[0] * h) : 0;
            if (!lead) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const double r_k = sm.ycur[k * NL + lane], v_k = sm.ycur[(3 + k) * NL + lane];
                    sm.kst[(0 * 6 + k) * NL + lane] = v_k;                                            // k_0[k] = V_0
                    sm.ysp[(0 * 3 + k) * NL + lane] = r_k;                                            // P_0
                    if (stages > 1) sm.ysp[(1 * 3 + k) * NL + lane] = fma(h, ta[0] * v_k, r_k);      // P_1 = r + h a_10 V_0
                }
            }
            nb_sync(BAR_HB, NT_HB);
            TX_TRACE(TR_PRIMED, c, 0);
            if (gv.rot.kind != 0) {   // committed by helper 1 before the barrier above
                rb_.sa = sm.rot[lane]; rb_.ca = sm.rot[NL + lane]; rb_.sd = sm.rot[2 * NL + lane]; rb_.cd = sm.rot[3 * NL + lane];
                rb_.sw = sm.rot[4 * NL + lane]; rb_.cw = sm.rot[5 * NL + lane];
            }
            TxRotBase rb_next = rb_;
            if (lead) {
                tx_dcm(gv.rot, rb_, 0, Rn);
#pragma unroll
                for (int k = 0; k < 9; ++k) sm.rn[k * NL + lane] = Rn[k];
            } else if (stages > 1) {   // the DCM of stage 1 in parallel with the lead's (both sat on the serial path between attempts)
                tx_dcm(gv.rot, rb_, off1, Rn);
#pragma unroll
                for (int k = 0; k < 9; ++k) sm.rn[(9 + k) * NL + lane] = Rn[k];
            }
            nb_sync(BAR_HB, NT_HB);
            TX_TRACE(TR_DCM01, c, 0);
            tx_prologue<P, COLD>(S, sm, lane, 0, j, sm.ysp, epoch);
            tx_mbar_arrive(&ready_bar[c][0]);
            TX_TRACE(TR_READY, c, 0);
            if (stages > 1) {
                tx_prologue<P, COLD>(S, sm, lane, 1, j, sm.ysp + 3 * NL, epoch + off1);
                tx_mbar_arrive(&ready_bar[c][1]);
                TX_TRACE(TR_READY, c, 1);
            }
            nb_sync(BAR_HB, NT_HB);   // the lead overwrites rn[0] (DCM of stage 2) in the first slack below: both helpers have read it by now
            // ---- derive(): the stages of one attempt for the 32 trajectories (instance.rs:358-493), one walk ahead of the walkers.
            // Candidate state and error estimate (instance.rs:402-414) accumulate stage by stage in the reference's order.  Per stage
            // both helpers pass DONE[par] and, before the last stage, HB and the prologue of stage i+2, in the same order.
            if (lead) {
                double nx_r[3], er_r[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) { nx_r[k] = sm.ycur[k * NL + lane]; er_r[k] = 0.0; }
                for (int i = 0; i < stages; ++i) {
                    const int par = i & 1;
                    // -- slack: position side of the sums (V_i is known), DCM of stage i+2
                    long long off2 = 0;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const double vi = sm.kst[(i * 6 + k) * NL + lane];   // V_i
                        if (!fixed) er_r[k] = fma(h * S.tb.e[i], vi, er_r[k]);
                        nx_r[k] = fma(h * S.tb.b[i], vi, nx_r[k]);
                    }
                    if (i + 2 < stages) {   // DCM of stage i+2 (its parity buffer was last read in the prologue of stage i, two barriers ago)
                        off2 = dur_from_seconds(S.tb.c[i + 1] * h);
                        TX_TRACE(TR_PRE_DONE, c, i);
                        tx_dcm(gv.rot, rb_, off2, Rn);
#pragma unroll
                        for (int k = 0; k < 9; ++k) sm.rn[(par * 9 + k) * NL + lane] = Rn[k];
                    }
                    TX_TRACE(TR_DCM_DONE, c, i);
                    if (kick_pending && i == stages / 2) {
                        if (lane == 0) tx_mbar_arrive(&kick_bar);
                        kick_pending = false;
                    }
                    TX_TRACE(TR_DONE_WAIT, c, i);
                    nb_sync(BAR_DONE + par, NT_RW);   // the walkers' partial sums of stage i are back
                    TX_TRACE(TR_DONE_SEEN, c, i);
                    if (i + 1 < stages) {
                        nb_sync(BAR_HB, NT_HB);   // V_{i+1} and the position of stage i+2 are in shared memory
                        TX_TRACE(TR_HB_PASSED, c, i);
                        if (i + 2 < stages) {
                            tx_prologue<P, COLD>(S, sm, lane, par, 0, sm.ysp + par * 3 * NL, epoch + off2);
                            tx_mbar_arrive(&ready_bar[c][par]);   // walker inputs of stage i+2 are published
                            TX_TRACE(TR_READY, c, i + 2);
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) { sm.nxt[k * NL + lane] = nx_r[k]; sm.er[k * NL + lane] = er_r[k]; }
            } else {
                double r_own[3], v_own[3], nx_v[3], er_v[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    r_own[k] = sm.ycur[k * NL + lane]; v_own[k] = sm.ycur[(3 + k) * NL + lane];
                    nx_v[k] = v_own[k]; er_v[k] = 0.0;
                }
                int rc_acc = 0;
                for (int i = 0; i < stages; ++i) {
                    const int par = i & 1;
                    // -- slack: everything that does not need the acceleration of stage i
                    double preV[3] = {0.0, 0.0, 0.0}, preP[3] = {0.0, 0.0, 0.0};
                    long long off2 = 0;
                    if (i == 0 && gv.rot.kind != 0)
                        rb_next = tx_rot_base(gv.rot, epoch + (fixed ? sm.i64[TXI_STEP * NL + lane] : dur_from_seconds(h)));
                    if (i + 1 < stages) {   // V_{i+1} = v + h sum_{l<=i} a_{i+1,l} A_l: all terms but the last
                        const double* arow = ta + i * NYXB_MAX_STAGES;
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                            const double* kc = sm.kst + (3 + k) * NL + lane;
                            double w0 = 0.0, w1 = 0.0;
                            int l = 0;
                            for (; l + 1 < i; l += 2) { w0 = fma(arow[l], kc[l * 6 * NL], w0); w1 = fma(arow[l + 1], kc[(l + 1) * 6 * NL], w1); }
                            if (l < i) w0 = fma(arow[l], kc[l * 6 * NL], w0);
                            preV[k] = w0 + w1;
                        }
                    }
                    if (i + 2 < stages) {   // P_{i+2} = r + h sum_{m<=i+1} a_{i+2,m} V_m: all terms but the last (V_i is known)
                        const double* arow = ta + (i + 1) * NYXB_MAX_STAGES;
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                            const double* kc = sm.kst + k * NL + lane;
                            double w0 = 0.0, w1 = 0.0;
                            int m = 0;
                            for (; m + 1 <= i; m += 2) { w0 = fma(arow[m], kc[m * 6 * NL], w0); w1 = fma(arow[m + 1], kc[(m + 1) * 6 * NL], w1); }
                            if (m <= i) w0 = fma(arow[m], kc[m * 6 * NL], w0);
                            preP[k] = w0 + w1;
                        }
                        off2 = dur_from_seconds(S.tb.c[i + 1] * h);
                        TX_TRACE(TR_PRE_DONE, c, i);
                    }
                    TX_TRACE(TR_DONE_WAIT, c, i);
                    nb_sync(BAR_DONE + par, NT_RW);   // the walkers' partial sums of stage i are back
                    TX_TRACE(TR_DONE_SEEN, c, i);

                    // -- reduce the partial sums, assemble the acceleration of stage i (spacecraft.rs:216-247)
                    double X, Y, Z, Wt;
                    {
                        double ax[4] = {0.0, 0.0, 0.0, 0.0}, ay[4] = {0.0, 0.0, 0.0, 0.0}, az[4] = {0.0, 0.0, 0.0, 0.0}, aw4[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            const double* pt = sm.part + ((par * P + p) * 4) * NL + lane;
                            ax[p & 3] += pt[0]; ay[p & 3] += pt[NL]; az[p & 3] += pt[2 * NL]; aw4[p & 3] += pt[3 * NL];
                        }
                        X = (ax[0] + ax[1]) + (ax[2] + ax[3]); Y = (ay[0] + ay[1]) + (ay[2] + ay[3]);
                        Z = (az[0] + az[1]) + (az[2] + az[3]); Wt = (aw4[0] + aw4[1]) + (aw4[2] + aw4[3]);
                    }
                    TX_TRACE(TR_REDUCED, c, i);
                    const double* as = sm.as + par * AS_COUNT * NL + lane;
                    const double K0 = as[AS_K0 * NL], K1 = as[AS_K1 * NL];
                    const double aw = -K0 * Wt;
                    const double ab0 = fma(aw, as[AS_S * NL], K1 * X), ab1 = fma(aw, as[AS_T * NL], K1 * Y), ab2 = fma(aw, as[AS_U * NL], K1 * Z);
                    double acc[3];
#pragma unroll
                    for (int k = 0; k < 3; ++k)
                        acc[k] = fma(as[AS_FAC * NL], as[(AS_P0 + k) * NL],
                                     fma(as[(AS_R + 6 + k) * NL], ab2, fma(as[(AS_R + 3 + k) * NL], ab1, as[(AS_R + k) * NL] * ab0)));
                    if (has_extra) {
                        double yy[9], aa[3] = {0.0, 0.0, 0.0};
                        const double hz = (i > 0) ? h * 0.0 : 0.0;
                        yy[0] = as[AS_P0 * NL]; yy[1] = as[AS_P1 * NL]; yy[2] = as[AS_P2 * NL];
#pragma unroll
                        for (int e = 0; e < 3; ++e) yy[3 + e] = sm.kst[(i * 6 + e) * NL + lane];   // V_i
                        yy[6] = sm.f64[TXF_CR * NL + lane] + hz; yy[7] = sm.f64[TXF_CD * NL + lane] + hz; yy[8] = sm.f64[TXF_PM * NL + lane] + hz;
                        const long long offi = (i > 0) ? dur_from_seconds(S.tb.c[i - 1] * h) : 0;
                        const int rcx = accel_cold<true>(S, sm.f64[TXF_DRY * NL + lane], sm.f64[TXF_EXTRA * NL + lane], sm.f64[TXF_SRPA * NL + lane],
                                                         sm.f64[TXF_DRAGA * NL + lane], epoch + offi, yy, aa);
#pragma unroll
                        for (int k = 0; k < 3; ++k) acc[k] += aa[k];
                        if (rcx && !rc_acc) rc_acc = rcx | ((i + 1) << 8);
                    }
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        sm.kst[(i * 6 + 3 + k) * NL + lane] = acc[k];     // k_i[3+k] = A_i
                        if (!fixed) er_v[k] = fma(h * S.tb.e[i], acc[k], er_v[k]);
                        nx_v[k] = fma(h * S.tb.b[i], acc[k], nx_v[k]);
                    }
                    if (i + 1 < stages) {
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                            const double vn = fma(h, fma(ta[i * NYXB_MAX_STAGES + i], acc[k], preV[k]), v_own[k]);   // V_{i+1}
                            sm.kst[((i + 1) * 6 + k) * NL + lane] = vn;                                            // k_{i+1}[k]
                            if (i + 2 < stages)
                                sm.ysp[(par * 3 + k) * NL + lane] = fma(h, fma(ta[(i + 1) * NYXB_MAX_STAGES + i + 1], vn, preP[k]), r_own[k]);   // P_{i+2}
                        }
                        TX_TRACE(TR_ACC_DONE, c, i);
                        nb_sync(BAR_HB, NT_HB);   // V_{i+1} and the position of stage i+2 are in shared memory
                        TX_TRACE(TR_HB_PASSED, c, i);
                        if (i + 2 < stages) {
                            tx_prologue<P, COLD>(S, sm, lane, par, 1, sm.ysp + par * 3 * NL, epoch + off2);
                            tx_mbar_arrive(&ready_bar[c][par]);   // walker inputs of stage i+2 are published
                            TX_TRACE(TR_READY, c, i + 2);
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) { sm.nxt[(3 + k) * NL + lane] = nx_v[k]; sm.er[(3 + k) * NL + lane] = er_v[k]; }
                sm.i32[TXW_RCST * NL + lane] = rc_acc;
            }
            TX_TRACE(TR_STAGES_END, c, 0);
            nb_sync(BAR_HB, NT_HB);
            TX_TRACE(TR_CTRL_IN, c, 0);
            if (lead) {
                tx_controller(S, sink, sm, lane, n, tr, stages);
                TX_TRACE(TR_CTRL_OUT, c, 0);
                const bool slice_end = q.slice > 0 && it + 1 >= q.slice;
                if (!slice_end) tx_pick_step(sm, lane, end_epoch);
                TX_TRACE(TR_PICKED, c, 0);
                const bool done = sm.i32[TXW_FLAGS * NL + lane] & F_DONE;
                const bool all = __all_sync(FULL, done);
                if (lane == 0) { s_done[c] = all; s_slice_end[c] = slice_end; }
            }
            nb_sync(BAR_HB, NT_HB);
            TX_TRACE(TR_CTRL_END, c, 0);
            if (!lead && sm.i32[TXW_ACC * NL + lane]) {
                if (gv.rot.kind != 0) tx_rot_store(sm.rot, lane, rb_next);   // read by both helpers after the next HB barrier
                const long long ns = sm.i64[TXI_NSTEPS * NL + lane];
#pragma unroll
                for (int cc = 0; cc < 6; ++cc) {
                    const double nx = sm.nxt[cc * NL + lane];
                    sm.ycur[cc * NL + lane] = nx;
                    // the channel send of instance.rs:186-193 / 255-259: lanes are consecutive trajectories, one 256-byte store per warp
                    if (valid && ns < sink.cap) sink.state[((size_t)cc * sink.cap + (size_t)ns) * n + tr] = nx;
                }
            }
            TX_TRACE(TR_COMMITTED, c, 0);
            if (s_slice_end[c]) break;
        }

        if (kick_pending) {
            if (lane == 0) tx_mbar_arrive(&kick_bar);
            kick_pending = false;
        }
        // ---------------------------------------------------------------- park the set (== final outputs when it is done)
        if (!lead && valid) {
#pragma unroll
            for (int cc = 0; cc < 6; ++cc) out_state[(size_t)cc * n + tr] = sm.ycur[cc * NL + lane];
        }
        if (lead) tx_park_ctl(sink, q, sm, lane, n, tr, step_io, out_state, out_epoch, out_status);
        __threadfence();
        nb_sync(BAR_HB, NT_HB);
        if (lead && lane == 0 && !s_done[c]) {   // park: the set becomes resumable by any context
            while (atomicCAS(q.ctl + TXQ_LOCK, 0, 1) != 0) __nanosleep(64);
            __threadfence();
            volatile int* vc = q.ctl;
            const int tail = vc[TXQ_TAIL];
            ((volatile int*)q.ring)[tail % q.n_sets] = set;
            vc[TXQ_TAIL] = tail + 1;
            __threadfence();
            atomicExch(q.ctl + TXQ_LOCK, 0);
        }
        nb_sync(BAR_HB, NT_HB);   // s_* of this context are rewritten by its lead lane only after this barrier
    }
}

// walker positions and set contexts for a field of degree N: two sets in flight while both fit in shared memory
template <int P, int NCTX, bool COLD>
cudaError_t tx_launch_p(const DevSetup* S, const DevTx* Tx, const DevTxQueue* q, size_t n, const double* state, const double* consts,
                        const long long* epoch0, long long end_epoch, long long* step_io, double* out_state, long long* out_epoch,
                        int* out_status, const DevSink* sink, int grid, size_t smem, unsigned blob_bytes, unsigned off_recK,
                        unsigned off_seed, unsigned off_sched, cudaStream_t stream) {
    cudaError_t e = cudaFuncSetAttribute(nyxb_k_tx<P, NCTX, COLD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    nyxb_k_tx<P, NCTX, COLD><<<grid, (P + HW * NCTX) * 32, smem, stream>>>(*S, *Tx, *q, n, state, consts, epoch0, end_epoch, step_io, out_state,
                                                                  out_epoch, out_status, *sink, blob_bytes, off_recK, off_seed, off_sched);
    return cudaGetLastError();
}

// blob layout shared by the host builder, the launcher and the kernel: [recA | recK | colseed | sched]
struct TxBlob { unsigned off_recK, off_seed, off_sched, bytes; };
TxBlob tx_blob(int N, int P, int n_rec, int kmax) {
    TxBlob b;
    unsigned o = (unsigned)(n_rec + 1) * 32u;
    b.off_recK = o; o += (((unsigned)(n_rec + 2) + 1u) & ~1u) * 8u;
    b.off_seed = o; o += (unsigned)(N + 2) * 32u;
    b.off_sched = o; o += (unsigned)P * (2u + 2u * (unsigned)kmax) * 4u;
    b.bytes = (o + 15u) & ~15u;
    return b;
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// host: zigzag column -> position schedule and record table
// ------------------------------------------------------------------------------------------------
void nyxb_tx_build_host(int N, int M, const double* c_nm, const double* s_nm, int P, TxHost& out) {
    const double sqrt2 = std::sqrt(2.0);
    auto C = [&](int n, int m) { return (n <= N && m <= M && m <= n) ? c_nm[(size_t)n * (N + 1) + m] : 0.0; };
    auto Sx = [&](int n, int m) { return (n <= N && m <= M && m <= n) ? s_nm[(size_t)n * (N + 1) + m] : 0.0; };
    auto vr01 = [&](int n, int m) {
        double nf = n, mf = m;
        double v = std::sqrt((nf - mf) * (nf + mf + 1.0));
        return m == 0 ? v / sqrt2 : v;
    };
    auto vr11 = [&](int n, int m) {
        double nf = n, mf = m;
        double v = std::sqrt(((2.0 * nf + 1.0) * (nf + mf + 2.0) * (nf + mf + 1.0)) / (2.0 * nf + 3.0));
        return m == 0 ? v / sqrt2 : v;
    };
    // scale[n][m] = A_ref[n][m] / Q[n][m] (see nyxb_coop.cu: same normalisation algebra, long double)
    auto scale = [&](int n, int m) -> long double {
        long double adiag = 1.0L, dfact = 1.0L;
        for (int k = 1; k <= m; ++k) { adiag *= sqrtl(1.0L + 1.0L / (2.0L * k)); dfact *= (2.0L * k - 1.0L); }
        long double g = adiag / dfact;
        for (int k = m + 1; k <= n; ++k) g *= sqrtl(((2.0L * k + 1.0L) * (k - m)) / ((2.0L * k - 1.0L) * (k + m)));
        for (int k = 2; k <= n - m; ++k) g /= (long double)k;
        return g;
    };
    const int mcols = std::min(M + 1, N + 1);   // columns m = 1..mcols
    // entries n = m..N, padded with null records to an even count (the walk takes two entries per iteration); column N+1 is all
    // null entries (only its seed W term counts)
    auto col_len = [&](int m) { return (std::max(N + 1 - m, 1) + 1) & ~1; };
    std::vector<std::vector<int>> cols(P);
    for (int m = 1; m <= mcols; ++m) {
        const int r = (m - 1) % (2 * P);
        cols[r < P ? r : 2 * P - 1 - r].push_back(m);   // ascending m per position: exponents alternate between the two sequences
    }
    out.P = P;
    out.kmax = 1;
    for (auto& cl : cols) out.kmax = std::max(out.kmax, (int)cl.size());
    out.kmax += 1;   // every schedule row ends with a null column (m = 0, len = 0): the walk prefetches the next column's seeds
    out.n_rec = 0;
    for (int m = 1; m <= mcols; ++m) out.n_rec += col_len(m);
    out.recA.assign((size_t)(out.n_rec + 1) * 4, 0.0);
    out.recK.assign((size_t)(out.n_rec + 2), 0.0);
    out.colseed.assign((size_t)(N + 2) * 4, 0.0);
    out.sched.assign((size_t)P * (2 + 2 * out.kmax), 0);
    for (int m = 1; m <= mcols; ++m) {
        long double dfact = 1.0L;
        for (int k = 1; k <= m; ++k) dfact *= (2.0L * k - 1.0L);
        double* s = &out.colseed[(size_t)m * 4];
        s[0] = (double)dfact;
        if (m >= 2) {   // W term of the first entry (n = m): degree n-1 = m-1 >= 1
            long double f = (long double)sqrt2 * vr11(m - 1, m - 1) * scale(m, m);
            s[1] = (double)(f * C(m - 1, m - 1));
            s[2] = (double)(f * Sx(m - 1, m - 1));
        }
        s[3] = 2.0 * m + 1.0;
    }
    int e = 0;
    for (int w = 0; w < P; ++w) {
        int* sc = &out.sched[(size_t)w * (2 + 2 * out.kmax)];
        sc[0] = e;
        sc[1] = (int)cols[w].size();
        // the kernel alternates between the sequences e = w + 2P j and e = 2P-1-w + 2P j: the columns of a position must come in
        // exactly that order (they do: consecutive m cover every residue; a truncated last period only drops the tail)
        for (size_t k = 0; k < cols[w].size(); ++k) {
            const int m = cols[w][k];
            sc[2 + 2 * k] = m;
            sc[3 + 2 * k] = col_len(m);
            auto kappa = [&](int n) -> double {   // W term of degree n = kappa * (Z term of degree n-1), n > m
                return (double)(((long double)vr11(n - 1, m - 1) * scale(n, m)) / ((long double)vr01(n - 1, m - 1) * scale(n - 1, m)));
            };
            for (int n = m; n < m + col_len(m); ++n, ++e) {
                if (n > N) continue;   // null entry (padding, column N+1)
                const long double sc_ = scale(n, m);
                double* a = &out.recA[(size_t)e * 4];
                a[0] = (double)(sc_ * sqrt2 * (double)m * C(n, m));
                a[1] = (double)(sc_ * sqrt2 * (double)m * Sx(n, m));
                a[2] = (double)(sc_ * sqrt2 * vr01(n, m - 1) * C(n, m - 1));
                a[3] = (double)(sc_ * sqrt2 * vr01(n, m - 1) * Sx(n, m - 1));
                out.recK[e] = kappa(n + 1);   // applied to Q[n+1] (p3, p4) of THIS entry
            }
        }
    }
}

// set contexts per CTA: two sets in flight while both fit beside the table (P = 8: degrees up to ~40), one otherwise
static int tx_contexts(const DevSetup* S, const DevTx* Tx, size_t* smem_bytes) {
    const TxBlob b = tx_blob(S->grav.N, Tx->P, Tx->n_rec, Tx->kmax);
    for (int nctx = (Tx->P <= 10 ? 2 : 1); nctx >= 1; --nctx) {
        const size_t smem = tx_layout(b.bytes, Tx->P, S->grav.N, nctx).total;
        if (smem <= 227 * 1024) { if (smem_bytes) *smem_bytes = smem; return nctx; }
    }
    return 0;
}

// set contexts one SM holds for this setup (one persistent CTA per SM; 0: the tables do not fit) and its dynamic shared memory
extern "C" int nyxb_tx_occupancy(const DevSetup* S, const DevTx* Tx, size_t* smem_bytes) {
    if (Tx->P != 8 && Tx->P != 10 && Tx->P != 16) return 0;
    return tx_contexts(S, Tx, smem_bytes);
}

// `grid` CTAs, each with nyxb_tx_occupancy() set contexts
extern "C" cudaError_t nyxb_launch_tx(const DevSetup* S, const DevTx* Tx, const DevTxQueue* q, size_t n, const double* state,
                                      const double* consts, const long long* epoch0, long long end_epoch, long long* step_io,
                                      double* out_state, long long* out_epoch, int* out_status, const DevSink* sink,
                                      int grid, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const TxBlob b = tx_blob(S->grav.N, Tx->P, Tx->n_rec, Tx->kmax);
    size_t smem = 0;
    const int nctx = tx_contexts(S, Tx, &smem);
    if (nctx < 1 || grid < 1) return cudaErrorInvalidConfiguration;
    const bool cold = tx_cold(*S) || S->grav_body >= 0;
#define NYXB_TX_GO(PP, CC) (cold ? tx_launch_p<PP, CC, true>(S, Tx, q, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_status, sink, grid, smem, b.bytes, b.off_recK, b.off_seed, b.off_sched, stream) \
                             : tx_launch_p<PP, CC, false>(S, Tx, q, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_status, sink, grid, smem, b.bytes, b.off_recK, b.off_seed, b.off_sched, stream))
    if (Tx->P == 8) return nctx == 2 ? NYXB_TX_GO(8, 2) : NYXB_TX_GO(8, 1);
    if (Tx->P == 10) return nctx == 2 ? NYXB_TX_GO(10, 2) : NYXB_TX_GO(10, 1);
    if (Tx->P == 16) return NYXB_TX_GO(16, 1);
    return cudaErrorInvalidValue;
#undef NYXB_TX_GO
}

// host-side view of the blob (nyxb_api.cu uploads it as one allocation; the kernel copies it with one TMA bulk copy)
size_t nyxb_tx_pack_blob(const TxHost* h, int N, unsigned char* dst) {
    const TxBlob b = tx_blob(N, h->P, h->n_rec, h->kmax);
    if (dst) {
        std::memset(dst, 0, b.bytes);
        std::memcpy(dst, h->recA.data(), h->recA.size() * 8);
        std::memcpy(dst + b.off_recK, h->recK.data(), h->recK.size() * 8);
        std::memcpy(dst + b.off_seed, h->colseed.data(), h->colseed.size() * 8);
        std::memcpy(dst + b.off_sched, h->sched.data(), h->sched.size() * 4);
    }
    return b.bytes;
}
