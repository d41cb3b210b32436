// nyxb_coop.cu — host side of the lane-cooperative kernel (nyxb_coop_kernel.cuh): column -> lane schedule,
// record table, dispatch on the lane count.  Kernel summary: G lanes of one warp integrate
// one trajectory.  The spherical-harmonic double sum (gravity_field.rs:217-249), which is >98 % of
// the arithmetic for a 21x21 field, is split across the lanes by COLUMNS of the derived-Legendre
// triangle: every A[n][m] is produced by its own column recursion (gravity_field.rs:175-181) in a
// register, and the four partial sums are regrouped so that each A[n][m] is consumed exactly once,
// by the lane that produced it:
//     X += rr_n   m A[n][m] E(n,m)              Y += rr_n m A[n][m] F(n,m)
//     Z += rr_n   vr01[n][m-1] A[n][m] D(n,m-1)  W -= rr_{n-1} vr11[n-1][m-1] A[n][m] D(n-1,m-1)
// (all three of E/F/D use the same (cos,sin)((m-1) lambda) pair, a per-column constant), so there is
// no A matrix in memory, no cross-lane traffic inside the sum, and one butterfly reduction at the end.
// RK stage vectors live in shared memory ([stage][6] per trajectory), lane c < 6 owns state component c;
// the error norm and the step-size controller are evaluated redundantly by every lane of the group
// (identical inputs -> identical decisions, no broadcast).  HBM is touched only to read the initial
// state and write the final one; coefficient records stream from L1/L2 (17.7 KB for 21x21).
//
// Reference behaviour: instance.rs:87-262, 343-352, 358-493 (propagate/single_step/derive) and
// spacecraft.rs:191-310 (eom).  FMA contraction and the regrouped summation make this a
// tolerance-parity path (tests assert < 1e-6 km, the north-star's sub-mm bound).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <functional>
#include <numeric>
#include <set>
#include <string>

#include "nyxb_coop.h"

// ------------------------------------------------------------------------------------------------
// host: column -> lane schedule (longest-processing-time greedy) and record table
// ------------------------------------------------------------------------------------------------

// Aligned column schedule (measured faster on the 21x21 benchmark): keep the bin packing, but reorder
// each lane's columns and insert idle gaps (null records) so that column STARTS of different lane positions fall on the same entries.  The kernel executes its
// column-switch block whenever ANY lane of the warp starts a column, so what costs is the number of DISTINCT start entries, not
// the number of columns (DESIGN.md §11).  Lanes with the fewest columns fix the boundary set first; every other lane searches
// the orders of its columns (multiset permutations) and, before each column, either continues where the previous one ended or
// waits for a boundary that already exists.
static void align_boundaries(int L, const std::function<int(int)>& col_len, std::vector<std::vector<int>>& cols,
                             std::vector<std::vector<int>>& starts, std::vector<int>& load) {
    const int G = (int)cols.size();
    std::set<int> B;
    std::vector<int> lane_order(G);
    std::iota(lane_order.begin(), lane_order.end(), 0);
    std::stable_sort(lane_order.begin(), lane_order.end(), [&](int a, int b) { return cols[a].size() < cols[b].size(); });
    for (int lane : lane_order) {
        std::vector<int> ms = cols[lane];
        const int k = (int)ms.size();
        if (k == 0) continue;
        if (k > 8) { for (int s0 : starts[lane]) if (s0) B.insert(s0); continue; }
        std::vector<int> lens(k);
        for (int i = 0; i < k; ++i) lens[i] = col_len(ms[i]);
        std::sort(lens.begin(), lens.end());
        int best_cost = 1 << 30, best_end = 1 << 30;
        std::vector<int> best_lens, best_starts, cur(k);
        std::function<void(int, int, int)> dfs = [&](int i, int pos, int cost) {
            if (cost > best_cost) return;
            if (i == k) {
                if (cost < best_cost || (cost == best_cost && pos < best_end)) { best_cost = cost; best_end = pos; best_lens = lens; best_starts = cur; }
                return;
            }
            int rem = 0;
            for (int j = i; j < k; ++j) rem += lens[j];
            if (pos + rem > L) return;
            cur[i] = pos;   // contiguous (or entry 0 for the first column)
            dfs(i + 1, pos + lens[i], cost + ((pos != 0 && !B.count(pos)) ? 1 : 0));
            for (int b : B)   // wait for an existing boundary
                if (b > pos && b + rem <= L) { cur[i] = b; dfs(i + 1, b + lens[i], cost); }
        };
        do { dfs(0, 0, 0); } while (std::next_permutation(lens.begin(), lens.end()));
        // hand the columns out per length, ascending m among equals
        std::vector<int> pool = ms;
        std::sort(pool.begin(), pool.end());
        std::vector<int> new_cols(k);
        for (int i = 0; i < k; ++i) {
            auto it = std::find_if(pool.begin(), pool.end(), [&](int m) { return col_len(m) == best_lens[i]; });
            new_cols[i] = *it;
            pool.erase(it);
        }
        cols[lane] = new_cols;
        starts[lane] = best_starts;
        load[lane] = best_starts[k - 1] + best_lens[k - 1];
        for (int s0 : best_starts) if (s0) B.insert(s0);
    }
}

void nyxb_coop_build_host(int N, int M, const double* c_nm, const double* s_nm, int G, CoopHost& out) {
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
    const int mcols = std::min(M + 1, N + 1);  // columns m = 1..mcols
    // entries of column m: n = m..N (the W term of degree n+1 is carried by entry n, so n = N+1 needs no entry of its own);
    // column N+1 keeps one null entry (only its seed W term is non-zero).  Lengths are padded to EVEN: the kernel walks
    // two entries per iteration and tests for a column switch once per pair.
    auto col_len = [&](int m) { int l = std::max(N + 1 - m, 1); return l + (l & 1); };
    // column -> lane schedule: first-fit-decreasing bin packing (every lane walks at most L entries), then the column starts of
    // the lane positions are aligned (align_boundaries)
    std::vector<int> order(mcols);
    std::iota(order.begin(), order.end(), 1);  // already sorted by decreasing length (N + 2 - m)
    std::vector<int> load(G, 0);
    std::vector<std::vector<int>> cols(G);
    std::vector<std::vector<int>> starts(G);
    {
        // first-fit decreasing into G bins of capacity cap, smallest feasible even cap (LPT alone leaves 34 where 32 fits for 21x21)
        int total = 0;
        for (int m : order) total += col_len(m);
        int cap = std::max((total + G - 1) / G, col_len(order[0]));
        cap += cap & 1;
        for (;; cap += 2) {
            std::fill(load.begin(), load.end(), 0);
            for (auto& cl : cols) cl.clear();
            for (auto& st : starts) st.clear();
            bool ok = true;
            for (int m : order) {
                int b = 0;
                while (b < G && load[b] + col_len(m) > cap) ++b;
                if (b == G) { ok = false; break; }
                cols[b].push_back(m);
                starts[b].push_back(load[b]);
                load[b] += col_len(m);
            }
            if (ok) break;
        }
        align_boundaries(cap, col_len, cols, starts, load);
    }
    // Through an idle gap of its lane (null records) a column's recursion keeps running past its last degree, and
    // |Q[n][m]| <= rho^n (n+m)! / (2^m m!) grows without bound: near the surface it overflows once n reaches ~160 (95x95 on 32 lanes
    // idles for 62 entries), and inf x 0 = NaN would enter the sums.  Where that bound passes 1e300 before the lane's next column
    // (or the end of the walk), a stop column m = N + 2 starts at the end of the column: its seed is zero, so Q stays 0.
    const int L = *std::max_element(load.begin(), load.end());
    for (int lane = 0; lane < G; ++lane) {
        std::vector<std::pair<int, int>> sc;
        for (size_t k = 0; k < cols[lane].size(); ++k) sc.push_back({starts[lane][k], cols[lane][k]});
        std::sort(sc.begin(), sc.end());
        std::vector<std::pair<int, int>> with_stops;
        for (size_t k = 0; k < sc.size(); ++k) {
            with_stops.push_back(sc[k]);
            const int m = sc[k].second, end = sc[k].first + col_len(m), next = k + 1 < sc.size() ? sc[k + 1].first : L;
            const int n_top = m + (next - sc[k].first) + 2;   // highest degree the recursion reaches before the next switch
            if (next > end && std::lgamma(n_top + m + 1.0) - m * std::log(2.0) - std::lgamma(m + 1.0) > 300.0 * std::log(10.0))
                with_stops.push_back({end, N + 2});
        }
        cols[lane].clear();
        starts[lane].clear();
        for (auto& p : with_stops) { starts[lane].push_back(p.first); cols[lane].push_back(p.second); }
    }
    out.G = G;
    out.L = *std::max_element(load.begin(), load.end());
    out.kmax = 1;
    for (auto& cl : cols) out.kmax = std::max(out.kmax, (int)cl.size());
    out.recs.assign((size_t)(out.L + 2) * G * 5, 0.0);  // +2: one null pair behind the last one
    out.col_start.assign((size_t)G * out.kmax, out.L + 1);
    out.col_m.assign((size_t)G * out.kmax, 1);
    out.colseed.assign((size_t)(N + 2) * 4, 0.0);

    // scale[n][m] = A_ref[n][m] / Q[n][m]  (long double; both sides are multiples of d^m P_n / du^m):
    //   A_ref[m][m] = a_diag[m] (gravity_field.rs:61-66),  Q[m][m] = (2m-1)!!,
    //   ratio step  gamma_n = gamma_{n-1} * sqrt((2n+1)(n-m) / ((2n-1)(n+m))),  then divide by (n-m)!
    auto scale = [&](int n, int m) -> long double {
        long double adiag = 1.0L, dfact = 1.0L;
        for (int k = 1; k <= m; ++k) { adiag *= sqrtl(1.0L + 1.0L / (2.0L * k)); dfact *= (2.0L * k - 1.0L); }
        long double g = adiag / dfact;
        for (int k = m + 1; k <= n; ++k) g *= sqrtl(((2.0L * k + 1.0L) * (k - m)) / ((2.0L * k - 1.0L) * (k + m)));
        for (int k = 2; k <= n - m; ++k) g /= (long double)k;
        return g;
    };
    for (int m = 1; m <= mcols; ++m) {
        long double dfact = 1.0L;
        for (int k = 1; k <= m; ++k) dfact *= (2.0L * k - 1.0L);
        double* s = &out.colseed[(size_t)m * 4];
        s[0] = (double)dfact;
        if (m >= 2) {  // W term of the first entry (n = m): degree n-1 = m-1 >= 1
            long double f = (long double)sqrt2 * vr11(m - 1, m - 1) * scale(m, m);
            s[1] = (double)(f * C(m - 1, m - 1));
            s[2] = (double)(f * Sx(m - 1, m - 1));
        }
        s[3] = 2.0 * m + 1.0;
    }
    for (int lane = 0; lane < G; ++lane) {
        for (size_t k = 0; k < cols[lane].size(); ++k) {
            int m = cols[lane][k];
            int e = starts[lane][k];
            out.col_start[(size_t)lane * out.kmax + k] = e;
            out.col_m[(size_t)lane * out.kmax + k] = m;
            if (m == N + 2) continue;   // stop column: no records
            auto kappa = [&](int n) -> double {  // W term of degree n = kappa * (Z term of degree n-1), n > m
                return (double)(((long double)vr11(n - 1, m - 1) * scale(n, m)) / ((long double)vr01(n - 1, m - 1) * scale(n - 1, m)));
            };
            for (int n = m; n <= std::max(N, m); ++n, ++e) {
                const long double sc = scale(n, m);
                double p1 = 0, p2 = 0, p3 = 0, p4 = 0, kn = 0.0;
                if (n <= N) {
                    p1 = (double)(sc * sqrt2 * (double)m * C(n, m));
                    p2 = (double)(sc * sqrt2 * (double)m * Sx(n, m));
                    p3 = (double)(sc * sqrt2 * vr01(n, m - 1) * C(n, m - 1));
                    p4 = (double)(sc * sqrt2 * vr01(n, m - 1) * Sx(n, m - 1));
                    kn = kappa(n + 1);  // applied to Q[n+1] p3/p4 of THIS entry
                }
                // device layout: [pair][piece][lane], 16-byte pieces: (p1,p2)a (p3,p4)a (p1,p2)b (p3,p4)b (kappa a, kappa b)
                double* base = out.recs.data() + (size_t)(e / 2) * G * 10;
                const int h = e & 1;
                base[(2 * h) * 2 * G + lane * 2] = p1; base[(2 * h) * 2 * G + lane * 2 + 1] = p2;
                base[(2 * h + 1) * 2 * G + lane * 2] = p3; base[(2 * h + 1) * 2 * G + lane * 2 + 1] = p4;
                base[8 * G + lane * 2 + h] = kn;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// dispatch: one translation unit per lane count (nyxb_coop_g{8,16,32}.cu) so that they build in parallel
// ------------------------------------------------------------------------------------------------
#define NYXB_COOP_DECL(G) \
    cudaError_t nyxb_launch_coop_g##G(const DevSetup*, const DevCoop*, size_t, const double*, const double*, const long long*, \
                                      long long, long long*, double*, long long*, nyxb_details*, int*, const DevSink*, cudaStream_t);
NYXB_COOP_DECL(8)
NYXB_COOP_DECL(16)
NYXB_COOP_DECL(32)

extern "C" cudaError_t nyxb_launch_coop(const DevSetup* S, const DevCoop* Cp, size_t n, const double* state,
                                        const double* consts, const long long* epoch0, long long end_epoch,
                                        long long* step_io, double* out_state, long long* out_epoch,
                                        nyxb_details* out_details, int* out_status, const DevSink* sink, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    switch (Cp->G) {
    case 8: return nyxb_launch_coop_g8(S, Cp, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    case 16: return nyxb_launch_coop_g16(S, Cp, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    case 32: return nyxb_launch_coop_g32(S, Cp, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    default: return cudaErrorInvalidValue;
    }
}
