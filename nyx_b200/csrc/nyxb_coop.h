// nyxb_coop.h — lane-cooperative harmonic tables shared between nyxb_api.cu (owner of the
// device buffers) and nyxb_coop.cu (builder + kernel).
#pragma once
#include <vector>

#include "nyxb_device.cuh"

// Compact records of the FAST cooperative kernel, 40 bytes per lane and entry (n, m), 1 <= m <= N+1, m <= n <= N,
// stored as PAIRS of consecutive entries (a, b) of a column, [pair][piece][lane] in the order each lane walks its columns
// (columns are padded to an even number of entries with null records):
//   pieces 0 / 2 (16 B): p1, p2 = sqrt2 * m * (Cbar, Sbar)[n][m] * scale[n][m]                 -> X, Y sums
//   pieces 1 / 3 (16 B): p3, p4 = sqrt2 * vr01[n][m-1] * (Cbar, Sbar)[n][m-1] * scale[n][m]    -> Z sum
//   piece  4     (16 B): kappa(a), kappa(b); kappa(n) = vr11[n][m-1] scale[n+1][m] / (vr01[n][m-1] scale[n][m])
//                        -> W sum: the term of degree n+1 is kappa(n) * Q[n+1] * (p3, p4)(n)
// The four sums are accumulated per column WITHOUT the column's (cos, sin)((m-1) lambda) factor and folded into the
// totals at the column switch (8 FMAs per column instead of 6 per entry).
// scale[n][m] = A_ref[n][m] / Q[n][m] converts the integer-coefficient recursion
//   Q[n] = (2n-1) u Q[n-1] - (n+m-1)(n-m-1) Q[n-2],  Q[m] = (2m-1)!!
// (whose coefficients are generated in registers, no loads) to the reference's normalised A[n][m].
#define NYXB_COOP_REC_BYTES 40

struct DevCoop {
    int G, L, kmax;
    const double* recs;      // (L+2) * G * 5 doubles (L even)
    const int* col_start;    // [G][kmax] entry index at which the k-th column of the lane starts (L+1: none)
    const int* col_m;        // [G][kmax] order m of that column
    const double* colseed;   // [N+2][4]: (2m-1)!!, pd1, pd2 (W term of the column's first entry), 2m+1
};

struct CoopHost {
    int G = 0, L = 0, kmax = 0;
    std::vector<double> recs;
    std::vector<int> col_start, col_m;
    std::vector<double> colseed;
};

// ---- STRICT cooperative kernel (nyxb_coop_strict.cu): column lists for phase 1, degree lists for phase 2
struct DevCoopStrict {
    int G, kc, kr;
    const int* cols;  // [G][kc+1], -1 terminated, ascending m
    const int* rows;  // [G][kr+1], -1 terminated, ascending n
};
struct CoopStrictHost {
    int G = 0, kc = 0, kr = 0;
    std::vector<int> cols, rows;
};
void nyxb_coop_strict_build_host(int N, int M, int G, CoopStrictHost& out);
// dynamic shared memory of one CTA of the STRICT cooperative kernel at degree N and G lanes per trajectory, and its limit (the
// opt-in maximum per block on sm_90): the per-trajectory triangle grows as N^2 / 2, so 8 lanes fit up to degree 50, 16 up to 75
size_t nyxb_coop_strict_smem(int N, int G);
#define NYXB_COOP_STRICT_SMEM_MAX (227 * 1024)
extern "C" cudaError_t nyxb_launch_coop_strict(const DevSetup* S, const DevCoopStrict* Cs, size_t n, const double* state,
                                               const double* consts, const long long* epoch0, long long end_epoch,
                                               long long* step_io, double* out_state, long long* out_epoch,
                                               nyxb_details* out_details, int* out_status, const DevSink* sink, cudaStream_t stream);

void nyxb_coop_build_host(int N, int M, const double* c_nm, const double* s_nm, int G, CoopHost& out);

// one trajectory per group of Cp->G lanes
extern "C" cudaError_t nyxb_launch_coop(const DevSetup* S, const DevCoop* Cp, size_t n, const double* state,
                                        const double* consts, const long long* epoch0, long long end_epoch,
                                        long long* step_io, double* out_state, long long* out_epoch,
                                        nyxb_details* out_details, int* out_status, const DevSink* sink, cudaStream_t stream);
