// nyxb_smooth.h — the 9x9 part of ODSolution::smooth (od/process/solution/smooth.rs:104-249) as host/device inline functions.
// Used by the smoothing kernel (nyxb_smooth.cu); plain C++ when not compiled by nvcc, so that a CPU test can check the very same
// arithmetic against the numpy restatement (tests/cpp/smooth_core_shim.cpp, tests/test_oracle_smooth.py).  Built without FMA
// contraction on both sides, the host and the device results are bit-identical.
//
// The reference inverts Phi with nalgebra's `lu().try_inverse()`; nalgebra is not in the reference tree.  The inverse here is LU with
// partial pivoting as Golub & Van Loan (Matrix Computations, 4th ed., Alg. 3.4.1, the row-interchange form of Gaussian elimination;
// the first largest |a_rj| of the column is the pivot), followed by one forward and one back substitution per column of the identity.
// "Singular" is an exactly zero pivot, which is what nalgebra documents for `try_inverse` (None when U has a zero on its diagonal).
// That rule and the summation order of the products are not pinned against nalgebra.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define NYXB_SHD __host__ __device__ __forceinline__
#else
#define NYXB_SHD inline
#endif

// Ainv = A^-1 for a row-major 9x9 A.  LU is scratch (81).  False when a pivot is exactly zero (Ainv is then unspecified).
NYXB_SHD bool nyxb_inv9(const double* A, double* LU, double* Ainv) {
    int perm[9];
    for (int e = 0; e < 81; ++e) LU[e] = A[e];
    for (int r = 0; r < 9; ++r) perm[r] = r;
    for (int j = 0; j < 9; ++j) {
        int p = j;
        double best = fabs(LU[j * 9 + j]);
        for (int r = j + 1; r < 9; ++r) {
            const double v = fabs(LU[r * 9 + j]);
            if (v > best) { best = v; p = r; }
        }
        if (LU[p * 9 + j] == 0.0) return false;
        if (p != j) {
            for (int c = 0; c < 9; ++c) { const double t = LU[j * 9 + c]; LU[j * 9 + c] = LU[p * 9 + c]; LU[p * 9 + c] = t; }
            const int t = perm[j]; perm[j] = perm[p]; perm[p] = t;
        }
        const double d = LU[j * 9 + j];
        for (int r = j + 1; r < 9; ++r) {
            const double l = LU[r * 9 + j] / d;
            LU[r * 9 + j] = l;
            for (int c = j + 1; c < 9; ++c) LU[r * 9 + c] -= l * LU[j * 9 + c];
        }
    }
    // column c of the inverse: L y = P e_c, U x = y
    for (int c = 0; c < 9; ++c) {
        double y[9];
        for (int r = 0; r < 9; ++r) {
            double s = (perm[r] == c) ? 1.0 : 0.0;
            for (int k = 0; k < r; ++k) s -= LU[r * 9 + k] * y[k];
            y[r] = s;
        }
        for (int r = 8; r >= 0; --r) {
            double s = y[r];
            for (int k = r + 1; k < 9; ++k) s -= LU[r * 9 + k] * Ainv[k * 9 + c];
            Ainv[r * 9 + c] = s / LU[r * 9 + r];
        }
    }
    return true;
}

// One smoothed estimate from the FILTER estimate k+1, in the reference's order (smooth.rs:154-169): Phi^-1 first, then
// x_s = Phi^-1 x_{k+1} and P_s = (Phi^-1 P_{k+1}) Phi^-T.  Row-major phi, P and outputs; T is scratch (81), Pi receives Phi^-1.
// Ps may be phi itself (phi is read only while it is inverted).  False on a singular Phi (ODError::SingularStateTransitionMatrix).
NYXB_SHD bool nyxb_smooth_core(const double* phi, const double* P, const double* x, double* Pi, double* T, double* Ps, double* xs) {
    if (!nyxb_inv9(phi, T, Pi)) return false;
    for (int r = 0; r < 9; ++r) {
        double s = 0.0;
        for (int k = 0; k < 9; ++k) s += Pi[r * 9 + k] * x[k];
        xs[r] = s;
    }
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) {
            double s = 0.0;
            for (int k = 0; k < 9; ++k) s += Pi[r * 9 + k] * P[k * 9 + c];
            T[r * 9 + c] = s;
        }
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) {
            double s = 0.0;
            for (int k = 0; k < 9; ++k) s += T[r * 9 + k] * Pi[c * 9 + k];
            Ps[r * 9 + c] = s;
        }
    return true;
}

// estimate.state() as a vector: nominal + deviation, Cr clamped to [0, 2] (`Spacecraft + OVector<9>`, cosmic/spacecraft.rs:713-728)
NYXB_SHD void nyxb_est_state(const double* nominal, const double* dev, double* y) {
    for (int r = 0; r < 9; ++r) y[r] = nominal[r] + dev[r];
    y[6] = y[6] < 0.0 ? 0.0 : (y[6] > 2.0 ? 2.0 : y[6]);
}

// Filter-smoother ratios (smooth.rs:217-228): (state_f - state_s)_q / sqrt((P_f - P_s)_qq), on state() vectors; a negative variance
// difference gives NaN and a zero one +-inf or NaN, as in the reference.  Pf_diag, Ps_diag: the two diagonals.
NYXB_SHD void nyxb_fs_ratios(const double* yf, const double* ys, const double* Pf_diag, const double* Ps_diag, double* ratio) {
    for (int q = 0; q < 9; ++q) ratio[q] = (yf[q] - ys[q]) / sqrt(Pf_diag[q] - Ps_diag[q]);
}
