"""TEST INFRASTRUCTURE — numpy restatement of the reference's batch least-squares estimator for ONE problem (never imported by
nyx_b200), on the C oracle's 90-vector `PropInstance` (oracle/nyx_oracle_od.c) and the tracking geometry of oracle/pyoracle_od.py.
It follows, line by line (paths relative to the reference's nyx-core/src):

  BatchLeastSquares::estimate            od/blse/mod.rs:146-446
  BatchLeastSquares::evaluate            od/blse/mod.rs:450-541
  ScalarSensitivity::new (h_tilde)       od/msr/sensitivity.rs:118-239, one type at a time (U1)

nalgebra is not in the tree, so the 9x9 algebra is restated from textbook algorithms, in the order the kernels use: the Cholesky
factor column by column (Golub & Van Loan, Alg. 4.2.2) with forward and back substitution, and the UDU^T factorisation from the last
column to the first (Bierman 1977) with U^-1 by back substitution.  Parity with the reference is by tolerance at that boundary.
Every sum (the STM product, h, the covariance) runs in the kernels' order, left to right, so that the STRICT kernel can be held to
the filter's bound.

The h_tilde rows are the ones `oracle/pyoracle_od.process_arc` builds inline for a measurement window; here they are built for one
type at a time, as the estimator asks (`h_tilde::<U1>`).
"""
import math

import numpy as np

from nyx_b200 import abi
from oracle import pyoracle
from oracle.pyoracle_od import measure, station_state

F64_MAX = np.finfo(np.float64).max
OK, TOO_FEW, SINGULAR, INVALID = 0, abi.ERR_TOO_FEW_MEASUREMENTS, abi.ERR_SINGULAR_INFORMATION, abi.ERR_INVALID_MEASUREMENT


def h_tilde_row(gs, dyn_c, t_ns, y, t, o):
    """The 1x9 h_tilde of type t (sensitivity.rs:145-192): the observed range (range) or range rate (Doppler) in the denominators."""
    r_tx, v_tx, _ = station_state(gs, dyn_c, t_ns)
    dr, dv = y[:3] - r_tx, y[3:6] - v_tx
    H = np.zeros(9)
    if t == abi.MSR_DOPPLER:
        _, (rho, _rr) = measure(gs, dyn_c, t_ns, y)
        rho_dot = o[abi.MSR_DOPPLER]
        H[:3] = dv / rho - rho_dot * dr / rho ** 2
        H[3:6] = dr / rho
    else:
        H[:3] = dr / o[abi.MSR_RANGE]
    return H


def cholesky(A, add):
    """Lower Cholesky factor of A + diag(add), or None when a pivot is not positive."""
    L = np.zeros((9, 9))
    for j in range(9):
        d = A[j, j] + add[j]
        for k in range(j):
            d -= L[j, k] * L[j, k]
        if not d > 0.0:
            return None
        d = math.sqrt(d)
        L[j, j] = d
        for r in range(j + 1, 9):
            s = A[r, j]
            for k in range(j):
                s -= L[r, k] * L[j, k]
            L[r, j] = s / d
    return L


def chol_solve(L, b):
    y = np.zeros(9)
    for r in range(9):
        s = b[r]
        for k in range(r):
            s -= L[r, k] * y[k]
        y[r] = s / L[r, r]
    x = np.zeros(9)
    for r in range(8, -1, -1):
        s = y[r]
        for k in range(r + 1, 9):
            s -= L[k, r] * x[k]
        x[r] = s / L[r, r]
    return x


def udu_inverse(A):
    """A^-1 = U^-T D^-1 U^-1 from A = U D U^T, or None when a d_j is zero (the reference then takes I)."""
    U = np.zeros((9, 9))
    d = np.zeros(9)
    d[8] = A[8, 8]
    if d[8] == 0.0:
        return None
    U[:, 8] = (1.0 / d[8]) * A[:, 8]
    for j in range(7, -1, -1):
        dj = 0.0
        for k in range(j + 1, 9):
            dj += d[k] * (U[j, k] * U[j, k])
        d[j] = A[j, j] - dj
        if d[j] == 0.0:
            return None
        for i in range(j - 1, -1, -1):
            u = 0.0
            for k in range(j + 1, 9):
                u += (d[k] * U[j, k]) * U[i, k]
            U[i, j] = (A[i, j] - u) / d[j]
        U[j, j] = 1.0
    V = np.zeros((9, 9))
    for c in range(9):
        V[c, c] = 1.0
        for r in range(c - 1, -1, -1):
            s = 0.0
            for k in range(r + 1, c + 1):
                s += U[r, k] * V[k, c]
            V[r, c] = -s
    P = np.zeros((9, 9))
    for r in range(9):
        for c in range(9):
            acc = 0.0
            for k in range(min(r, c) + 1):                                # V is upper triangular
                acc += V[k, r] * ((1.0 / d[k]) * V[k, c])
            P[r, c] = acc
    return P


def _matmul(A, B):
    """A @ B with every sum taken left to right (the kernels' order)."""
    out = np.zeros((A.shape[0], B.shape[1]))
    for r in range(A.shape[0]):
        for c in range(B.shape[1]):
            acc = 0.0
            for q in range(A.shape[1]):
                acc += A[r, q] * B[q, c]
            out[r, c] = acc
    return out


class Config:
    """The reference's builder defaults (od/blse/mod.rs:80-135)."""

    def __init__(self, solver=abi.BLS_NORMAL_EQUATIONS, tolerance_pos_km=1e-4, max_iterations=10, max_step_ns=30 * 10**9,
                 epoch_precision_ns=1_000, lm_lambda_init=10.0, lm_lambda_decrease=10.0, lm_lambda_increase=10.0, lm_lambda_min=1e-12,
                 lm_lambda_max=1e12, lm_use_diag_scaling=True):
        self.__dict__.update(locals())
        del self.__dict__["self"]


def _pass(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, x, consts4, t0, with_stm, trace=None):
    """One iteration's walk over the arc: (info, normal, ssq, n_steps, status)."""
    inst = pyoracle.Inst(dyn_c, opts_c, x, consts4, t0)                   # prop.with(current_estimate.with_stm()), no set_step
    info = np.eye(9)                                                      # :186 the identity, not zero
    normal = np.zeros(9)
    ssq = 0.0
    stm_acc = np.eye(9)
    epoch = int(t0)
    for k in range(len(msr_epoch_ns)):
        o = obs[k]
        if np.isnan(o[0]) and np.isnan(o[1]):                             # `rejected`
            continue
        t_k = int(msr_epoch_ns[k])
        while True:
            delta_t = t_k - epoch
            if delta_t <= 0:
                break
            y, ep, step, fixed, _ = inst.get()
            next_step = min(delta_t, step, cfg.max_step_ns)               # :213
            rc = inst.for_duration(next_step)
            if rc:
                return None, None, None, inst, rc
            y, ep, *_ = inst.get()
            epoch = ep
            if trace is not None:
                trace.append((ep, next_step))
            if with_stm:
                stm_acc = _matmul(y[9:].reshape(9, 9).T, stm_acc)        # :220-222 the STM is cumulative: never reset
            if not abs(epoch - t_k) < cfg.epoch_precision_ns:
                continue
            trk = int(msr_tracker[k])
            if trk < 0:                                                   # unknown tracker :226-237
                continue
            gs = stations_c[trk]
            for q in range(gs.n_types):                                   # each type on its own, in the station's order
                t = gs.types[q]
                if np.isnan(o[t]):                                        # not in msr.data
                    continue
                computed, _ = measure(gs, dyn_c, epoch, y)                # measure_instantaneous(state, None): no noise, no bias
                if computed is None:
                    continue
                real = o[t]
                if not math.isfinite(real):
                    return None, None, None, inst, INVALID
                resid = real - computed[t]
                w = 1.0 / gs.noise_var[q]
                if with_stm:
                    h = _matmul(h_tilde_row(gs, dyn_c, epoch, y, t, o)[None, :], stm_acc)[0]
                    info = info + np.outer(h, h) * w
                    normal = normal + (h * resid) * w
                ssq += (w * resid) * resid
    return info, normal, ssq, inst, OK


def count_measurements(obs):
    return int(np.sum(~(np.isnan(obs[:, 0]) & np.isnan(obs[:, 1]))))


def estimate(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns, trace=None):
    """One `estimate(initial_guess, arc)`.  obs: [m][2] (both NaN = measurement absent).  Returns a dict with the fields of
    BLSSolution, the status, the lambda sequence (lambdas[j] = lambda after iteration j + 1) and the step count."""
    n_msr = count_measurements(obs)
    x = np.array(y9[:9], dtype=np.float64)
    res = dict(state=x.copy(), epoch=int(epoch0_ns), covar=np.zeros((9, 9)), iterations=0, final_rms=F64_MAX, final_corr_pos_km=F64_MAX,
               converged=False, status=OK, lambdas=[], rms=[], corrs=[], n_steps=0)
    if n_msr < 2:
        res["status"] = TOO_FEW
        return res
    lm = cfg.solver == abi.BLS_LEVENBERG_MARQUARDT
    lam, cur_rms, corr, cov = cfg.lm_lambda_init, F64_MAX, F64_MAX, np.zeros((9, 9))
    it = 0
    status = OK
    while it < cfg.max_iterations:
        it += 1
        info, normal, ssq, inst, rc = _pass(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, x, consts4, epoch0_ns, True, trace)
        res["n_steps"] += int(inst.get()[4]["n_steps"])
        if rc:
            status = rc
            break
        rms = math.sqrt(ssq / n_msr)
        res["rms"].append(rms)
        if not lm:
            L = cholesky(info, np.zeros(9))
            if L is None:
                status = SINGULAR
                break
            dx = chol_solve(L, normal)
            accept = True
            cur_rms = rms
        else:
            dsq = np.ones(9)
            if cfg.lm_use_diag_scaling:
                for q in range(6):
                    dsq[q] = info[q, q] if info[q, q] > 0.0 else 1e-6
            L = cholesky(info, dsq * lam)
            if L is None:                                                  # :369-377
                lam = min(lam * (cfg.lm_lambda_increase * 10.0), cfg.lm_lambda_max)
                res["lambdas"].append(lam)
                continue
            dx = chol_solve(L, normal)
            if rms < cur_rms:
                accept = True
                lam = max(lam / cfg.lm_lambda_decrease, cfg.lm_lambda_min)
                cur_rms = rms
            else:
                accept = False
                lam = min(lam * cfg.lm_lambda_increase, cfg.lm_lambda_max)
            res["lambdas"].append(lam)
        if not accept:
            corr = F64_MAX
            res["corrs"].append(corr)
            continue
        x = x + dx                                                         # `Spacecraft + OVector<9>`
        x[6] = min(max(x[6], 0.0), 2.0)
        corr = math.sqrt((dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2])
        res["corrs"].append(corr)
        inv = udu_inverse(info)
        cov = np.eye(9) if inv is None else inv
        if corr < cfg.tolerance_pos_km:
            res["converged"] = True
            break
    res.update(state=x, covar=cov, iterations=it, final_rms=cur_rms, final_corr_pos_km=corr, status=status)
    return res


def evaluate(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns):
    """One `evaluate(state, arc)`: (rms, status)."""
    n_msr = count_measurements(obs)
    if n_msr < 1:
        return 0.0, TOO_FEW
    _, _, ssq, _, rc = _pass(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, np.asarray(y9[:9], dtype=np.float64),
                             consts4, epoch0_ns, False)
    if rc:
        return 0.0, rc
    return math.sqrt(ssq / n_msr), OK
