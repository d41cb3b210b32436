"""TEST INFRASTRUCTURE — restatement of the filter loop (oracle/pyoracle_od.process_arc's structure, on the same C oracle
`PropInstance`) with a PositionDevice (od/position) in place of the ground station, for ONE filter (never imported by nyx_b200).

  window      process/mod.rs:270-333 with the position device: the computed observation of the type at list position ii is position
              component ii, bias added and subtracted ((r + 0) + b) - b; H has the type's unit row at the TYPE's component; zero rows
              and zero real observations for slots without a type or with an absent type; R keeps the type's variance.
  ratio/gain  filtering.rs:152-231: msr_size <= 2 the ground station's arithmetic (od_ratio / od_sinv); msr_size 3 the Cholesky factor of
              S column by column (fallback: of R), forward substitution for the whitened residual, the Cholesky solve for the gain
              (fallback: the closed-form 3x3 inverse), in the kernels' order.
An estimate sink receives dicts as tests/smooth_oracle.py's, tagged with abi.od_pos_tag.
"""
from __future__ import annotations

import math

import numpy as np

from nyx_b200 import abi
from oracle import pyoracle
from oracle.pyoracle_od import MSRF_ABSENT, MSRF_PROCESSED, MSRF_REJECTED, _snc

SINGULAR = 1   # NYXB_ERR_PROP_MATH, the status of SingularNoiseRk / SingularKalmanGain


def window(dev, M, wno, o, y):
    """(cur types, avail, real_obs[M], H[M][9], Rk[M], comp[M]) or a string: 'empty' / 'unavailable'."""
    cur = [dev.types[q] for q in range(wno * M, min((wno + 1) * M, dev.n_types))]
    if not cur:
        return "empty"
    avail = [not np.isnan(o[t - abi.MSR_X]) for t in cur]
    if not any(avail):
        return "unavailable"
    real_obs, Rk, comp, H = np.zeros(M), np.zeros(M), np.zeros(M), np.zeros((M, 9))
    for q, t in enumerate(cur):
        slot = wno * M + q
        Rk[q] = dev.noise_var[slot]
        comp[q] = ((y[slot] + 0.0) + dev.bias[slot]) - dev.bias[slot]
        if avail[q]:
            real_obs[q] = o[t - abi.MSR_X]
            H[q, t - abi.MSR_X] = 1.0
    return cur, avail, real_obs, H, Rk, comp


def chol3(A):
    """Lower Cholesky factor of a 3x3, or None when a pivot is not positive (kernel order)."""
    L = np.zeros((3, 3))
    if not A[0, 0] > 0.0:
        return None
    L[0, 0] = math.sqrt(A[0, 0])
    L[1, 0] = A[1, 0] / L[0, 0]
    L[2, 0] = A[2, 0] / L[0, 0]
    d1 = A[1, 1] - L[1, 0] * L[1, 0]
    if not d1 > 0.0:
        return None
    L[1, 1] = math.sqrt(d1)
    L[2, 1] = (A[2, 1] - L[2, 0] * L[1, 0]) / L[1, 1]
    d2 = (A[2, 2] - L[2, 0] * L[2, 0]) - L[2, 1] * L[2, 1]
    if not d2 > 0.0:
        return None
    L[2, 2] = math.sqrt(d2)
    return L


def fwd3(L, b):
    y0 = b[0] / L[0, 0]
    t1, t2 = b[1] - y0 * L[1, 0], b[2] - y0 * L[2, 0]
    y1 = t1 / L[1, 1]
    t2 = t2 - y1 * L[2, 1]
    return np.array([y0, y1, t2 / L[2, 2]])


def inv3(S):
    """The closed-form 3x3 inverse, or None when the determinant is 0 or NaN."""
    (m11, m12, m13), (m21, m22, m23), (m31, m32, m33) = S
    c11, c12, c13 = m22 * m33 - m32 * m23, m21 * m33 - m31 * m23, m21 * m32 - m31 * m22
    det = (m11 * c11 - m12 * c12) + m13 * c13
    if det == 0.0 or det != det:
        return None
    return np.array([[c11, m13 * m32 - m33 * m12, m12 * m23 - m22 * m13],
                     [-c12, m11 * m33 - m31 * m13, m13 * m21 - m23 * m11],
                     [c13, m12 * m31 - m32 * m11, m11 * m22 - m21 * m12]]) / det


def ratio(M, S, Rk, pre):
    """Residual ratio, or None on SingularNoiseRk."""
    if M < 3:                                                    # od_ratio
        L00, L10, L11, ok = 1.0, 0.0, 1.0, S[0, 0] > 0.0
        if ok:
            L00 = math.sqrt(S[0, 0])
            if M == 2:
                L10 = S[1, 0] / L00
                d = S[1, 1] - L10 * L10
                if d > 0.0:
                    L11 = math.sqrt(d)
                else:
                    ok = False
        if not ok:
            if not Rk[0] > 0.0 or (M == 2 and not Rk[1] > 0.0):
                return None
            L00, L10, L11 = math.sqrt(Rk[0]), 0.0, math.sqrt(Rk[1]) if M == 2 else 1.0
        w0 = pre[0] / L00
        w1 = (pre[1] - L10 * w0) / L11 if M == 2 else 0.0
        return math.sqrt((w0 * w0 + w1 * w1 if M == 2 else w0 * w0) / M)
    L = chol3(S)
    if L is None:
        if not (Rk > 0.0).all():
            return None
        L = np.diag(np.sqrt(Rk))
    w = fwd3(L, pre)
    return math.sqrt(((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]) / 3.0)


def gain(M, S, PHt):
    """K = P H^T S^-1 as the kernels form it, or None on SingularKalmanGain."""
    if M < 3:
        if M == 1:
            Si = np.array([[1.0 / S[0, 0]]])
        else:
            det = S[0, 0] * S[1, 1] - S[0, 1] * S[1, 0]
            if det == 0.0 or det != det:
                return None
            Si = np.array([[S[1, 1] / det, -S[0, 1] / det], [-S[1, 0] / det, S[0, 0] / det]])
        return PHt @ Si
    L = chol3(S)
    if L is None:
        Si = inv3(S)
        return None if Si is None else PHt @ Si
    K = np.zeros((9, 3))
    for r in range(9):
        y = fwd3(L, PHt[r])
        x2 = y[2] / L[2, 2]
        x1 = (y[1] - L[2, 1] * x2) / L[1, 1]
        x0 = (y[0] - (L[1, 0] * x1 + L[2, 0] * x2)) / L[0, 0]
        K[r] = (x0, x1, x2)
    return K


def process_arc(dyn_c, opts_c, cfg, devices_c, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns, covar0, sink=None):
    """One position-fix filter; obs [m][3].  Returns the outputs of nyxb_od_position_batch for it ([m][3] residual arrays)."""
    m = len(msr_epoch_ns)
    inst = pyoracle.Inst(dyn_c, opts_c, y9, consts4, epoch0_ns)
    y, ep, step, fixed, _ = inst.get()
    if not fixed:
        inst.set_step(cfg.max_step_ns, False)
    P = np.array(covar0, dtype=np.float64).reshape(9, 9).copy()
    xdev = np.zeros(9)
    prev_epoch = epoch = int(epoch0_ns)
    rat_o, prefit_o, postfit_o = np.full((m, 3), np.nan), np.full((m, 3), np.nan), np.full((m, 3), np.nan)
    flags = np.zeros(m, dtype=np.int32)
    est_state = np.full((m, 9), np.nan); est_cov = np.full((m, 9), np.nan)
    status = 0
    ekf = cfg.variant == abi.KF_REFERENCE_UPDATE
    reject = cfg.reject_num_sigmas if cfg.reject_num_sigmas >= 0.0 else None
    M = cfg.msr_size

    def push(tag, y, ep):
        if sink is not None:
            sink.append(dict(epoch=int(ep), tag=int(tag), nominal=np.array(y[:9]), deviation=xdev.copy(), covar=P.copy(),
                             stm=y[9:].reshape(9, 9).T.copy()))

    def reset_stm():
        y, ep, *_ = inst.get()
        y[9:] = np.eye(9).reshape(81)
        inst.set(y, ep)

    def covar_bar(y, ep):
        stm = y[9:].reshape(9, 9).T
        P_bar = stm @ P @ stm.T
        q = _snc(cfg, y, ep, prev_epoch, ep - prev_epoch)
        return P_bar + q if q is not None else P_bar

    def time_update(y, ep):
        nonlocal P, xdev, prev_epoch
        P_bar = covar_bar(y, ep)
        xdev = y[9:].reshape(9, 9).T @ xdev if not ekf else np.zeros(9)
        P = P_bar
        prev_epoch = ep

    for k in range(m):
        t_k = int(msr_epoch_ns[k])
        o = obs[k]
        if np.isnan(o).all():
            flags[k] = MSRF_ABSENT
            continue
        while True:
            y, ep, step, fixed, _ = inst.get()
            rc = inst.for_duration(min(t_k - epoch, step, cfg.max_step_ns))
            if rc:
                status = rc
                break
            y, ep, step, fixed, _ = inst.get()
            epoch = ep
            if abs(ep - t_k) < cfg.epoch_precision_ns:
                inst.set(y, t_k)
                trk = int(msr_tracker[k])
                if trk < 0 or trk >= len(devices_c):
                    break
                dev = devices_c[trk]
                for wno in range(dev.n_types // M + 1):
                    y, ep_now, *_ = inst.get()
                    w = window(dev, M, wno, o, y)
                    if w == "empty":
                        break
                    if w == "unavailable":
                        continue
                    cur, _avail, real_obs, H, Rk, comp = w
                    P_bar = covar_bar(y, ep_now)
                    PHt = P_bar @ H.T
                    S = H @ PHt + np.diag(Rk)
                    pre = real_obs - comp
                    rat = ratio(M, S, Rk, pre)
                    if rat is None:
                        status = SINGULAR                            # SingularNoiseRk
                        break
                    rat_o[k, wno if M == 1 else 0] = rat
                    for q in range(len(cur)):
                        prefit_o[k, wno * M + q] = pre[q]
                    flags[k] |= MSRF_PROCESSED
                    if reject is not None and rat > reject:
                        time_update(y, ep_now)
                        flags[k] |= MSRF_REJECTED
                        push(abi.od_pos_tag(k, wno, 1, M), y, ep_now)
                    else:
                        K = gain(M, S, PHt)
                        if K is None:
                            status = SINGULAR                        # SingularKalmanGain
                            break
                        stm = y[9:].reshape(9, 9).T
                        if ekf:
                            x_hat = K @ pre
                            post = pre - H @ x_hat
                        else:
                            x_bar = stm @ xdev
                            post = pre - H @ x_bar
                            x_hat = x_bar + K @ post
                        first = np.eye(9) - K @ H
                        cov = first @ P_bar @ first.T + K @ np.diag(Rk) @ K.T
                        P = 0.5 * (cov + cov.T)
                        xdev = x_hat
                        prev_epoch = ep_now
                        for q in range(len(cur)):
                            postfit_o[k, wno * M + q] = post[q]
                        push(abi.od_pos_tag(k, wno, 0, M), y, ep_now)
                        if ekf:
                            ynew = y.copy()
                            ynew[:9] = y[:9] + x_hat
                            ynew[6] = min(max(ynew[6], 0.0), 2.0)
                            inst.set(ynew, ep_now)
                    reset_stm()
                y, _, *_ = inst.get()
                est_state[k] = y[:9]
                est_cov[k] = np.diag(P)
                break
            time_update(y, ep)
            push(abi.OD_TAG_TIME_UPDATE, y, ep)
            reset_stm()
        if status:
            break
    y, ep, step, fixed, det = inst.get()
    return dict(state=y[:9].copy(), epoch=ep, covar=P, state_dev=xdev, resid_ratio=rat_o, prefit=prefit_o, postfit=postfit_o,
                flags=flags, est_state=est_state, est_covar_diag=est_cov, n_steps=int(det["n_steps"]), status=status)
