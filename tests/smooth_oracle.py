"""TEST INFRASTRUCTURE — restatement of the reference's estimate stream and smoother for ONE filter (never imported by nyx_b200).

  process_arc   oracle/pyoracle_od.process_arc with an estimate sink: the same loop on the same C oracle `PropInstance`, appending
                one KfEstimate at each point where the reference pushes to ODSolution.estimates (od/process/mod.rs:211-426):
                a time update per chunk that does not land on a measurement (:417-424), and a measurement update per window that
                reaches `measurement_update`, sigma-rejected ones included (:350-381, filtering.rs:186-200).  Nothing is pushed for
                absent measurements, unknown trackers or windows that are not visible (:382-410), and the STM is not reset there.
                With `sink=None` its results are those of oracle/pyoracle_od.process_arc (pinned bit for bit by
                tests/test_oracle_smooth.py); the oracle package itself stays unchanged.
  smooth        ODSolution::smooth (od/process/solution/smooth.rs:104-249) line by line, including its off-by-one residuals.

An estimate is a dict: epoch, tag (-1 or include/nyxb.h NYXB_OD_TAG), nominal[9], deviation[9], covar[9][9], stm[9][9] (Phi since
the previous estimate).  Its residual is looked up through the tag in the filter's per-measurement outputs, as nyxb_od_records does.
"""
from __future__ import annotations

import math

import numpy as np

from nyx_b200 import abi
from oracle import pyoracle
from oracle.pyoracle_od import MSRF_ABSENT, MSRF_NOT_VISIBLE, MSRF_PROCESSED, MSRF_REJECTED, _snc, measure, station_state


def process_arc(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns, covar0, sink=None):
    """oracle/pyoracle_od.process_arc, plus `sink.append(estimate)` at the reference's push points."""
    m = len(msr_epoch_ns)
    inst = pyoracle.Inst(dyn_c, opts_c, y9, consts4, epoch0_ns)            # prop.with(nominal.with_stm()) :167
    y, ep, step, fixed, _ = inst.get()
    if not fixed:
        inst.set_step(cfg.max_step_ns, False)                               # :170-172
    P = np.array(covar0, dtype=np.float64).reshape(9, 9).copy()
    xdev = np.zeros(9)
    prev_epoch = int(epoch0_ns)
    epoch = int(epoch0_ns)
    ratio = np.full((m, 2), np.nan); prefit_o = np.full((m, 2), np.nan); postfit_o = np.full((m, 2), np.nan)
    flags = np.zeros(m, dtype=np.int32)
    est_state = np.full((m, 9), np.nan); est_cov = np.full((m, 9), np.nan)
    status = 0
    ekf = cfg.variant == abi.KF_REFERENCE_UPDATE
    reject = cfg.reject_num_sigmas if cfg.reject_num_sigmas >= 0.0 else None

    def push(tag, y, ep):
        if sink is not None:
            sink.append(dict(epoch=int(ep), tag=int(tag), nominal=np.array(y[:9]), deviation=xdev.copy(), covar=P.copy(),
                             stm=y[9:].reshape(9, 9).T.copy()))

    def reset_stm():
        y, ep, *_ = inst.get()
        y[9:] = np.eye(9).reshape(81)
        inst.set(y, ep)

    def time_update(y, ep):
        nonlocal P, xdev, prev_epoch
        stm = y[9:].reshape(9, 9).T
        P_bar = stm @ P @ stm.T                                              # filtering.rs:61
        q = _snc(cfg, y, ep, prev_epoch, ep - prev_epoch)
        if q is not None:
            P_bar = P_bar + q
        xdev = stm @ xdev if not ekf else np.zeros(9)                        # :81-85
        P = P_bar
        prev_epoch = ep
        return P_bar

    for k in range(m):
        t_k = int(msr_epoch_ns[k])
        o = obs[k]
        if np.isnan(o[0]) and np.isnan(o[1]):
            flags[k] = MSRF_ABSENT
            continue
        while True:
            delta_t = t_k - epoch
            y, ep, step, fixed, _ = inst.get()
            next_step = min(delta_t, step, cfg.max_step_ns)                  # :218
            rc = inst.for_duration(next_step)                                # :232-234
            if rc:
                status = rc
                break
            y, ep, step, fixed, _ = inst.get()
            epoch = ep
            if abs(ep - t_k) < cfg.epoch_precision_ns:                       # :250
                inst.set(y, t_k)                                             # :254 set_epoch
                ep = epoch_for_msr = t_k
                trk = int(msr_tracker[k])
                if trk < 0:                                                  # unknown tracker :400-410
                    break
                gs = stations_c[trk]
                n_types = gs.n_types
                windows = n_types // cfg.msr_size
                for wno in range(windows + 1):                               # :270-398
                    y, ep_now, *_ = inst.get()
                    cur = [gs.types[q] for q in range(wno * cfg.msr_size, min((wno + 1) * cfg.msr_size, n_types))]
                    if not cur:
                        break
                    avail = [not np.isnan(o[t]) for t in cur]
                    if not any(avail):
                        continue
                    M = cfg.msr_size
                    real_obs = np.zeros(M)
                    for i, t in enumerate(cur):
                        if avail[i]:
                            real_obs[i] = o[t]
                    H = np.eye(M, 9)
                    r_tx, v_tx, _up = station_state(gs, dyn_c, epoch_for_msr)
                    dr = y[:3] - r_tx
                    dv = y[3:6] - v_tx
                    computed, (rng_now, _rr) = measure(gs, dyn_c, epoch_for_msr, y)
                    for i, t in enumerate(cur):
                        if not avail[i]:
                            continue
                        if t == abi.MSR_DOPPLER:
                            rho = rng_now
                            rho_dot = o[abi.MSR_DOPPLER]
                            H[i] = [dv[0] / rho - rho_dot * dr[0] / rho ** 2, dv[1] / rho - rho_dot * dr[1] / rho ** 2,
                                    dv[2] / rho - rho_dot * dr[2] / rho ** 2, dr[0] / rho, dr[1] / rho, dr[2] / rho, 0, 0, 0]
                        else:
                            rho = o[abi.MSR_RANGE]
                            H[i] = [dr[0] / rho, dr[1] / rho, dr[2] / rho, 0, 0, 0, 0, 0, 0]
                    Rk = np.zeros((M, M))
                    bias = np.zeros(M)
                    for i, t in enumerate(cur):
                        q = [gs.types[j] for j in range(n_types)].index(t)
                        Rk[i, i] = gs.noise_var[q]
                        bias[i] = gs.bias[q]
                    if computed is None:                                     # :386-392, nothing pushed, no STM reset
                        flags[k] |= MSRF_NOT_VISIBLE
                        continue
                    comp = np.zeros(M)
                    for i, t in enumerate(cur):
                        comp[i] = computed[t]
                    comp = comp - bias
                    stm = y[9:].reshape(9, 9).T
                    P_bar = stm @ P @ stm.T
                    q = _snc(cfg, y, ep_now, prev_epoch, ep_now - prev_epoch)
                    if q is not None:
                        P_bar = P_bar + q
                    PHt = P_bar @ H.T
                    S = H @ PHt + Rk
                    pre = real_obs - comp
                    try:
                        L = np.linalg.cholesky(S)
                    except np.linalg.LinAlgError:
                        L = np.linalg.cholesky(Rk)
                    white = np.linalg.solve(L, pre)
                    rat = math.sqrt(float(white @ white) / M)
                    slot = wno if cfg.msr_size == 1 else 0
                    ratio[k, slot] = rat
                    for i, t in enumerate(cur):
                        prefit_o[k, wno * cfg.msr_size + i] = pre[i]
                    flags[k] |= MSRF_PROCESSED
                    if reject is not None and rat > reject:                  # :169-184
                        time_update(y, ep_now)
                        flags[k] |= MSRF_REJECTED
                        push(abi.od_tag(k, wno, 1, M), y, ep_now)            # the time update made inside measurement_update
                    else:
                        K = np.linalg.solve(S, PHt.T).T
                        if ekf:
                            x_hat = K @ pre
                            post = pre - H @ x_hat
                        else:
                            x_bar = stm @ xdev
                            post = pre - H @ x_bar
                            x_hat = x_bar + K @ post
                        first = np.eye(9) - K @ H
                        cov = first @ P_bar @ first.T + K @ Rk @ K.T
                        P = 0.5 * (cov + cov.T)
                        xdev = x_hat
                        prev_epoch = ep_now
                        for i, t in enumerate(cur):
                            postfit_o[k, wno * cfg.msr_size + i] = post[i]
                        push(abi.od_tag(k, wno, 0, M), y, ep_now)            # the pre-update nominal and x-hat
                        if ekf:
                            ynew = y.copy()
                            ynew[:9] = y[:9] + x_hat
                            ynew[6] = min(max(ynew[6], 0.0), 2.0)
                            inst.set(ynew, ep_now)
                    reset_stm()                                              # :371
                y, ep_now, *_ = inst.get()
                est_state[k] = y[:9]
                est_cov[k] = np.diag(P)
                break
            else:
                time_update(y, ep)                                           # :417-421
                push(abi.OD_TAG_TIME_UPDATE, y, ep)
                reset_stm()
        if status:
            break
    y, ep, step, fixed, det = inst.get()
    return dict(state=y[:9].copy(), epoch=ep, covar=P, state_dev=xdev, resid_ratio=ratio, prefit=prefit_o, postfit=postfit_o,
                msr_flags=flags, est_state=est_state, est_covar_diag=est_cov, n_steps=int(det["n_steps"]), status=status)


def state_of(est):
    """KfEstimate::state(): nominal + deviation, Cr clamped (cosmic/spacecraft.rs:713-728)."""
    v = est["nominal"] + est["deviation"]
    v[6] = min(max(v[6], 0.0), 2.0)
    return v


class SingularSTM(Exception):
    pass


def zero_pivot(A):
    """The singularity rule of the kernel (nyx_b200/csrc/nyxb_smooth.h): Gaussian elimination with partial pivoting (the first largest
    |a_rj| of the column) meets an exactly zero pivot.  nalgebra documents `try_inverse` as None when U has a zero on its diagonal;
    the rule is not pinned against nalgebra itself."""
    U = np.array(A, dtype=np.float64)
    for j in range(9):
        p = j + int(np.argmax(np.abs(U[j:, j])))
        if U[p, j] == 0.0:
            return True
        U[[j, p]] = U[[p, j]]
        for r in range(j + 1, 9):
            l = U[r, j] / U[j, j]
            U[r, j] = l
            U[r, j + 1:] -= l * U[j, j + 1:]
    return False


def residual_of(est, filt, msr_size):
    """The filter's Residual of an estimate (None for a time update): dict of the tag fields and real_obs-free quantities."""
    if est["tag"] < 0:
        return None
    k, w, rej, _ = abi.od_tag_fields(est["tag"])
    slots = [w * msr_size + q for q in range(msr_size)]
    return dict(k=k, w=w, rejected=bool(rej), slots=slots, prefit=filt["prefit"][k, slots].copy(), postfit=filt["postfit"][k, slots].copy(),
                ratio=float(filt["resid_ratio"][k, w if msr_size == 1 else 0]))


def smooth(estimates, filt, msr_size, stations_c, dyn_c, msr_tracker, obs, inv=np.linalg.inv):
    """ODSolution::smooth, smooth.rs:104-249, for one filter: (estimates, residuals, ratios), each a list in estimate order.
    filt: the filter's per-measurement outputs (process_arc's dict), obs: [m][2].  Raises SingularSTM; IndexError / ValueError where
    the reference panics (fewer than two estimates)."""
    residuals = [residual_of(e, filt, msr_size) for e in estimates]
    l = len(estimates) - 1                                                   # :107 (usize: panics on an empty list)
    if l < 0:
        raise IndexError("no estimate")
    sm_est, sm_res, sm_rat = [dict(estimates[-1])], [residuals[-1]], [None]   # :119-127
    while True:
        k = l - len(sm_est)                                                  # :130 (usize: underflow panics when l == 0)
        if k < 0:
            raise ValueError("attempt to subtract with overflow")
        est_kp1 = estimates[k + 1]
        x_kp1_l = est_kp1["deviation"]
        p_kp1_l = est_kp1["covar"]
        est_k = estimates[k]
        if zero_pivot(est_kp1["stm"]):                                       # `try_inverse` -> None
            raise SingularSTM()
        phi_kp1_k = inv(est_kp1["stm"])                                     # :149-154
        x_k_l = phi_kp1_k @ x_kp1_l
        p_k_l = phi_kp1_k @ p_kp1_l @ phi_kp1_k.T
        smoothed_est_k = dict(est_k)
        smoothed_est_k["deviation"] = x_k_l
        smoothed_est_k["covar"] = p_k_l
        res = residuals[k + 1]
        if res is not None:                                                  # :171-210
            mk = res["k"]
            gs = stations_c[int(msr_tracker[mk])]
            y = state_of(smoothed_est_k)
            computed, _ = measure(gs, dyn_c, smoothed_est_k["epoch"], y)
            if computed is not None:
                types = [gs.types[q] for q in res["slots"]]
                o = obs[mk]
                real_obs = np.array([o[t] if not np.isnan(o[t]) else 0.0 for t in types])   # msr/measurement.rs:84-96
                comp = np.array([computed[t] for t in types]) - np.array([gs.bias[q] for q in res["slots"]])
                res = dict(res, postfit=real_obs - comp, computed_obs=comp)
                sm_res.append(res)
            else:
                sm_res.append(None)
        else:
            sm_res.append(None)
        delta_covar = est_k["covar"] - smoothed_est_k["covar"]               # :213-228
        delta_state = state_of(est_k) - state_of(smoothed_est_k)
        with np.errstate(divide="ignore", invalid="ignore"):                 # NaN / +-inf kept, as in the reference
            fs = np.array([dx / np.sqrt(delta_covar[i, i]) if delta_covar[i, i] >= 0.0 else np.nan for i, dx in enumerate(delta_state)])
        sm_est.append(smoothed_est_k)
        sm_rat.append(fs)
        if len(sm_est) == len(estimates):
            break
    return sm_est[::-1], sm_res[::-1], sm_rat[::-1]


def rms(residuals, key):
    """stats.rs:148-173: the sum over the Some residuals, divided by the number of ALL entries."""
    tot = 0.0
    for r in residuals:
        if r is None:
            continue
        v = r[key]
        tot += float(v @ v) if key != "ratio" else v ** 2
    return math.sqrt(tot / len(residuals))
