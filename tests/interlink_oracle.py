"""TEST INFRASTRUCTURE — restatement of the filter loop (oracle/pyoracle_od.process_arc's structure, on the same C oracle `PropInstance`)
with interlink transmitters (nyxb_interlink_tx), for ONE filter (never imported by nyx_b200).

  window      process/mod.rs:270-352 with InterlinkTxSpacecraft (interlink/trk_device.rs:180-232, interlink/sensitivity.rs:50-172), as
              coded: h_tilde first, with the transmitter at the nominal state's epoch (the measurement epoch), the observed range and
              Doppler in its rows and an error for a Doppler row without an observed range; then the computed observation with the
              transmitter at the propagator's epoch, Vallado's SIGHT against the body at the frame's centre (receiver first), range
              |rho| and range rate rho . v_rx / |rho| (the transmitter's velocity left out), minus the bias.  An epoch outside the
              transmitter's trajectory is an error of the run (the `?` of traj.at), not "not visible".
  loop        the loop of tests/aer_oracle.py at two slots, with the ground station's record tags and ratio slot.
  transmitter nyx_b200.trajectory.Traj.at, the host twin of nyxb_traj_at (tests/test_trajectory.py pins them bit for bit).
"""
from __future__ import annotations

import math

import numpy as np

from nyx_b200 import abi
from nyx_b200.trajectory import TrajError
from oracle import pyoracle
from oracle.pyoracle_od import MSRF_ABSENT, MSRF_NOT_VISIBLE, MSRF_PROCESSED, MSRF_REJECTED, _snc
from tests.position_oracle import SINGULAR, gain, ratio

TX_NO_DATA, NO_RANGE = "tx_no_data", "no_range"
STATUS = {TX_NO_DATA: abi.ERR_TX_NO_DATA, NO_RANGE: abi.ERR_NO_RANGE}


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def tx_state(traj, t_ns):
    """The transmitter's (r, v) at t_ns from its trajectory, or None outside it."""
    try:
        return np.asarray(traj.at(int(t_ns)).orbit.to_cartesian_pos_vel(), dtype=np.float64)
    except TrajError:
        return None


def obstructed(tx, y, radius):
    """Vallado's SIGHT (anise line_of_sight_obstructed) with r1 = receiver, r2 = transmitter (the ground station's order), the body at
    the origin."""
    if not radius > 0.0:
        return False
    r1sq, r2sq, r12 = _dot(y, y), _dot(tx, tx), _dot(y, tx)
    tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12)
    return 0.0 <= tau <= 1.0 and (1.0 - tau) * r1sq + r12 * tau <= radius * radius


def computed(tx, y):
    """measure_instantaneous as coded: (range, range rate) with rho = r_rx - r_tx and rho . v_rx / |rho|."""
    rho = [y[0] - tx[0], y[1] - tx[1], y[2] - tx[2]]
    rng = math.sqrt(_dot(rho, rho))
    return rng, _dot(rho, y[3:6]) / rng


def h_row(t, tx, y, o):
    """interlink/sensitivity.rs:93-150: the row of type t from the OBSERVED range (and Doppler), dr and dv against the transmitter."""
    dr = [y[0] - tx[0], y[1] - tx[1], y[2] - tx[2]]
    dv = [y[3] - tx[3], y[4] - tx[4], y[5] - tx[5]]
    rho = o[abi.MSR_RANGE]
    if t == abi.MSR_DOPPLER:
        rho_dot, rho2 = o[abi.MSR_DOPPLER], rho * rho
        return [dv[0] / rho - rho_dot * dr[0] / rho2, dv[1] / rho - rho_dot * dr[1] / rho2, dv[2] / rho - rho_dot * dr[2] / rho2,
                dr[0] / rho, dr[1] / rho, dr[2] / rho, 0.0, 0.0, 0.0]
    return [dr[0] / rho, dr[1] / rho, dr[2] / rho, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]


def window(dev, traj, M, wno, o, t_nom, t_prop, y):
    """(cur types, avail, real_obs[M], H[M][9], Rk[M], comp[M]) or a string: 'empty' / 'unavailable' / 'not_visible' / TX_NO_DATA /
    NO_RANGE.  dev: abi.InterlinkTxC; traj: its transmitter's trajectory."""
    cur = [dev.types[q] for q in range(wno * M, min((wno + 1) * M, dev.n_types))]
    if not cur:
        return "empty"
    avail = [not np.isnan(o[t]) for t in cur]
    if not any(avail):
        return "unavailable"
    real_obs, Rk, comp, H = np.zeros(M), np.zeros(M), np.zeros(M), np.eye(M, 9)
    tx = tx_state(traj, t_nom)                              # h_tilde: location(tx, rx.epoch).unwrap()
    if tx is None:
        return TX_NO_DATA
    for q, t in enumerate(cur):
        if not avail[q]:
            continue
        if t == abi.MSR_DOPPLER and np.isnan(o[abi.MSR_RANGE]):
            return NO_RANGE
        real_obs[q] = o[t]
        H[q] = h_row(t, tx, y, o)
    tx = tx_state(traj, t_prop)                             # measure: self.traj.at(rx.epoch())?
    if tx is None:
        return TX_NO_DATA
    if obstructed(tx, y, dev.body_radius_km):
        return "not_visible"
    rng, rr = computed(tx, y)
    for q, t in enumerate(cur):
        slot = wno * M + q
        Rk[q] = dev.noise_var[slot]
        comp[q] = (rng if t == abi.MSR_RANGE else rr) - dev.bias[slot]
    return cur, avail, real_obs, H, Rk, comp


def process_arc(dyn_c, opts_c, cfg, devs_c, trajs, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns, covar0, sink=None):
    """One filter over interlink devices (devs_c[s] reads column devs_c[s].tx of `trajs`); obs [m][2].  Returns the outputs of
    nyxb_od_interlink_batch for it ([m][2] residual arrays; the ratio in slot w at msr_size 1, else slot 0)."""
    m = len(msr_epoch_ns)
    inst = pyoracle.Inst(dyn_c, opts_c, y9, consts4, epoch0_ns)
    y, ep, step, fixed, _ = inst.get()
    if not fixed:
        inst.set_step(cfg.max_step_ns, False)
    P = np.array(covar0, dtype=np.float64).reshape(9, 9).copy()
    xdev = np.zeros(9)
    prev_epoch = epoch = int(epoch0_ns)
    rat_o, prefit_o, postfit_o = np.full((m, 2), np.nan), np.full((m, 2), np.nan), np.full((m, 2), np.nan)
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
                if trk < 0 or trk >= len(devs_c):
                    break
                dev = devs_c[trk]
                for wno in range(dev.n_types // M + 1):
                    y, ep_now, *_ = inst.get()
                    w = window(dev, trajs[dev.tx], M, wno, o, t_k, epoch, y)
                    if w == "empty":
                        break
                    if w == "unavailable":
                        continue
                    if isinstance(w, str) and w in STATUS:
                        status = STATUS[w]
                        break
                    if w == "not_visible":
                        flags[k] |= MSRF_NOT_VISIBLE
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
                        push(abi.od_tag(k, wno, 1, M), y, ep_now)
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
                        push(abi.od_tag(k, wno, 0, M), y, ep_now)
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


def smooth_restated(rec, i, devs_c, trajs, M, arc_obs, tracker):
    """ODSolution::smooth (smooth.rs:104-249) of filter i from its records: (status, [(smoothed state, covariance, postfit[2])] for every
    estimate but the last).  The postfit is measure_instantaneous of the smoothed state at record k's epoch, the transmitter at that
    epoch too; NaN when not visible; a record epoch outside the transmitter's trajectory fails the smoothing (ERR_TX_NO_DATA), and then
    every output is NaN."""
    L = int(rec["count"][i])
    out, status = [], 0
    for k in range(L - 1):
        phi = rec["stm"][k + 1, :, i].reshape(9, 9).T
        Pi = np.linalg.inv(phi)
        xs = Pi @ rec["deviation"][k + 1, :, i]
        Ps = Pi @ rec["covar"][k + 1, :, i].reshape(9, 9).T @ Pi.T
        ys = rec["nominal"][k, :, i] + xs
        ys[6] = min(max(ys[6], 0.0), 2.0)
        post = np.full(2, np.nan)
        tg = int(rec["tag"][k + 1, i])
        if tg >= 0:
            mk, w, _, _ = abi.od_tag_fields(tg)
            dev = devs_c[tracker[mk]]
            ek = int(rec["epoch"][k, i])
            win = window(dev, trajs[dev.tx], M, w, arc_obs[mk, :, i], ek, ek, ys)
            if win == TX_NO_DATA:
                status = abi.ERR_TX_NO_DATA
            elif not isinstance(win, str):
                cur, _, real, _, _, comp = win
                for q in range(len(cur)):
                    post[w * M + q] = real[q] - comp[q]
        out.append((ys, Ps, post))
    if status:                                               # the reference has no solution: every output of the filter is NaN
        out = [(np.full(9, np.nan), np.full((9, 9), np.nan), np.full(2, np.nan)) for _ in out]
    return status, out
