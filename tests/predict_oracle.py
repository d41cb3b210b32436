"""TEST INFRASTRUCTURE — numpy restatement of the reference's covariance mapping for ONE estimate (never imported by nyx_b200),
on the C oracle's 90-vector `PropInstance` (oracle/nyx_oracle_od.c) and the SNC helper of oracle/pyoracle_od.py.  It follows,
line by line (paths relative to the reference's nyx-core/src):

  KalmanODProcess::predict_until         od/process/mod.rs:440-486
  KalmanFilter::time_update              od/kalman/filtering.rs:59-102
  ProcessNoise::propagate                od/snc.rs:175-286

`kf.initialize_process_noises()` is not called by predict_until; it only resets the SNC decay, which the C ABI does not carry.
"""
import numpy as np

from nyx_b200 import abi
from oracle import pyoracle
from oracle.pyoracle_od import _snc


def estimate_state(y9, xdev):
    """KfEstimate::state(): nominal + deviation (`Spacecraft + OVector<9>`, Cr clamped to [0, 2])."""
    v = np.asarray(y9[:9], dtype=np.float64) + xdev
    v[6] = min(max(v[6], 0.0), 2.0)
    return v


def predict_until(dyn_c, opts_c, cfg, y9, consts4, epoch0_ns, covar0, end_epoch_ns, dev0=None):
    """One `predict_until(initial_estimate, end_epoch)`.  Returns the final nominal state / epoch / covariance / deviation, the
    records (state()[K][9], covariance [K][9][9], epochs [K]), the step count and the status of the propagation."""
    if cfg.max_step_ns <= 0:
        raise ValueError("max_step must be positive (the reference would never reach the end epoch)")
    inst = pyoracle.Inst(dyn_c, opts_c, y9, consts4, epoch0_ns)        # prop.with(nominal.with_stm()) :452, no set_step
    P = np.array(covar0, dtype=np.float64).reshape(9, 9).copy()
    xdev = np.zeros(9) if dev0 is None else np.array(dev0, dtype=np.float64)
    ekf = cfg.variant == abi.KF_REFERENCE_UPDATE
    prev_epoch = int(epoch0_ns)
    rec_state = [estimate_state(y9, xdev)]                              # push_time_update(initial_estimate) :448
    rec_cov = [P.copy()]
    rec_ep = [int(epoch0_ns)]
    status = 0
    while True:                                                         # :466-483
        rc = inst.for_duration(cfg.max_step_ns)
        if rc:
            status = rc
            break
        y, ep, *_ = inst.get()
        stm = y[9:].reshape(9, 9).T                                      # column-major tail
        P_bar = stm @ P @ stm.T                                          # filtering.rs:61
        q = _snc(cfg, y, ep, prev_epoch, ep - prev_epoch)
        if q is not None:
            P_bar = P_bar + q
        xdev = stm @ xdev if not ekf else np.zeros(9)                    # :81-85
        P = P_bar
        prev_epoch = ep
        rec_state.append(estimate_state(y, xdev))
        rec_cov.append(P.copy())
        rec_ep.append(ep)
        y[9:] = np.eye(9).reshape(81)                                    # reset_stm
        inst.set(y, ep)
        if ep >= end_epoch_ns:
            break
    y, ep, _, _, det = inst.get()
    return dict(state=y[:9].copy(), epoch=ep, covar=P, state_dev=xdev, rec_state=np.array(rec_state), rec_covar=np.array(rec_cov),
                rec_epoch=np.array(rec_ep, dtype=np.int64), count=len(rec_ep), n_steps=int(det["n_steps"]), status=status)
