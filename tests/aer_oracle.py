"""TEST INFRASTRUCTURE — restatement of the filter loop (oracle/pyoracle_od.process_arc's structure, on the same C oracle
`PropInstance`) with a ground station that also measures azimuth and elevation (nyxb_aer_station), for ONE filter (never imported by
nyx_b200).

  window      process/mod.rs:270-352 with GroundStation::measure_instantaneous (trk_device.rs:158-208): the ground station's range and
              Doppler, plus azimuth and elevation in degrees (msr/types.rs:102-117) from rho = r_sc - r_station in the integration
              frame; h_tilde rows of msr/sensitivity.rs:118-226 as coded, identity rows for absent types; slot = type value.
  ratio/gain  filtering.rs:152-231 on the leading 2x2 block (tests/position_oracle.ratio / gain at msr_size <= 2).

PARITY UNPINNED: anise's `azimuth_elevation_range_sez_from_location` is not in the tree.  The SEZ frame is restated from its published
definition (Vallado, Fundamentals of Astrodynamics and Applications, RAZEL): S = -N, E and Z = up of the geodetic station, azimuth =
atan2(rho_SEZ.y, -rho_SEZ.x) mapped into [0, 360), elevation = asin(rho_SEZ.z / |rho|).  Here N and E are rotated into the integration
frame with the station's own R^T, as up is, and the dot products are written in the kernels' order.
An estimate sink receives dicts as tests/smooth_oracle.py's, tagged with abi.od_pos_tag.
"""
from __future__ import annotations

import math

import numpy as np

from nyx_b200 import abi
from oracle import pyoracle
from oracle.pyoracle_od import MSRF_ABSENT, MSRF_NOT_VISIBLE, MSRF_PROCESSED, MSRF_REJECTED, _rotation, _snc, station_state
from tests.position_oracle import SINGULAR, gain, ratio

RAD2DEG = 180.0 / 3.14159265358979323846


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def geometry(gs, dyn_c, t_ns, y):
    """(dr, dv, rng, range rate, elevation, azimuth) of the nominal y seen from station gs at t_ns."""
    r_tx, v_tx, up = station_state(gs, dyn_c, t_ns)
    R, _ = _rotation(gs.rot, t_ns)
    north, east = R.T @ np.array(list(gs.north_fixed)), R.T @ np.array(list(gs.east_fixed))
    dr = [y[0] - r_tx[0], y[1] - r_tx[1], y[2] - r_tx[2]]
    dv = [y[3] - v_tx[0], y[4] - v_tx[1], y[5] - v_tx[2]]
    rng = math.sqrt(_dot(dr, dr))
    rr = _dot(dr, dv) / rng
    elev = math.asin(_dot(dr, up) / rng) * RAD2DEG
    az = math.fmod(math.atan2(_dot(dr, east), _dot(dr, north)) * RAD2DEG, 360.0)
    if az < 0.0:
        az += 360.0
    return dict(dr=dr, dv=dv, rng=rng, rr=rr, elev=elev, az=az, r_tx=r_tx)


def visible(gs, g, y):
    """measure_instantaneous's test: the elevation above the mask (the same `elev` value), then Vallado's SIGHT past the body."""
    if g["elev"] - gs.elevation_mask_deg < 0.0:
        return False
    if gs.body != abi.NYXB_CENTRAL_BODY and gs.body_radius_km > 0.0:
        r1, r2 = y[:3], g["r_tx"]
        r1sq, r2sq, r12 = _dot(r1, r1), _dot(r2, r2), _dot(r1, r2)
        tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12)
        if 0.0 <= tau <= 1.0 and (1.0 - tau) * r1sq + r12 * tau <= gs.body_radius_km ** 2:
            return False
    return True


def h_row(t, g, o):
    """msr/sensitivity.rs:118-226 as coded (rad/km for the angles; the observed range / range rate in the denominators)."""
    dr, dv = g["dr"], g["dv"]
    if t == abi.MSR_DOPPLER:
        rho, rho_dot = g["rng"], o[abi.MSR_DOPPLER]
        rho2 = rho * rho
        return [dv[0] / rho - rho_dot * dr[0] / rho2, dv[1] / rho - rho_dot * dr[1] / rho2, dv[2] / rho - rho_dot * dr[2] / rho2,
                dr[0] / rho, dr[1] / rho, dr[2] / rho, 0.0, 0.0, 0.0]
    if t == abi.MSR_RANGE:
        rho = o[abi.MSR_RANGE]
        return [dr[0] / rho, dr[1] / rho, dr[2] / rho, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    xy2 = dr[0] * dr[0] + dr[1] * dr[1]
    if t == abi.MSR_AZIMUTH:
        return [-dr[1] / xy2, dr[0] / xy2, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    nrm = math.sqrt(xy2 + dr[2] * dr[2])
    r2, z2 = nrm * nrm, dr[2] * dr[2]
    return [-(dr[0] * dr[2]) / (r2 * math.sqrt(r2 - z2)), -(dr[1] * dr[2]) / (r2 * math.sqrt(r2 - z2)), math.sqrt(xy2) / r2,
            0.0, 0.0, 0.0, 0.0, 0.0, 0.0]


def computed(t, g):
    return {abi.MSR_RANGE: g["rng"], abi.MSR_DOPPLER: g["rr"], abi.MSR_AZIMUTH: g["az"], abi.MSR_ELEVATION: g["elev"]}[t]


def window(gs, dyn_c, M, wno, o, t_ns, y):
    """(cur types, avail, real_obs[M], H[M][9], Rk[M], comp[M]) or a string: 'empty' / 'unavailable' / 'not_visible'."""
    cur = [gs.types[q] for q in range(wno * M, min((wno + 1) * M, gs.n_types))]
    if not cur:
        return "empty"
    avail = [not np.isnan(o[t]) for t in cur]
    if not any(avail):
        return "unavailable"
    g = geometry(gs, dyn_c, t_ns, y)
    if not visible(gs, g, y):
        return "not_visible"
    real_obs, Rk, comp, H = np.zeros(M), np.zeros(M), np.zeros(M), np.eye(M, 9)
    for q, t in enumerate(cur):
        slot = wno * M + q
        Rk[q] = gs.noise_var[slot]
        comp[q] = computed(t, g) - gs.bias[slot]
        if avail[q]:
            real_obs[q] = o[t]
            H[q] = h_row(t, g, o)
    return cur, avail, real_obs, H, Rk, comp


def process_arc(dyn_c, opts_c, cfg, stations_c, msr_epoch_ns, msr_tracker, obs, y9, consts4, epoch0_ns, covar0, sink=None):
    """One filter over stations with angles; obs [m][4].  Returns the outputs of nyxb_od_aer_batch for it ([m][4] residual arrays;
    the ratio of window w in slot w)."""
    m = len(msr_epoch_ns)
    inst = pyoracle.Inst(dyn_c, opts_c, y9, consts4, epoch0_ns)
    y, ep, step, fixed, _ = inst.get()
    if not fixed:
        inst.set_step(cfg.max_step_ns, False)
    P = np.array(covar0, dtype=np.float64).reshape(9, 9).copy()
    xdev = np.zeros(9)
    prev_epoch = epoch = int(epoch0_ns)
    rat_o, prefit_o, postfit_o = np.full((m, 4), np.nan), np.full((m, 4), np.nan), np.full((m, 4), np.nan)
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
                if trk < 0 or trk >= len(stations_c):
                    break
                gs = stations_c[trk]
                for wno in range(gs.n_types // M + 1):
                    y, ep_now, *_ = inst.get()
                    w = window(gs, dyn_c, M, wno, o, t_k, y)
                    if w == "empty":
                        break
                    if w == "unavailable":
                        continue
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
                    rat_o[k, wno] = rat
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


def smooth_restated(rec, i, stations_c, dyn_c, M, arc_obs, tracker):
    """ODSolution::smooth (smooth.rs:104-249) of filter i from its records: [(smoothed state, covariance, recomputed postfit[4])] for
    every estimate but the last; the postfit goes through the AER window at record k's epoch, NaN when not visible."""
    L = int(rec["count"][i])
    out = []
    for k in range(L - 1):
        phi = rec["stm"][k + 1, :, i].reshape(9, 9).T
        Pi = np.linalg.inv(phi)
        xs = Pi @ rec["deviation"][k + 1, :, i]
        Ps = Pi @ rec["covar"][k + 1, :, i].reshape(9, 9).T @ Pi.T
        ys = rec["nominal"][k, :, i] + xs
        ys[6] = min(max(ys[6], 0.0), 2.0)
        post = np.full(4, np.nan)
        tg = int(rec["tag"][k + 1, i])
        if tg >= 0:
            mk, w, _, _ = abi.od_pos_tag_fields(tg)
            win = window(stations_c[tracker[mk]], dyn_c, M, w, arc_obs[mk, :, i], int(rec["epoch"][k, i]), ys)
            if not isinstance(win, str):
                cur, _, real, _, _, comp = win
                for q in range(len(cur)):
                    post[w * M + q] = real[q] - comp[q]
        out.append((ys, Ps, post))
    return out
