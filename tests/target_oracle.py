"""Restatement of `Targeter::try_achieve_fd` (md/opti/raphson_finite_diff.rs:41-747), impulsive variables only, over the C oracle's
propagation: what `nyxb_target_batch` computes, in plain Python floats in the operation order of nyx_b200/csrc/nyxb_target.h (the LU is
nyxb_inv9's, restated).  `math.acos` / `math.asin` are the host libm's, so the host build of the header agrees bit for bit; the device
agrees up to the ulps of its own acos / asin.

`cfg` is an `abi.TargetConfigC`.  `per_objective=True` propagates the perturbed states once per objective, as the reference does.
"""
from __future__ import annotations

import math

import numpy as np

from nyx_b200 import abi
from oracle import pyoracle

CONTINUE = -1
FRAME_NONE, FRAME_VNC, FRAME_RIC = abi.TGT_FRAME_NONE, abi.TGT_FRAME_VNC, abi.TGT_FRAME_RIC
PI = 3.14159265358979323846
(X, Y, Z, VX, VY, VZ, RMAG, VMAG, SMA, ECC, INC, RAAN, AOP, TA, AOL, TLONG, PERIOD, ENERGY, HMAG, APO, PERI, C3, DECL) = range(23)


def deg(x):
    return x * (180.0 / PI)


def wrap360(a):
    m = math.fmod(a, 360.0)
    if m != 0.0 and m < 0.0:
        m += 360.0
    return 0.0 if m == 0.0 else m


def angle(c, flip):
    cc = -1.0 if c < -1.0 else (1.0 if c > 1.0 else c)
    a = deg(math.acos(cc))
    return 360.0 - a if flip else a


def _div(a, b):
    """IEEE division (Python raises on a zero divisor)"""
    if b == 0.0:
        with np.errstate(all="ignore"):
            return float(np.float64(a) / np.float64(b))
    return a / b


def evaluate(param, rv, mu):
    rv = [float(x) for x in rv]
    if param <= VZ:
        return rv[param]
    r, v = rv[:3], rv[3:]
    rmag = math.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    vmag = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if param == RMAG:
        return rmag
    if param == VMAG:
        return vmag
    with np.errstate(all="ignore"):
        if param == DECL:
            q = _div(r[2], rmag)
            return deg(math.asin(q)) if -1.0 <= q <= 1.0 else math.nan
        energy = 0.5 * vmag * vmag - _div(mu, rmag)
        if param == ENERGY:
            return energy
        sma = _div(-mu, 2.0 * energy)
        if param == SMA:
            return sma
        if param == C3:
            return _div(-mu, sma)
        if param == PERIOD:
            q = _div(sma * sma * sma, mu)
            return 2.0 * PI * math.sqrt(q) if q >= 0.0 else math.nan
        h = [r[1] * v[2] - r[2] * v[1], r[2] * v[0] - r[0] * v[2], r[0] * v[1] - r[1] * v[0]]
        hmag = math.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
        if param == HMAG:
            return hmag
        rdv = r[0] * v[0] + r[1] * v[1] + r[2] * v[2]
        k = vmag * vmag - _div(mu, rmag)
        e = [_div(k * r[i] - rdv * v[i], mu) for i in range(3)]
        ecc = math.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
        if param == ECC:
            return ecc
        if param == APO:
            return sma * (1.0 + ecc)
        if param == PERI:
            return sma * (1.0 - ecc)

        def ang(c, flip):
            return math.nan if math.isnan(c) else angle(c, flip)

        if param == INC:
            return ang(_div(h[2], hmag), False)
        nd = [-h[1], h[0], 0.0]
        nmag = math.sqrt(nd[0] * nd[0] + nd[1] * nd[1] + nd[2] * nd[2])
        raan = ang(_div(nd[0], nmag), nd[1] < 0.0)
        if param == RAAN:
            return raan
        aop = ang(_div(nd[0] * e[0] + nd[1] * e[1] + nd[2] * e[2], nmag * ecc), e[2] < 0.0)
        if param == AOP:
            return aop
        ta = ang(_div(e[0] * r[0] + e[1] * r[1] + e[2] * r[2], ecc * rmag), rdv < 0.0)
        if param == TA:
            return ta
        if param == AOL:
            return wrap360(aop + ta) if math.isfinite(aop + ta) else math.nan
        s = aop + raan + ta
        return wrap360(s) if math.isfinite(s) else math.nan


def dcm(frame, rv):
    """row-major local -> inertial DCM (nyxb_tgt_dcm)"""
    r, v = [float(x) for x in rv[:3]], [float(x) for x in rv[3:6]]
    h = [r[1] * v[2] - r[2] * v[1], r[2] * v[0] - r[0] * v[2], r[0] * v[1] - r[1] * v[0]]
    hm = math.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
    c = [h[i] / hm for i in range(3)]
    a = v if frame == FRAME_VNC else r
    am = math.sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2])
    u = [a[i] / am for i in range(3)]
    cross = lambda p, q: [p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]]
    cols = [u, c, cross(u, c)] if frame == FRAME_VNC else [u, cross(c, u), c]
    return [cols[j][i] for i in range(3) for j in range(3)]


def apply(frame, sc, rv):
    rv = [float(x) for x in rv]
    if frame == FRAME_NONE:
        return [rv[i] + sc[i] for i in range(6)]
    D = dcm(frame, rv)
    dv = [D[i * 3 + 0] * sc[3] + D[i * 3 + 1] * sc[4] + D[i * 3 + 2] * sc[5] for i in range(3)]
    return rv[:3] + [rv[3 + i] + dv[i] for i in range(3)]


def apply_vars(cfg, x, rv):
    sc = [0.0] * 6
    for j in range(cfg.n_vars):
        sc[cfg.vars[j].component] += x[j]
    return apply(cfg.correction_frame, sc, rv)


def perturbed(cfg, j, xi):
    sc = [0.0] * 6
    sc[cfg.vars[j].component] += cfg.vars[j].perturbation
    return apply(cfg.correction_frame, sc, xi)


def inv9(A):
    """nyxb_inv9 (nyx_b200/csrc/nyxb_smooth.h): LU with partial pivoting, row-major 81 list; None on an exactly zero pivot"""
    LU = list(A)
    perm = list(range(9))
    for j in range(9):
        p, best = j, abs(LU[j * 9 + j])
        for r in range(j + 1, 9):
            if abs(LU[r * 9 + j]) > best:
                best, p = abs(LU[r * 9 + j]), r
        if LU[p * 9 + j] == 0.0:
            return None
        if p != j:
            for c in range(9):
                LU[j * 9 + c], LU[p * 9 + c] = LU[p * 9 + c], LU[j * 9 + c]
            perm[j], perm[p] = perm[p], perm[j]
        d = LU[j * 9 + j]
        for r in range(j + 1, 9):
            l = LU[r * 9 + j] / d
            LU[r * 9 + j] = l
            for c in range(j + 1, 9):
                LU[r * 9 + c] -= l * LU[j * 9 + c]
    Ai = [0.0] * 81
    for c in range(9):
        y = [0.0] * 9
        for r in range(9):
            s = 1.0 if perm[r] == c else 0.0
            for k in range(r):
                s -= LU[r * 9 + k] * y[k]
            y[r] = s
        for r in range(8, -1, -1):
            s = y[r]
            for k in range(r + 1, 9):
                s -= LU[r * 9 + k] * Ai[k * 9 + c]
            Ai[r * 9 + c] = s / LU[r * 9 + r]
    return Ai


def pinv(J, O, V):
    """the reference's pseudo-inverse (utils.rs:429-445) as nyxb_tgt_step forms it; J row-major O x V; returns P row-major V x O"""
    m = min(O, V)
    A = [1.0 if e % 10 == 0 else 0.0 for e in range(81)]
    for a in range(m):
        for b in range(m):
            s = 0.0
            if O < V:
                for k in range(V):
                    s += J[a * V + k] * J[b * V + k]
            else:
                for k in range(O):
                    s += J[k * V + a] * J[k * V + b]
            A[a * 9 + b] = s
    Ai = inv9(A)
    if Ai is None:
        return None
    P = [0.0] * (V * O)
    for r in range(V):
        for c in range(O):
            s = 0.0
            if O < V:
                for k in range(O):
                    s += J[k * V + r] * Ai[k * 9 + c]
            else:
                for k in range(V):
                    s += Ai[r * 9 + k] * J[c * V + k]
            P[r * O + c] = s
    return P


def clamp(var, s):
    if abs(s) > abs(var.max_step):
        return abs(var.max_step) * (-1.0 if s < 0.0 else 1.0)
    if s > var.max_value:
        return var.max_value
    if s < var.min_value:
        return var.min_value
    return s


def step(cfg, mu, it, xf, xi, total, prev_norm):
    """nyxb_tgt_step: xf = [(V + 1)][6] final states.  Returns (rc, xi, total, err, prev_norm, jac)"""
    V, O = cfg.n_vars, cfg.n_objs
    err = [math.nan] * O
    ach = [evaluate(cfg.objs[i].parameter, xf[0], mu) for i in range(O)]
    if not all(math.isfinite(a) for a in ach):
        return abi.ERR_TGT_NON_FINITE, xi, total, err, prev_norm, None
    J = [0.0] * (O * V)
    for j in range(V):
        for i in range(O):
            a = evaluate(cfg.objs[i].parameter, xf[j + 1], mu)
            if not math.isfinite(a):
                return abi.ERR_TGT_NON_FINITE, xi, total, err, prev_norm, None
            d = _div(a - ach[i], cfg.vars[j].perturbation)
            if not math.isfinite(d):
                return abi.ERR_TGT_NON_FINITE, xi, total, err, prev_norm, None
            J[i * V + j] = d
    converged = True
    for i in range(O):
        o = cfg.objs[i]
        err[i] = o.multiplicative_factor * (o.desired - ach[i]) + o.additive_factor
        if not abs(err[i]) <= o.tolerance:
            converged = False
    if converged:
        return 0, xi, total, err, prev_norm, J
    nsq = 0.0
    for e in err:
        nsq += e * e
    norm = math.sqrt(nsq)
    if abs(norm - prev_norm) < 1e-10:
        return abi.ERR_TGT_CORRECTION_INEFFECTIVE, xi, total, err, prev_norm, J
    prev_norm = norm
    P = pinv(J, O, V)
    if P is None:
        return abi.ERR_TGT_SINGULAR_JACOBIAN, xi, total, err, prev_norm, J
    delta = []
    for r in range(V):
        s = 0.0
        for c in range(O):
            s += P[r * O + c] * err[c]
        delta.append(clamp(cfg.vars[r], s))
    xi = apply_vars(cfg, delta, xi)
    total = [total[r] + delta[r] for r in range(V)]
    rc = abi.ERR_TGT_TOO_MANY_ITERATIONS if it >= cfg.iterations else CONTINUE
    return rc, xi, total, err, prev_norm, J


def target_batch(dyn_c, opts_c, cfg, state_soa, consts_soa, epoch0_ns, t_c, t_f, per_objective=False, trace=None):
    """Same contract as nyxb_target_batch, on the oracle.  Returns a dict like `Engine.target_batch`, plus "xi" (the iterated states
    [6][n]); `trace` (a list) receives
    (iteration, problem, err, jac) for every evaluation."""
    state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
    consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
    epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
    n = state_soa.shape[1]
    V, O = cfg.n_vars, cfg.n_objs
    mu = dyn_c.mu_central_km3_s2
    pre, pre_ep, _, pre_st = pyoracle.propagate_batch(dyn_c, opts_c, state_soa, consts_soa, epoch0_ns, t_c)
    start = pre.copy()
    total = [[cfg.vars[j].init_guess for j in range(V)] for _ in range(n)]
    err = [[math.nan] * O for _ in range(n)]
    achieved = [list(pre[:6, p]) for p in range(n)]
    iters = [0] * n
    prev = [math.inf] * n
    status = [int(s) for s in pre_st]
    xi = [None] * n
    active = []
    for p in range(n):
        if status[p] & 0xFF:
            continue
        xi[p] = apply_vars(cfg, [cfg.vars[j].init_guess for j in range(V)], pre[:6, p])
        active.append(p)
    reps = O if per_objective else 1
    while active:
        starts = []
        for p in active:
            starts.append(xi[p])
            for _ in range(reps):
                for j in range(V):
                    starts.append(perturbed(cfg, j, xi[p]))
        W = 1 + reps * V
        m = len(starts)
        st = np.empty((9, m))
        cs = np.empty((4, m))
        ep = np.empty(m, dtype=np.int64)
        for a, p in enumerate(active):
            for w in range(W):
                k = a * W + w
                st[:6, k] = starts[k]
                st[6:, k] = start[6:, p]
                cs[:, k] = consts_soa[:, p]
                ep[k] = pre_ep[p]
        out, _, _, ost = pyoracle.propagate_batch(dyn_c, opts_c, st, cs, ep, t_f)
        nxt = []
        for a, p in enumerate(active):
            ks = list(range(a * W, a * W + W))
            warn = status[p]
            fail = 0
            for k in ks:
                warn |= int(ost[k]) & ~0xFF
                if (int(ost[k]) & 0xFF) and not fail:
                    fail = int(ost[k]) & 0xFF
            xf = [list(out[:6, ks[0]])]
            if per_objective:
                # every objective's perturbed runs must give the same final states as the first objective's
                for i in range(1, O):
                    for j in range(V):
                        assert np.array_equal(out[:6, ks[1 + i * V + j]], out[:6, ks[1 + j]]), (p, i, j)
            xf += [list(out[:6, ks[1 + j]]) for j in range(V)]
            achieved[p] = xf[0]
            rc = fail
            if not fail:
                rc, xi[p], total[p], err[p], prev[p], jac = step(cfg, mu, iters[p], xf, xi[p], total[p], prev[p])
                if trace is not None:
                    trace.append((iters[p], p, list(err[p]), jac))
            if rc == CONTINUE:
                status[p] = warn
                iters[p] += 1
                nxt.append(p)
            else:
                status[p] = rc | warn
        active = nxt
    corrected = start.copy()
    ach = start.copy()
    for p in range(n):
        corrected[:6, p] = apply_vars(cfg, total[p], start[:6, p])
        ach[:6, p] = achieved[p]
    xi_out = start[:6].copy()
    for p in range(n):
        if xi[p] is not None:
            xi_out[:, p] = xi[p]
    return {"xi": xi_out, "corrected": corrected, "achieved": ach, "correction": np.array(total).T.reshape(V, n),
            "errors": np.array(err).T.reshape(O, n), "iterations": np.array(iters, dtype=np.int32), "status": np.array(status, dtype=np.int32)}


def config(variables, objectives, frame=FRAME_NONE, iterations=100):
    """abi.TargetConfigC from (component, perturbation, init_guess, max_step, max_value, min_value) and
    (parameter, desired, tolerance[, mult, add]) tuples"""
    c = abi.TargetConfigC()
    c.n_vars, c.n_objs, c.correction_frame, c.iterations = len(variables), len(objectives), frame, iterations
    for j, v in enumerate(variables):
        v = tuple(v) + (1e-4, 0.0, 0.2, 5.0, -5.0)[len(v) - 1:] if len(v) < 6 else v
        c.vars[j].component, c.vars[j].perturbation, c.vars[j].init_guess, c.vars[j].max_step, c.vars[j].max_value, c.vars[j].min_value = v
    for i, o in enumerate(objectives):
        o = tuple(o) + (1.0, 0.0)[len(o) - 3:] if len(o) < 5 else o
        c.objs[i].parameter, c.objs[i].desired, c.objs[i].tolerance, c.objs[i].multiplicative_factor, c.objs[i].additive_factor = o
    return c
