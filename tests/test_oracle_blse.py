"""Batch least squares (`BatchLeastSquares::estimate` / `evaluate`, od/blse/mod.rs:146-541) without a GPU: the restatement
(tests/blse_oracle.py) reproduces the reference's quirks, its cumulative-STM product is pinned against independent oracle
propagations, and the C ABI rejects bad arguments before any device work."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi

from .blse_util import S, blse_scenario, bls, oracle_args


@pytest.fixture(scope="module")
def bo(oracle):
    from . import blse_oracle

    return blse_oracle


@pytest.fixture(scope="module")
def sc(oracle):
    return blse_scenario(oracle, n=2, n_msr=8, cadence_s=10, pos_err_km=0.1, vel_err_km_s=1e-4)


def _with_obs(sc, obs, epochs=None, tracker=None):
    a = sc["arc"]
    return nb.TrackingDataArc(a.epoch_ns if epochs is None else epochs, list(a.tracker if tracker is None else tracker), obs)


def test_cumulative_stm_product_is_pinned(oracle, bo, sc):
    """NE, one iteration, every measurement one 10 s step away: cov^-1 = I + sum W h_i^T h_i with h_i = h_tilde_i Phi(t_i, t0) ...
    Phi(t_1, t0), from independent oracle STM propagations.  The textbook h_i = h_tilde_i Phi(t_i, t0) misses by far more."""
    b = bls(sc, max_iterations=1, tolerance_pos_km=1e-12)
    args = oracle_args(sc, b, 0)
    r = bo.estimate(*args)
    assert r["status"] == 0 and r["iterations"] == 1
    dyn_c, opts_c, _, st_c, ep_k, trk, obs, y9, cs, t0 = args
    g = sc["guesses"][0]
    st, cs_, ep = nb.pack_spacecraft([g])
    info_quirk, info_book = np.eye(9), np.eye(9)
    acc = np.eye(9)
    for k in range(len(ep_k)):
        y, _, stm, _, status = oracle.propagate_batch_stm(dyn_c, opts_c, st, cs_, np.array([t0]), int(ep_k[k]))
        assert status[0] == 0
        Phi = stm[:, 0].reshape(9, 9).T                      # Phi(t_k, t0) from t0 in one propagation
        acc = Phi @ acc
        gs = st_c[int(trk[k])]
        y90 = np.concatenate([y[:, 0], stm[:, 0]])
        for q in range(gs.n_types):
            t = gs.types[q]
            ht = bo.h_tilde_row(gs, dyn_c, int(ep_k[k]), y90, t, obs[k])
            w = 1.0 / gs.noise_var[q]
            info_quirk += np.outer(ht @ acc, ht @ acc) * w
            info_book += np.outer(ht @ Phi, ht @ Phi) * w
    got = np.linalg.inv(r["covar"])
    scale = np.abs(info_quirk).max()
    assert np.abs(got - info_quirk).max() < 1e-6 * scale
    assert np.abs(info_book - info_quirk).max() > 1e3 * 1e-6 * scale


def test_information_starts_at_identity(bo, sc):
    """Cd and mass have no partials, so their rows of h are zero: the identity start is all that their diagonal holds."""
    b = bls(sc, max_iterations=1, tolerance_pos_km=1e-12)
    r = bo.estimate(*oracle_args(sc, b, 0))
    info = np.linalg.inv(r["covar"])
    assert info[7, 7] == pytest.approx(1.0, abs=1e-9) and info[8, 8] == pytest.approx(1.0, abs=1e-9)   # Cd, mass: no partials


def test_measurement_count_includes_skipped_measurements(bo, sc):
    """The RMS denominator counts every present measurement: unknown tracker, invisible and at-or-before-epoch ones included."""
    b = bls(sc)
    a = sc["arc"]
    base, st = bo.evaluate(*oracle_args(sc, b, 0, arc=a))
    assert st == 0
    m = len(a)
    for extra_epoch, extra_trk in ((a.epoch_ns[-1] + 10 * S, "Nowhere"), (0, "Madrid"), (-10 * S, "Madrid")):
        ep = np.concatenate([[extra_epoch], a.epoch_ns]) if extra_epoch <= 0 else np.concatenate([a.epoch_ns, [extra_epoch]])
        tr = (["Madrid"] + list(a.tracker)) if extra_epoch <= 0 else (list(a.tracker) + [extra_trk])
        row = np.full((1, 2, a.n), 1234.5)
        obs = np.concatenate([row, a.obs]) if extra_epoch <= 0 else np.concatenate([a.obs, row])
        rms, st = bo.evaluate(*oracle_args(sc, b, 0, arc=nb.TrackingDataArc(ep, tr, obs)))
        assert st == 0 and rms == pytest.approx(base * math.sqrt(m / (m + 1)), rel=1e-12)
    # invisible: a 90 deg mask hides Canberra's passes; they stay in the count.  The same sum over the visible ones, with Canberra's
    # measurements absent instead, has the smaller count: rms_hidden^2 * m = rms_absent^2 * m_visible
    g = sc["guesses"][0]
    hb = bls(sc)
    hb.devices = {k: dataclasses.replace(d, elevation_mask_deg=90.0 if k == "Canberra" else d.elevation_mask_deg) for k, d in sc["devices"].items()}
    rms_h, st = bo.evaluate(*oracle_args(sc, hb, 0, g, arc=a))
    assert st == 0
    obs = a.obs.copy()
    can = np.array([t == "Canberra" for t in a.tracker])
    obs[can] = np.nan
    rms_a, st = bo.evaluate(*oracle_args(sc, bls(sc), 0, g, arc=_with_obs(sc, obs)))
    m_vis = int((~can).sum())
    assert st == 0 and 0 < m_vis < m and rms_h > 0.0
    assert rms_h == pytest.approx(rms_a * math.sqrt(m_vis / m), rel=1e-12)


def test_no_bias_subtraction(oracle, bo):
    """The station bias does not enter: measure_instantaneous(state, None) has no bias, unlike process_arc, where a 50 m bias on a
    10 m sigma would move every range residual by five sigmas."""
    s0 = blse_scenario(oracle, n=1, n_msr=8, cadence_s=10)
    s1 = blse_scenario(oracle, n=1, n_msr=8, cadence_s=10, bias_km=0.05)
    g = s0["truth0"]
    r0, _ = bo.evaluate(*oracle_args(s0, bls(s0), 0, g))
    r1, _ = bo.evaluate(*oracle_args(s1, bls(s1), 0, g, arc=s0["arc"]))
    assert r0 < 1e-3 and r1 == r0
    e0 = bo.estimate(*oracle_args(s0, bls(s0, max_iterations=2), 0))
    e1 = bo.estimate(*oracle_args(s1, bls(s1, max_iterations=2), 0, s0["guesses"][0], arc=s0["arc"]))
    assert np.array_equal(e0["state"], e1["state"])


def test_each_iteration_restarts_from_init_step(bo, oracle):
    s = blse_scenario(oracle, n=1, n_msr=4, cadence_s=60, stepping="adaptive")
    b = bls(s, max_iterations=2, tolerance_pos_km=1e-12)
    trace = []
    r = bo.estimate(*oracle_args(s, b, 0), trace=trace)
    assert r["iterations"] == 2
    starts = [i for i, (ep, _) in enumerate(trace) if ep == trace[0][0]]
    assert len(starts) == 2 and trace[0][1] == trace[starts[1]][1] == 7 * S    # the first chunk is init_step, not max_step


def test_lm_lambda_sequences(bo, sc):
    b = bls(sc, solver=nb.BLSSolver.LevenbergMarquardt, max_iterations=4, tolerance_pos_km=1e-12)
    r = bo.estimate(*oracle_args(sc, b, 0))
    assert r["lambdas"] == pytest.approx([1.0, 0.1, 0.01, 0.001], rel=1e-15) and r["rms"] == sorted(r["rms"], reverse=True)
    # rejection: a 6-minute arc and an almost undamped first step (lambda0 = 1e-12); from the third iteration on the RMS rises, the
    # step is rejected, lambda grows tenfold and corr_pos is reset
    s = blse_scenario(bo.pyoracle, n=1, n_msr=12, cadence_s=30, pos_err_km=0.1, vel_err_km_s=1e-4)
    b = bls(s, solver=nb.BLSSolver.LevenbergMarquardt, max_iterations=6, tolerance_pos_km=1e-12, lm_lambda_init=1e-12)
    r = bo.estimate(*oracle_args(s, b, 0))
    rejected = [j for j in range(1, len(r["rms"])) if not r["rms"][j] < min(r["rms"][:j])]
    assert rejected, r["rms"]                                                   # the path is taken
    for j in rejected:
        assert r["corrs"][j] == bo.F64_MAX                                      # corr_pos reset after a rejected step
    for j in range(1, len(r["rms"])):
        prev_best = min(r["rms"][:j])
        want = max(r["lambdas"][j - 1] / 10.0, 1e-12) if r["rms"][j] < prev_best else min(r["lambdas"][j - 1] * 10.0, 1e12)
        assert r["lambdas"][j] == pytest.approx(want, rel=1e-15)
    # singular: a huge negative lambda floor makes info + lambda D^2 indefinite; lambda *= increase * 10 and nothing moves
    b = bls(sc, solver=nb.BLSSolver.LevenbergMarquardt, max_iterations=2, lm_lambda_init=-1e9, lm_lambda_max=-1e9)
    r = bo.estimate(*oracle_args(sc, b, 0))
    assert r["iterations"] == 2 and r["lambdas"] == [-1e11, -1e13] and np.array_equal(r["covar"], np.zeros((9, 9))) and r["final_rms"] == bo.F64_MAX


def test_errors_and_zero_iterations(bo, sc):
    b = bls(sc, max_iterations=0)
    r = bo.estimate(*oracle_args(sc, b, 0))
    assert r["status"] == 0 and r["iterations"] == 0 and np.array_equal(r["covar"], np.zeros((9, 9)))
    assert r["final_rms"] == r["final_corr_pos_km"] == bo.F64_MAX and not r["converged"]
    obs = sc["arc"].obs.copy()
    obs[1:, :, 0] = np.nan
    assert bo.estimate(*oracle_args(sc, bls(sc), 0, arc=_with_obs(sc, obs)))["status"] == bo.TOO_FEW
    assert bo.evaluate(*oracle_args(sc, bls(sc), 0, arc=_with_obs(sc, obs)))[1] == 0
    obs = sc["arc"].obs.copy()
    obs[3, 0, 0] = np.inf
    assert bo.estimate(*oracle_args(sc, bls(sc), 0, arc=_with_obs(sc, obs)))["status"] == bo.INVALID
    long = blse_scenario(bo.pyoracle, n=1, n_msr=20, cadence_s=60)
    assert bo.estimate(*oracle_args(long, bls(long), 0))["status"] == bo.SINGULAR   # the STM product overflows the conditioning


def test_from_solution_zeroes_cr_cd_mass_variances(sc):
    cov = np.arange(81, dtype=float).reshape(9, 9) + 1.0
    sol = nb.BLSSolution(sc["truth0"], cov, 3, 1.0, 1e-5, True)
    kf = sol.to_kf_estimate()
    assert kf.covar[6, 6] == kf.covar[7, 7] == kf.covar[8, 8] == 0.0 and kf.covar[6, 7] == cov[6, 7] and kf.covar[0, 0] == cov[0, 0]
    assert kf.nominal_state is sc["truth0"] and np.array_equal(kf.state_deviation, np.zeros(9))


def test_filter_by_offset_bounds():
    ep = np.arange(0, 10, dtype=np.int64) * 60 * S + 5 * S
    arc = nb.TrackingDataArc(ep, ["A"] * 10, np.zeros((10, 2, 1)))
    assert np.array_equal(arc.filter_by_offset().epoch_ns, ep[:-1])               # the open end stands for the last epoch, excluded
    assert np.array_equal(arc.filter_by_offset(120 * S).epoch_ns, ep[2:-1])       # start included
    assert np.array_equal(arc.filter_by_offset(None, 120 * S).epoch_ns, ep[:2])   # end excluded
    assert np.array_equal(arc.filter_by_offset(60 * S, 61 * S).epoch_ns, ep[1:2])
    assert len(arc.filter_by_offset(300 * S, 300 * S)) == 0
    empty = nb.TrackingDataArc(np.zeros(0, dtype=np.int64), [], np.zeros((0, 2, 1)))
    assert len(empty.filter_by_offset(0, S)) == 0


def test_defaults_and_config(sc):
    b = bls(sc)
    c = b.config_c()
    assert (c.solver, c.max_iterations, c.tolerance_pos_km, c.max_step_ns, c.epoch_precision_ns) == (0, 10, 1e-4, 30 * S, 1000)
    assert (c.lm_lambda_init, c.lm_lambda_decrease, c.lm_lambda_increase, c.lm_lambda_min, c.lm_lambda_max, c.lm_use_diag_scaling) == \
        (10.0, 10.0, 10.0, 1e-12, 1e12, 1)
    assert C.sizeof(abi.BlsConfigC) == 80 and C.sizeof(abi.BlsOutputsC) == 72 and abi.BlsConfigC.lm_use_diag_scaling.offset == 72


def test_abi_rejects_null_arguments():
    lib = abi.load_library()
    assert lib.nyxb_od_bls_batch(None, None, 0, None, None, 1, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
    cfg = abi.BlsConfigC()
    cfg.max_step_ns = 30 * S
    assert lib.nyxb_od_bls_batch(None, C.byref(cfg), 0, None, None, 1, None, None, None, None) == -1
    assert lib.nyxb_od_bls_evaluate_batch(None, C.byref(cfg), 0, None, None, 1, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()


def test_abi_rejects_bad_settings_with_engine(sc):
    lib = abi.load_library()
    try:
        eng = sc["prop"].engine(sc["frame"], None)
    except Exception:
        pytest.skip("no engine without a device")
    b = bls(sc)
    names = list(b.devices)
    st_c = (abi.GroundStationC * 2)(*[b.devices[k].to_c(sc["frame"], None) for k in names])
    st, cs, ep = nb.pack_spacecraft(sc["guesses"][:1])
    a = sc["arc"]
    trk = np.zeros(len(a), dtype=np.int32)
    obs = np.ascontiguousarray(a.obs[:, :, :1])
    arc = abi.TrackingArcC(len(a), a.epoch_ns.ctypes.data, trk.ctypes.data, obs.ctypes.data)
    status = np.zeros(1, dtype=np.int32)
    out = abi.BlsOutputsC(None, None, None, None, None, None, None, None, status.ctypes.data)

    def call(cfg, stations=st_c):
        return lib.nyxb_od_bls_batch(eng._h, C.byref(cfg), 2, stations, C.byref(arc), 1, st.ctypes.data, cs.ctypes.data, ep.ctypes.data,
                                     C.byref(out))
    for field, bad, msg in (("max_step_ns", 0, b"max_step"), ("max_iterations", -1, b"max_iterations"), ("solver", 5, b"solver")):
        cfg = b.config_c()
        setattr(cfg, field, bad)
        assert call(cfg) == -1 and msg in lib.nyxb_last_error()
    cfg = b.config_c()
    cfg.solver = abi.BLS_LEVENBERG_MARQUARDT
    cfg.lm_lambda_increase = 0.0
    assert call(cfg) == -1 and b"lambda" in lib.nyxb_last_error()
    cfg.solver = abi.BLS_NORMAL_EQUATIONS                  # the lambda settings are not read by the normal equations
    bad_st = (abi.GroundStationC * 2)(*st_c)
    bad_st[1].noise_var[0] = 0.0
    assert call(cfg, bad_st) == -1 and b"SingularNoiseRk" in lib.nyxb_last_error()
    assert lib.nyxb_od_bls_evaluate_batch(eng._h, C.byref(cfg), 2, st_c, C.byref(arc), 1, st.ctypes.data, cs.ctypes.data, ep.ctypes.data,
                                          None, None) == -1                         # status is required
