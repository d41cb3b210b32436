"""GPU batch least squares (`BatchLeastSquares::estimate` / `evaluate`, od/blse/mod.rs:146-541) through `nyxb_od_bls_batch` /
`nyxb_od_bls_evaluate_batch`: parity with the restatement (tests/blse_oracle.py) on every kernel family, per-problem behaviour, and
oracle-free checks.

Branches: iterations, convergence and status must be equal.  The guesses are chosen so that no decision sits near its threshold: the
tolerance is 1e-9 km (never reached in 4 iterations from a dispersed guess) or the guess is the truth (first correction ~1e-12 km).
Values (the as-coded product of cumulative STMs makes the information matrix ill-conditioned, so the state correction carries the
conditioning): STRICT at fixed step |dr| < 1e-6 km, RMS within 1e-8 relative; FAST and adaptive stepping 1e-4 km and 1e-5 relative;
the covariance's 3x3 blocks within 1e-4 (STRICT 1e-6) of the largest entry of each block; the RMS also within 1e-7 absolute (from
the truth it is ~1e-6 of a sigma, the integrator's own error)."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi

from .blse_util import S, blse_scenario, bls, oracle_args

pytestmark = pytest.mark.gpu

FAMILIES = ["thread_strict", "thread_fast", "coop"]


@pytest.fixture(scope="module")
def bo(oracle):
    from . import blse_oracle

    return blse_oracle


def _scenario(oracle, family, stepping, types=(nb.MeasurementType.Range, nb.MeasurementType.Doppler), **kw):
    mode = nb.MODE_STRICT if family == "thread_strict" else nb.MODE_FAST
    sc = blse_scenario(oracle, n_msr=8, cadence_s=10, pos_err_km=0.1, vel_err_km_s=1e-4, degree=12, stepping=stepping, mode=mode,
                       types=types, **kw)
    eng = sc["prop"].engine(sc["frame"], None)
    eng.set_kernel(nb.KERNEL_THREAD if family == "thread_fast" else nb.KERNEL_AUTO)
    sc["eng"], sc["strict"] = eng, mode == nb.MODE_STRICT
    return sc


def _blocks_close(a, b, rtol):
    for rs in (slice(0, 3), slice(3, 6)):
        for cs_ in (slice(0, 3), slice(3, 6)):
            scale = np.abs(b[rs, cs_]).max()
            assert np.abs(a[rs, cs_] - b[rs, cs_]).max() <= rtol * scale, (rs, cs_)


def _check(bo, sc, b, sol, i, exact_tol, guess=None):
    ref = bo.estimate(*oracle_args(sc, b, i, guess))
    assert sol.status[i] == ref["status"]
    assert sol.iterations[i] == ref["iterations"] and bool(sol.converged[i]) == ref["converged"]
    tight = sc["strict"] and exact_tol
    tr, trel = (1e-6, 1e-8) if tight else (1e-4, 1e-5)
    assert np.abs(sol.state_soa[:3, i] - ref["state"][:3]).max() < tr
    assert np.abs(sol.state_soa[3:6, i] - ref["state"][3:6]).max() < tr * 1e-2
    assert sol.epoch_ns[i] == ref["epoch"]
    assert abs(sol.final_rms[i] - ref["final_rms"]) <= trel * ref["final_rms"] + 1e-7   # the RMS from the truth is ~1e-6 sigma
    _blocks_close(sol.covar[i], ref["covar"], 1e-6 if tight else 1e-4)
    return ref


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stepping", ["fixed", "adaptive"])
@pytest.mark.parametrize("solver", [nb.BLSSolver.NormalEquations, nb.BLSSolver.LevenbergMarquardt])
@pytest.mark.parametrize("types", ["range", "doppler", "both"])
def test_estimate_matches_restatement(oracle, bo, family, stepping, solver, types):
    t = {"range": (nb.MeasurementType.Range,), "doppler": (nb.MeasurementType.Doppler,),
         "both": (nb.MeasurementType.Range, nb.MeasurementType.Doppler)}[types]
    sc = _scenario(oracle, family, stepping, types=t)
    b = bls(sc, solver=solver, max_iterations=4, tolerance_pos_km=1e-9)
    guesses = sc["guesses"][:3] + [sc["truth0"]]
    sol = b.estimate_ensemble(guesses, sc["arc"])
    assert sc["eng"].last_kernel() == (abi.KERNEL_COOP if family == "coop" else abi.KERNEL_THREAD)
    for i in range(3):
        _check(bo, sc, b, sol, i, stepping == "fixed")
    _check(bo, sc, b, sol, 3, stepping == "fixed", guess=sc["truth0"])


@pytest.mark.parametrize("family", FAMILIES)
def test_evaluate_matches_restatement(oracle, bo, family):
    sc = _scenario(oracle, family, "fixed")
    b = bls(sc)
    states = sc["guesses"][:3] + [sc["truth0"]]
    rms, status = b.evaluate_ensemble(states, sc["arc"])
    for i in range(4):
        r, st = bo.evaluate(*oracle_args(sc, b, i, states[i]))
        assert status[i] == st == 0
        assert abs(rms[i] - r) <= 1e-9 * r + 1e-7     # from the truth the RMS is ~1e-5 of a sigma
    a = sc["arc"]
    one = nb.TrackingDataArc(a.epoch_ns, a.tracker, a.obs[:, :, :1]).filter_by_offset()   # drops the last measurement
    r, _ = bo.evaluate(*oracle_args(sc, b, 0, states[0], arc=one))
    assert len(one) == len(a) - 1 and abs(b.evaluate(states[0], one) - r) <= 1e-9 * r


def test_per_problem_epochs_absent_measurements_and_errors(oracle, bo):
    sc = _scenario(oracle, "thread_fast", "fixed")
    b = bls(sc, max_iterations=3, tolerance_pos_km=1e-9)
    arc = sc["arc"]
    obs = arc.obs.copy()
    obs[2, :, 1] = np.nan                       # measurement 2 absent from problem 1
    obs[:, :, 2] = np.nan                       # problem 2 has no measurement: TooFewMeasurements
    obs[:7, :, 2] = np.nan
    obs[5, 0, 3] = np.inf                       # problem 3: InvalidMeasurement
    arc2 = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, obs)
    g = list(sc["guesses"])
    g[1] = g[1].with_vector(10 * S, g[1].to_vector())   # problem 1 starts at 10 s: measurement 0 lies at its epoch
    sol = b.estimate_ensemble(g, arc2)
    assert sol.status.tolist() == [0, 0, abi.ERR_TOO_FEW_MEASUREMENTS, abi.ERR_INVALID_MEASUREMENT]
    assert sol.epoch_ns[1] == 10 * S
    for i in (0, 1):
        ref = bo.estimate(*oracle_args(sc, b, i, g[i], arc2))
        assert sol.iterations[i] == ref["iterations"]
        assert np.abs(sol.state_soa[:3, i] - ref["state"][:3]).max() < 1e-4
    with pytest.raises(nb.ODError, match="TooFewMeasurements"):
        sol.solution(2)
    with pytest.raises(nb.ODError, match="InvalidMeasurement"):
        b.estimate(g[3], nb.TrackingDataArc(arc.epoch_ns, arc.tracker, obs[:, :, 3:4]))
    # one problem alone gives the same bits as inside the batch
    alone = b.estimate_ensemble([g[1]], nb.TrackingDataArc(arc.epoch_ns, arc.tracker, obs[:, :, 1:2]))
    assert np.array_equal(alone.state_soa[:, 0], sol.state_soa[:, 1]) and np.array_equal(alone.covar[0], sol.covar[1])
    assert alone.final_rms[0] == sol.final_rms[1]


@pytest.mark.parametrize("solver", [nb.BLSSolver.NormalEquations, nb.BLSSolver.LevenbergMarquardt])
def test_truth_is_a_fixed_point_and_dispersed_guesses_are_recovered(oracle, solver):
    """Oracle-free: noise-free range + Doppler every 10 s for 80 s from a truth propagated with the same dynamics and integrator (RK4,
    10 s: every measurement one step).  The truth is a fixed point whatever the STM product.  From guesses dispersed by about
    1 km / 1 m/s the as-coded estimator does NOT recover the truth: its Jacobian is the product of cumulative STMs, not the
    linearisation, so each iteration removes only part of the error, in proportion to its size (the same ratios at 10 m / 1 cm/s).
    Measured bound after the default 10 iterations: the largest final error below 0.7 of the largest initial one (2.1 and 1.75 km
    for 3.3 km with NE and LM) and the median below 0.6 km (0.53 km)."""
    sc = blse_scenario(oracle, n=16, n_msr=8, cadence_s=10, pos_err_km=1.0, vel_err_km_s=1e-3, stepping="fixed", mode=nb.MODE_FAST,
                       truth_method=nb.IntegratorMethod.RungeKutta4)
    b = bls(sc, solver=solver)
    truth = sc["truth0"].to_vector()
    sol = b.estimate_ensemble([sc["truth0"]] * 16, sc["arc"])
    assert (sol.status == 0).all() and sol.converged.all() and (sol.iterations == 1).all()
    assert np.abs(sol.state_soa[:6] - truth[:6, None]).max() < 1e-9
    sol = b.estimate_ensemble(sc["guesses"], sc["arc"])
    err0 = np.array([np.linalg.norm(g.to_vector()[:3] - truth[:3]) for g in sc["guesses"]])
    err1 = np.linalg.norm(sol.state_soa[:3] - truth[:3, None], axis=0)
    print(solver, "initial", err0.min(), err0.max(), "final", err1.max(), "iterations", sol.iterations.tolist())
    assert (sol.status == 0).all() and err1.max() < 0.7 * err0.max() and np.median(err1) < 0.6


@pytest.mark.parametrize("solver,sample_s,offset_s", [(nb.BLSSolver.NormalEquations, 60, 120), (nb.BLSSolver.LevenbergMarquardt, 10, 600)])
@pytest.mark.parametrize("disperse", [False, True])
def test_reference_blse_robust_large_disp(oracle, solver, sample_s, offset_s, disperse):
    """The reference's `blse_robust_large_disp` (tests/orbit_determination/blse.rs:36-199): 22 000 km orbit from 2020-01-01T04:00 UTC,
    Moon / Sun / Jupiter point masses, the default RK89 propagator, Canberra alone with a 0 deg mask and the default noises, one
    period of noisy tracking at `sample_s`, cut with filter_by_offset(..offset); guesses dispersed in SMA (0.02 km), RAAN and
    inclination (0.02 deg) and eccentricity (2e-4).  Its assertions: the epoch is unchanged, and evaluate(final) <= evaluate(initial)
    when dispersed."""
    from nyx_b200.cosmic import utc_iso_to_epochs

    t0 = int(utc_iso_to_epochs(["2020-01-01T04:00:00"])[0])
    frame = nb.EARTH_J2000
    alm = nb.Almanac.synthetic(frame, t0, 1.0, bodies=(nb.MOON, nb.SUN, nb.JUPITER_BARYCENTER), pad_days=1.0)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.point_masses([nb.MOON, nb.SUN, nb.JUPITER_BARYCENTER]))
    prop = nb.Propagator.default(dyn, mode=nb.MODE_FAST)
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0, 0.01, 30.0, 80.0, 40.0, 170.0, t0, frame))
    canberra = nb.GroundStation.dss34_canberra(0.0, nb.StochasticNoise.default_range_km(), nb.StochasticNoise.default_doppler_km_s())
    devices = {"Canberra": canberra}
    period_s = 2.0 * np.pi * np.sqrt(22000.0 ** 3 / frame.mu_km3_s2())
    epochs = t0 + (np.arange(1, int(period_s // sample_s) + 1) * sample_s * S).astype(np.int64)
    st, cs, ep = nb.pack_spacecraft([truth0])
    packed = dyn.pack(frame, alm)
    topts = nb.IntegratorOptions.with_fixed_step_s(float(sample_s)).to_c(nb.IntegratorMethod.RungeKutta89)
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(packed.c, topts, st, cs, ep, int(epochs[-1]), traj_capacity=len(epochs) + 2)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    truth = t_st[:, idx, 0].T[:, :, None]
    arc = nb.simulate_tracking(epochs, truth, devices, ["Canberra"] * len(epochs), frame, alm, np.random.default_rng(0))
    vis = ~np.isnan(arc.obs[:, 0, 0])
    arc = nb.TrackingDataArc(arc.epoch_ns[vis], [t for t, v in zip(arc.tracker, vis) if v], arc.obs[vis]).filter_by_offset(None, offset_s * S)
    assert len(arc) >= 2
    guess = truth0
    if disperse:
        rng = np.random.default_rng(0)
        o = truth0.orbit
        guess = nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0 + rng.normal(0, 0.02), 0.01 + rng.normal(0, 2e-4), 30.0 + rng.normal(0, 0.02),
                                                       80.0 + rng.normal(0, 0.02), 40.0, 170.0, t0, frame))
    b = nb.BatchLeastSquares(prop, devices, alm, solver=solver)
    initial_rms = b.evaluate(guess, arc)
    sol = b.estimate(guess, arc)
    assert sol.estimated_state.epoch() == truth0.epoch()
    final_rms = b.evaluate(sol.to_kf_estimate().state(), arc)
    print(f"disperse={disperse} msrs={len(arc)} iterations={sol.num_iterations} initial RMS={initial_rms:.4g} final RMS={final_rms:.4g}")
    if disperse:
        assert final_rms <= initial_rms


def test_unsupported_setups(oracle):
    sc = blse_scenario(oracle, n=1, n_msr=4, cadence_s=10)
    drag = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.two_body(), nb.Drag(nb.AtmDensity.Constant(1e-12), nb.IAU_EARTH_FRAME))
    b = nb.BatchLeastSquares(nb.Propagator.default(drag), sc["devices"], None)
    with pytest.raises(nb.PropagationError, match="rc=-4.*PartialsUndefined"):
        b.estimate_ensemble(sc["guesses"], sc["arc"])
    with pytest.raises(nb.PropagationError, match="rc=-4.*PartialsUndefined"):
        b.evaluate_ensemble(sc["guesses"], sc["arc"])


# --------------------------------------------------------------------------- the filter tests' configurations (tests/od_matrix.py)
def _om_case(config, family, degree=21, n_msr=4, bias_km=0.0):
    from . import od_matrix as om

    mode = nb.MODE_STRICT if family == "thread_strict" else nb.MODE_FAST
    prop = om.propagator(config, mode, degree)
    epochs, tr, y0 = om.truth(config, "regular")
    epochs, tr = epochs[:n_msr], tr[:n_msr]
    dev = om.devices(-90.0)
    if bias_km:
        for d in dev.values():
            d.stochastic_noises = {t: nb.StochasticNoise(z.sigma, bias_km) for t, z in d.stochastic_noises.items()}
    names = list(dev)
    schedule = [names[k % 3] for k in range(n_msr)]
    st, cs, ep, _ = om.filters(config)
    n = 4
    obs = nb.simulate_tracking(epochs, np.repeat(tr[:, :, None], n, axis=2), dev, schedule, om.frame(config), om.almanac(config),
                               np.random.default_rng(5)).obs
    tmpl = nb.Spacecraft(orbit=om.truth_orbit(config), mass=nb.Mass(500.0, 20.0, 50.0), srp=nb.SRPData(8.0, 1.3))
    guesses = []
    for i in range(n):
        v = st[:, i].copy()
        v[:6] = y0[:6] + 0.1 * (v[:6] - y0[:6])                   # 30 m / 3 cm/s: inside the STM product's reach
        g = nb.Spacecraft(orbit=tmpl.orbit, mass=nb.Mass(float(cs[0, i]), float(cs[1, i]), float(v[8])), srp=nb.SRPData(float(cs[2, i]), float(v[6])))
        guesses.append(g.with_vector(0, v))
    b = nb.BatchLeastSquares(prop, dev, om.almanac(config), max_iterations=3, tolerance_pos_km=1e-12)
    eng = None
    try:
        eng = prop.engine(om.frame(config), om.almanac(config))
        eng.set_kernel(nb.KERNEL_THREAD if family == "thread_fast" else nb.KERNEL_AUTO)
    except nb.PropagationError:
        pass                                                      # no device: the restatement side still builds
    arc = nb.TrackingDataArc(epochs, schedule, obs)
    packed = prop.dynamics.pack(om.frame(config), om.almanac(config))
    return dict(prop=prop, b=b, eng=eng, arc=arc, guesses=guesses, packed=packed, opts_c=prop.opts.to_c(prop.method), frame=om.frame(config),
                strict=mode == nb.MODE_STRICT)


def _om_oracle(bo, c, i):
    from .blse_util import consts, oracle_cfg

    b, arc, g = c["b"], c["arc"], c["guesses"][i]
    names = list(b.devices)
    st_c = (abi.GroundStationC * len(names))(*[b.devices[k].to_c(c["frame"], b.almanac) for k in names])
    tracker = np.array([names.index(t) for t in arc.tracker], dtype=np.int32)
    return bo.estimate(c["packed"].c, c["opts_c"], oracle_cfg(b), st_c, arc.epoch_ns, tracker, np.ascontiguousarray(arc.obs[:, :, i]),
                       g.to_vector(), consts(g), g.epoch())


def _om_compare(bo, c, sol):
    worst = dict(dr=0.0, dcov=0.0, drms=0.0)
    for i in range(len(c["guesses"])):
        ref = _om_oracle(bo, c, i)
        assert sol.status[i] == ref["status"] == 0
        assert sol.iterations[i] == ref["iterations"] and bool(sol.converged[i]) == ref["converged"]
        if c["strict"]:
            assert sol.details["n_steps"][i] == ref["n_steps"]
        assert sol.state_soa[6, i] == pytest.approx(ref["state"][6], abs=1e-9)
        worst["dr"] = max(worst["dr"], float(np.abs(sol.state_soa[:3, i] - ref["state"][:3]).max()))
        worst["dcov"] = max(worst["dcov"], float(np.abs(sol.covar[i][:6, :6] - ref["covar"][:6, :6]).max() / np.abs(ref["covar"][:6, :6]).max()))
        worst["drms"] = max(worst["drms"], abs(sol.final_rms[i] - ref["final_rms"]) / ref["final_rms"])
    return worst


@pytest.mark.parametrize("config", ["field", "third_body", "srp", "lunar"])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("solver", [nb.BLSSolver.NormalEquations, nb.BLSSolver.LevenbergMarquardt])
def test_od_matrix_configurations(oracle, bo, config, family, solver):
    """The filter tests' four configurations (21x21 field; Moon and Sun point masses; SRP with Cr estimated; lunar orbit tracked from
    Earth stations with the line-of-sight test), the first four measurements of their arc at fixed step, four problems each with
    its own Cr.  STRICT: equal step counts and the filter's bound (1e-9 km, covariance and RMS 1e-9 relative); FAST 1e-7.  The lunar
    case is held to 1e-8 (measured 3e-9 km STRICT): its Earth stations move on the Chebyshev ephemeris, whose velocity the oracle
    evaluates with numpy's series derivative."""
    c = _om_case(config, family)
    c["b"].solver = solver
    sol = c["b"].estimate_ensemble(c["guesses"], c["arc"])
    assert c["eng"].last_kernel() == (abi.KERNEL_COOP if family == "coop" else abi.KERNEL_THREAD)
    w = _om_compare(bo, c, sol)
    print(config, family, solver, w)
    tol = (1e-8 if config == "lunar" else 1e-9) if c["strict"] else 1e-7
    assert w["dr"] < tol and w["dcov"] < tol and w["drms"] < tol


def test_coop_at_70x70(oracle, bo):
    """The warp kernel with the largest Earth slab (70x70)."""
    c = _om_case("field", "coop", degree=70, n_msr=3)
    sol = c["b"].estimate_ensemble(c["guesses"], c["arc"])
    assert c["eng"].last_kernel() == abi.KERNEL_COOP
    w = _om_compare(bo, c, sol)
    print("70x70", w)
    assert w["dr"] < 1e-7 and w["dcov"] < 1e-7 and w["drms"] < 1e-7


@pytest.mark.parametrize("family", FAMILIES)
def test_station_bias_is_not_subtracted(oracle, bo, family):
    """A 50 m range bias on every station: the kernels match the restatement, which compares with the unbiased computed range, and
    the result equals the unbiased stations' bit for bit."""
    c = _om_case("field", family, bias_km=0.05)
    c0 = _om_case("field", family)
    sol = c["b"].estimate_ensemble(c["guesses"], c["arc"])
    sol0 = c0["b"].estimate_ensemble(c0["guesses"], c["arc"])
    w = _om_compare(bo, c, sol)
    assert w["dr"] < (1e-9 if c["strict"] else 1e-7)
    assert np.array_equal(sol.state_soa, sol0.state_soa) and np.array_equal(sol.final_rms, sol0.final_rms)


def test_null_optional_outputs(oracle):
    """Only the status array: the call completes, and its status matches a call with every output."""
    import ctypes as C

    c = _om_case("field", "thread_fast")
    b, arc = c["b"], c["arc"]
    eng, args = b._pack(c["guesses"], arc)
    full = eng.od_bls_batch(*args)
    cfg, nst, st_c, ep_k, trk, obs, st, cs, ep = args
    obs = np.ascontiguousarray(obs); trk = np.ascontiguousarray(trk); st = np.ascontiguousarray(st); cs = np.ascontiguousarray(cs)
    ep = np.ascontiguousarray(ep)
    carc = abi.TrackingArcC(len(ep_k), ep_k.ctypes.data, trk.ctypes.data, obs.ctypes.data)
    status = np.full(len(c["guesses"]), -7, dtype=np.int32)
    out = abi.BlsOutputsC(None, None, None, None, None, None, None, None, status.ctypes.data)
    lib = abi.load_library()
    assert lib.nyxb_od_bls_batch(eng._h, C.byref(cfg), nst, st_c, C.byref(carc), len(status), st.ctypes.data, cs.ctypes.data, ep.ctypes.data,
                                 C.byref(out)) == 0
    assert np.array_equal(status, full["status"])
    rms = np.full(len(status), np.nan); st2 = np.full(len(status), -7, dtype=np.int32)
    assert lib.nyxb_od_bls_evaluate_batch(eng._h, C.byref(cfg), nst, st_c, C.byref(carc), len(status), st.ctypes.data, cs.ctypes.data,
                                          ep.ctypes.data, None, st2.ctypes.data) == 0
    assert (st2 == 0).all()
