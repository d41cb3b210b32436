"""The estimate records of the filter kernels (nyxb_od_ekf_record_batch) and the smoothing kernel (nyxb_od_smooth_batch) against the
restatement (tests/smooth_oracle.py), on the parity matrix's inputs (tests/od_matrix.py).

  - `out` of nyxb_od_ekf_record_batch is bit-identical to nyxb_od_ekf_batch's, on every kernel family;
  - the records equal the oracle's estimate stream in count, tags and epochs, and match its nominal, deviation, covariance and STM;
  - the smoothing kernel fed the ORACLE's records matches the restated smoother to rounding (the kernel alone, free of filter
    differences), and the filter -> smooth chain matches it at the filter's tolerance;
  - per-filter statuses, a filter alone vs. in the batch, NULL optional outputs."""
import copy

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import od_matrix as om
from tests import smooth_oracle as so

pytestmark = pytest.mark.gpu

FAMILIES = ("STRICT", "FAST-thread", "FAST-coop")
# record tolerances: position-like km, velocity-like km/s, covariance at correlation scale, STM relative to its largest entry
TOL = dict(r=1e-7, v=1e-10, covar=1e-8, stm=1e-9)


def engine(family, config, degree=21):
    prop = om.propagator(config, nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST, degree)
    eng = prop.engine(om.frame(config), om.almanac(config))
    eng.set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    return prop, eng


def inputs(config, variant, prop):
    return om.od_inputs(config, variant, "regular", prop)


def oracle_streams(config, variant, filters):
    prop = om.propagator(config, nb.MODE_STRICT)
    odp, cfg, names, st_c, epochs, tracker, obs, st, cs, ep, cov = inputs(config, variant, prop)
    packed = prop.dynamics.pack(om.frame(config), om.almanac(config))
    oc = prop.opts.to_c(prop.method)
    streams, outs = [], []
    for i in filters:
        sink = []
        outs.append(so.process_arc(packed.c, oc, cfg, st_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]), st[:, i].copy(),
                                   cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy(), sink=sink))
        streams.append(sink)
    return streams, outs, packed


_STREAMS = {}


def streams_of(config, variant):
    if (config, variant) not in _STREAMS:
        _STREAMS[(config, variant)] = oracle_streams(config, variant, range(om.N_F))
    return _STREAMS[(config, variant)]


def run_both(family, config, variant, cap=400, degree=21):
    prop, eng = engine(family, config, degree)
    _, cfg, names, st_c, epochs, tracker, obs, st, cs, ep, cov = inputs(config, variant, prop)
    plain = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True)
    k_plain = eng.last_kernel()
    rec = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True, estimates_capacity=cap)
    assert eng.last_kernel() == k_plain == (nb.KERNEL_COOP if family == "FAST-coop" else nb.KERNEL_THREAD)
    return plain, rec, (cfg, names, st_c, tracker, obs, eng)


def assert_same_outputs(a, b):
    for f in ("final_state_soa", "final_epoch_ns", "covar", "state_deviation", "resid_ratio", "prefit", "postfit", "msr_flags", "est_state",
              "est_covar_diag", "status"):
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True), f
    assert np.array_equal(a.details, b.details)


def stack(streams, cap):
    """Oracle streams -> record arrays of nyxb_od_records."""
    n = len(streams)
    rec = {"epoch": np.full((cap, n), -1, dtype=np.int64), "tag": np.full((cap, n), -1, dtype=np.int64), "nominal": np.full((cap, 9, n), np.nan),
           "deviation": np.full((cap, 9, n), np.nan), "covar": np.full((cap, 81, n), np.nan), "stm": np.full((cap, 81, n), np.nan),
           "count": np.array([len(s) for s in streams], dtype=np.int64)}
    for i, s in enumerate(streams):
        for k, e in enumerate(s[:cap]):
            rec["epoch"][k, i], rec["tag"][k, i] = e["epoch"], e["tag"]
            rec["nominal"][k, :, i], rec["deviation"][k, :, i] = e["nominal"], e["deviation"]
            rec["covar"][k, :, i], rec["stm"][k, :, i] = e["covar"].T.reshape(81), e["stm"].T.reshape(81)
    return rec


def assert_records_match(rec, streams, tag):
    assert np.array_equal(rec["count"], [len(s) for s in streams]), tag
    ref = stack(streams, rec["epoch"].shape[0])
    L = int(rec["count"].max())
    assert np.array_equal(rec["tag"][:L], ref["tag"][:L]) and np.array_equal(rec["epoch"][:L], ref["epoch"][:L]), tag
    live = ~np.isnan(ref["nominal"][:L, 0])
    assert np.array_equal(live, ~np.isnan(rec["nominal"][:L, 0])), tag
    # nominal and deviation each on their own (an EKF measurement record holds the PRE-update nominal and x-hat, not their sum)
    err = {}
    for part in ("nominal", "deviation"):
        g, r = rec[part][:L], ref[part][:L]
        err[f"{part}_r"] = float(np.nanmax(np.abs(g[:, :3] - r[:, :3])))
        err[f"{part}_v"] = float(np.nanmax(np.abs(g[:, 3:6] - r[:, 3:6])))
    err["r"], err["v"] = max(err["nominal_r"], err["deviation_r"]), max(err["nominal_v"], err["deviation_v"])
    # an EKF measurement record's deviation is x-hat, so the two parts differ between a correct record and a summed one
    meas = rec["tag"][:L] >= 0
    assert np.array_equal(meas, ref["tag"][:L] >= 0)
    P, Pr = rec["covar"][:L], ref["covar"][:L]
    d = np.sqrt(np.abs(Pr[:, ::10]))                                 # [L][9][n] diagonal
    sc = d[:, :, None, :] * d[:, None, :, :]                          # [L][c][r][n]
    dP = np.abs(P - Pr).reshape(L, 9, 9, -1)
    ok = sc > 0
    err["covar"] = float(np.nanmax(np.where(ok, dP / np.where(ok, sc, 1.0), 0.0)))
    ph, phr = rec["stm"][:L], ref["stm"][:L]
    err["stm"] = float(np.nanmax(np.abs(ph - phr) / np.nanmax(np.abs(phr), axis=1, keepdims=True)))
    print(f"SMOOTH-REC {tag} " + " ".join(f"{k}={v:.2g}" for k, v in err.items()))
    assert all(err[k] <= TOL[k] for k in TOL), (tag, err)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("config", ("field", "third_body", "srp", "lunar"))
def test_records_match_the_oracle_stream_ekf(family, config):
    plain, rec, _ = run_both(family, config, "ekf")
    assert_same_outputs(plain, rec)
    assert_records_match(rec.records, streams_of(config, "ekf")[0], f"{family}/{config}/ekf")


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("variant", ("ekf_scalar_noreject", "ckf_reject", "ckf_scalar"))
def test_records_match_the_oracle_stream_variants(family, variant):
    plain, rec, _ = run_both(family, "field", variant)
    assert_same_outputs(plain, rec)
    assert_records_match(rec.records, streams_of("field", variant)[0], f"{family}/field/{variant}")


def test_warp_kernel_records_at_70x70():
    prop, eng = engine("FAST-coop", "field", 70)
    _, cfg, names, st_c, epochs, tracker, obs, st, cs, ep, cov = inputs("field", "ekf", prop)
    plain = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True)
    rec = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True, estimates_capacity=300)
    assert eng.last_kernel() == nb.KERNEL_COOP
    assert_same_outputs(plain, rec)
    sprop = om.propagator("field", nb.MODE_STRICT, 70)
    sodp, scfg, _, sst_c, *_ = inputs("field", "ekf", sprop)
    packed = sprop.dynamics.pack(om.frame("field"), om.almanac("field"))
    streams = []
    for i in range(om.N_F):
        sink = []
        so.process_arc(packed.c, sprop.opts.to_c(sprop.method), scfg, sst_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]), st[:, i].copy(),
                       cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy(), sink=sink)
        streams.append(sink)
    assert_records_match(rec.records, streams, "FAST-coop/field70/ekf")


def restated(streams, outs, packed, config, variant, st_c, tracker, obs):
    M = om.VARIANTS[variant][1]
    return [so.smooth(s, o, M, st_c, packed.c, tracker, np.ascontiguousarray(obs[:, :, i])) for i, (s, o) in enumerate(zip(streams, outs))]


def compare_smoothed(r, ref, rec, tol_rel, tag):
    """r: nyxb_od_smooth_batch dict; ref: restated (estimates, residuals, ratios) per filter."""
    worst = {}
    for i, (est, res, rat) in enumerate(ref):
        L = len(est)
        for k in range(L):
            y = so.state_of(est[k])
            for name, got, want in (("state", r["state"][k, :, i], y), ("dev", r["deviation"][k, :, i], est[k]["deviation"]),
                                    ("covar", r["covar"][k, :, i], est[k]["covar"].T.reshape(81))):
                if name == "state":           # relative to the largest position / velocity component
                    got, want = got[:6], want[:6]
                scale = np.abs(want).max()
                e = float(np.abs(got - want).max() / (scale if scale > 0 else 1.0))
                worst[name] = max(worst.get(name, 0.0), e)
            if rat[k] is None:
                assert np.isnan(r["fs_ratio"][k, :, i]).all(), (tag, i, k)
            else:
                # the NaN pattern where the variance difference is clear of rounding (a zero difference, e.g. behind an identity STM,
                # takes either sign); the values where both are finite
                pf = np.diag(rec["covar"][k, :, i].reshape(9, 9).T)
                dpf = pf - np.diag(est[k]["covar"])
                clear = np.abs(dpf) > 1e-9 * np.abs(pf)
                got = r["fs_ratio"][k, :, i]
                assert np.array_equal(np.isnan(got[clear]), np.isnan(rat[k][clear])), (tag, i, k)
                both = clear & np.isfinite(got) & np.isfinite(rat[k])
                if both.any():
                    worst["ratio"] = max(worst.get("ratio", 0.0), float((np.abs(got[both] - rat[k][both]) / np.maximum(np.abs(rat[k][both]), 1.0)).max()))
            if k < L - 1:
                M = len(res[k]["slots"]) if res[k] is not None else 0
                if res[k] is None:
                    assert np.isnan(r["postfit"][k, :, i]).all(), (tag, i, k)
                else:
                    got = r["postfit"][k, res[k]["slots"], i]
                    worst["postfit"] = max(worst.get("postfit", 0.0), float(np.abs(got - res[k]["postfit"]).max()))
    print(f"SMOOTH-KERNEL {tag} " + " ".join(f"{k}={v:.2g}" for k, v in worst.items()))
    assert all(v <= tol_rel[k] for k, v in worst.items()), (tag, worst)


@pytest.mark.parametrize("variant", ("ekf", "ekf_scalar_noreject", "ckf_reject", "ckf_scalar"))
def test_smoothing_kernel_on_the_oracle_records_matches_the_restatement(variant):
    streams, outs, packed = streams_of("srp", variant)
    prop, eng = engine("STRICT", "srp")
    _, cfg, names, st_c, epochs, tracker, obs, *_ = inputs("srp", variant, prop)
    rec = stack(streams, max(len(s) for s in streams) + 3)
    r = eng.od_smooth_batch(cfg, len(names), st_c, tracker, obs, rec, np.zeros(om.N_F, dtype=np.int32))
    assert (r["status"] == 0).all(), r["status"]
    ref = restated(streams, outs, packed, "srp", variant, st_c, tracker, obs)
    # the kernel alone: rounding of a 9x9 LU inverse and two products (state: absolute km / 1e4)
    compare_smoothed(r, ref, rec, dict(state=1e-15, dev=1e-12, covar=1e-12, postfit=1e-9, ratio=1e-6),
                     f"kernel/srp/{variant}")


@pytest.mark.parametrize("variant", ("ckf_reject", "ekf"))
@pytest.mark.parametrize("family", FAMILIES)
def test_filter_then_smooth_matches_the_restatement(family, variant):
    plain, rec, (cfg, names, st_c, tracker, obs, eng) = run_both(family, "field", variant)
    r = eng.od_smooth_batch(cfg, len(names), st_c, tracker, obs, rec.records, rec.status)
    assert (r["status"] == 0).all()
    streams, outs, packed = streams_of("field", variant)
    ref = restated(streams, outs, packed, "field", variant, st_c, tracker, obs)
    compare_smoothed(r, ref, rec.records, dict(state=1e-13, dev=1e-5, covar=1e-7, postfit=1e-7, ratio=1e-2), f"chain/{family}/{variant}")


def test_statuses_alone_vs_batch_and_null_outputs():
    plain, rec, (cfg, names, st_c, tracker, obs, eng) = run_both("STRICT", "field", "ekf")
    R = rec.records
    full = eng.od_smooth_batch(cfg, len(names), st_c, tracker, obs, R, rec.status)
    assert (full["status"] == 0).all()
    # a filter alone gives the same bits as in the batch
    i = 5
    one = {k: (v[..., i:i + 1].copy() if k != "count" else v[i:i + 1].copy()) for k, v in R.items()}
    alone = eng.od_smooth_batch(cfg, len(names), st_c, tracker, np.ascontiguousarray(obs[:, :, i:i + 1]), one, rec.status[i:i + 1])
    for k in ("state", "deviation", "covar", "fs_ratio", "postfit"):
        assert np.array_equal(alone[k][..., 0], full[k][..., i], equal_nan=True), k
    # NULL optional outputs: the others are unchanged
    part = eng.od_smooth_batch(cfg, len(names), st_c, tracker, obs, R, rec.status, outputs=("covar",))
    assert set(part) == {"covar", "status"} and np.array_equal(part["covar"], full["covar"], equal_nan=True)
    # per-filter statuses, never aborting the batch
    bad = {k: v.copy() for k, v in R.items()}
    fst = rec.status.copy()
    fst[0] = abi.ERR_PROP_MATH                       # a failed filter: skipped, its status copied
    bad["count"][1] = 1                              # fewer than two estimates
    bad["count"][2] = R["epoch"].shape[0] + 1        # truncated
    bad["stm"][7, :, 3] = 0.0                        # singular Phi at record 7
    r = eng.od_smooth_batch(cfg, len(names), st_c, tracker, obs, bad, fst)
    assert r["status"].tolist()[:4] == [abi.ERR_PROP_MATH, abi.ERR_TOO_FEW_MEASUREMENTS, abi.ERR_RECORDS_TRUNCATED, abi.ERR_SINGULAR_STM]
    for j in range(4):
        assert np.isnan(r["covar"][..., j]).all() and np.isnan(r["state"][..., j]).all()
    for k in ("state", "deviation", "covar", "fs_ratio", "postfit"):
        assert np.array_equal(r[k][..., 4:], full[k][..., 4:], equal_nan=True), k
    # records written with another msr_size are a bad argument
    cfg1 = copy.copy(cfg)
    cfg1.msr_size = 1
    with pytest.raises(nb.PropagationError, match="msr_size"):
        eng.od_smooth_batch(cfg1, len(names), st_c, tracker, obs, R, rec.status)


def test_odsolution_smooth_reruns_on_truncation_and_keeps_the_filter():
    prop = om.propagator("field", nb.MODE_FAST)
    odp = om.od_process(prop, "field", "ekf")
    epochs, schedule, obs, dev = om.arc("field", "regular")
    odp.devices = dict(dev)
    st, cs, ep, cov = om.filters("field")
    tmpl = nb.Spacecraft(orbit=om.truth_orbit("field"))
    ests = [nb.KfEstimate(tmpl.with_vector(int(ep[i]), st[:, i]), cov[:, i].reshape(9, 9).T.copy()) for i in range(om.N_F)]
    arc = nb.TrackingDataArc(epochs, list(schedule), obs)
    sol = odp.process_arcs(ests, arc, estimates_capacity=20)          # far too small: smooth() runs the filters again
    assert sol.records["count"].max() > 20
    sm = sol.smooth()
    assert sm.is_smoother_run() and not sol.is_smoother_run()
    assert sm.records["epoch"].shape[0] == sol.records["count"].max()
    assert all(sm.error(i) is None for i in range(om.N_F))
    assert np.array_equal(sm.prefit, sol.prefit, equal_nan=True) and np.array_equal(sm.resid_ratio, sol.resid_ratio, equal_nan=True)
    for i in range(om.N_F):
        n_est = sm.n_estimates(i)
        assert len(sm.residuals(i)) == n_est == sm.records["count"][i]
        assert np.isfinite(sm.rms_postfit_residuals(i)) and np.isfinite(sm.rms_prefit_residuals(i))
        assert sm.rms_prefit_residuals(i) == pytest.approx(np.sqrt(sum(float(r[0] @ r[0]) for r in sm.residuals(i) if r is not None) / n_est))
        est = sm.estimate(n_est - 1, i)
        assert np.array_equal(est.covar, sm.records["covar"][n_est - 1, :, i].reshape(9, 9).T)


# ---- adaptive step: the records of the STRICT filter against the oracle's stream at the same adaptive DP78 settings
@pytest.mark.parametrize("variant", ("ekf", "ckf_scalar"))
def test_records_match_the_oracle_stream_at_adaptive_step(variant):
    dyn = om.dynamics("field")
    prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions(init_step=7 * 10**9), mode=nb.MODE_STRICT)
    _, cfg, names, st_c, epochs, tracker, obs, st, cs, ep, cov = inputs("field", variant, prop)
    eng = prop.engine(om.frame("field"), om.almanac("field"))
    plain = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True)
    rec = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True, estimates_capacity=400)
    assert_same_outputs(plain, rec)
    packed = prop.dynamics.pack(om.frame("field"), om.almanac("field"))
    streams = []
    for i in range(om.N_F):
        sink = []
        so.process_arc(packed.c, prop.opts.to_c(prop.method), cfg, st_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]), st[:, i].copy(),
                       cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy(), sink=sink)
        streams.append(sink)
    assert_records_match(rec.records, streams, f"STRICT-adaptive/field/{variant}")


# ---- the reference's own smoothing tests (tests/orbit_determination/two_body.rs), restated on an ensemble
def _two_body_case(n, mode, variant, offsets):
    """22 000 km Keplerian orbit, two-body, RK4 at a fixed 10 s, 1 day; Madrid / Canberra / Goldstone at a 0 deg mask, noise-free
    tracking every 10 s (from t0) from every station that sees the spacecraft, processed with 1e-6 noise (StochasticNoise::MIN).
    As in the reference, the observations come from the same code as the filter's computed ones: a CKF started on the truth (whose
    nominal is never replaced) returns prefit = obs - computed, exact by Sterbenz's lemma, and obs - prefit is the computed value
    itself.  Returns the process, the arc, the n estimates, the truth at t0 and the truth by epoch (the CKF's nominal)."""
    frame = nb.EARTH_J2000
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    prop = nb.Propagator.new(dyn, nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=mode)
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0, 0.01, 30.0, 80.0, 40.0, 0.0, 0, frame))
    day = 86400 * 10**9
    st1, cs1, ep1 = nb.pack_spacecraft([truth0])
    _, _, _, tst, (t_ep, t_st, t_cnt) = prop.engine(frame, None).propagate_batch(st1, cs1, ep1, day, traj_capacity=8700)
    assert tst[0] == 0 and t_ep[t_cnt[0] - 1, 0] == day
    ep_all, st_all = t_ep[: t_cnt[0], 0], t_st[:, : t_cnt[0], 0].T
    sim = {"Madrid": nb.GroundStation.dss65_madrid(0.0, nb.StochasticNoise(0.0), nb.StochasticNoise(0.0)),
           "Canberra": nb.GroundStation.dss34_canberra(0.0, nb.StochasticNoise(0.0), nb.StochasticNoise(0.0)),
           "Goldstone": nb.GroundStation.dss13_goldstone(0.0, nb.StochasticNoise(0.0), nb.StochasticNoise(0.0))}
    epochs, names, obs = [], [], []
    for name in sim:
        a = nb.simulate_tracking(ep_all, st_all[:, :6, None], sim, [name] * len(ep_all), frame, None, None)
        vis = ~np.isnan(a.obs[:, 0, 0])
        epochs.append(ep_all[vis]); names += [name] * int(vis.sum()); obs.append(a.obs[vis])
    epochs = np.concatenate(epochs); obs = np.concatenate(obs)
    order = np.argsort(epochs, kind="stable")
    epochs, names, obs = epochs[order], [names[j] for j in order], obs[order]
    mn = nb.StochasticNoise(1e-6)
    proc = {"Madrid": nb.GroundStation.dss65_madrid(0.0, mn, mn), "Canberra": nb.GroundStation.dss34_canberra(0.0, mn, mn),
            "Goldstone": nb.GroundStation.dss13_goldstone(0.0, mn, mn)}
    cov = np.diag([1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0.0, 0.0, 0.0])
    sim_od = nb.KalmanODProcess(prop, nb.KalmanVariant.DeviationTracking, None, proc, None, msr_size=2)
    cap = len(ep_all) + len(epochs)                 # at most one time update per 10 s step plus one record per measurement window
    sim_sol = sim_od.process_arcs([nb.KfEstimate.from_covar(truth0, cov)], nb.TrackingDataArc(epochs, names, obs), estimates_capacity=cap)
    assert sim_sol.records["count"][0] <= cap
    assert sim_sol.status[0] == 0 and (sim_sol.msr_flags[:, 0] == abi.MSRF_PROCESSED).all()
    obs = obs - sim_sol.prefit
    L = sim_sol.n_estimates(0)
    truth_at = {int(e): sim_sol.records["nominal"][k, :, 0].copy() for k, e in enumerate(sim_sol.records["epoch"][:L, 0])}
    arc = nb.TrackingDataArc(epochs, names, np.repeat(obs, n, axis=2))
    odp = nb.KalmanODProcess(prop, variant, None, proc, None, msr_size=2)
    ests = []
    for i in range(n):
        v = truth0.to_vector()
        v[:3] += offsets[i]
        ests.append(nb.KfEstimate.from_covar(truth0.with_vector(0, v), cov))
    return odp, arc, ests, truth0.to_vector(), truth_at, cap


def test_od_tb_fixed_step_smooth_test_as_an_ensemble():
    """od_tb_fixed_step_smooth_test: EKF from (+0.1, -0.1, +0.05) km off (filter 0; the other 63 start at other offsets of the same
    size), smoothed.  Asserts, per filter, the reference's checks: the filter's final error below the station level (0.1 km,
    1 m/s), the smoothed first estimate (at t0) no worse in order of magnitude than the start, the final smoothed estimate within
    75 m / 50 mm/s."""
    rng = np.random.default_rng(11)
    base = np.array([0.1, -0.1, 0.05])
    offsets = [base] + [rng.permutation(base) * rng.choice([-1.0, 1.0], 3) for _ in range(63)]
    odp, arc, ests, y0, truth_at, cap = _two_body_case(64, nb.MODE_FAST, nb.KalmanVariant.ReferenceUpdate, offsets)
    sol = odp.process_arcs(ests, arc, estimates_capacity=cap)
    assert (sol.status == 0).all() and sol.records["count"].max() <= cap
    sm = sol.smooth()
    worst = [0.0, 0.0, 0.0]
    for i in range(64):
        assert sm.error(i) is None
        L = sol.n_estimates(i)
        assert sol.records["epoch"][0, i] == 0
        last = sol.estimate(L - 1, i)
        yf = truth_at[last.nominal_state.epoch()]
        y = last.state().to_vector()
        assert np.linalg.norm(y[:3] - yf[:3]) < 0.1 and np.linalg.norm(y[3:6] - yf[3:6]) < 1e-3, i
        d_no = np.linalg.norm(offsets[i])
        d_it = np.linalg.norm(sm.estimate(0, i).state().to_vector()[:3] - y0[:3])
        assert d_it < d_no or np.floor(np.log10(d_it)) <= np.floor(np.log10(d_no)), (i, d_it, d_no)
        fin = sm.estimate(L - 1, i).state().to_vector()
        e_r, e_v = np.linalg.norm(fin[:3] - yf[:3]), np.linalg.norm(fin[3:6] - yf[3:6])
        assert e_r < 75e-3 and e_v < 50e-6, (i, e_r, e_v)
        worst = [max(worst[0], d_it), max(worst[1], e_r), max(worst[2], e_v)]
    print(f"OD-TB-SMOOTH: {len(arc)} measurements; worst smoothed t0 error {worst[0]:.2e} km, final {worst[1]:.2e} km {worst[2]:.2e} km/s")


def test_od_tb_val_ckf_fixed_step_perfect_stations_smoothing():
    """od_tb_val_ckf_fixed_step_perfect_stations, its smoothing part: a CKF started on the truth, the same dynamics and step as the
    simulation; after smooth(), the last estimate has a deviation norm < 1e-12, a covariance diagonal norm < 1e-4, and is within
    1e-9 km and 1e-9 km/s of the truth.  The filter's own checks before smoothing are asserted too."""
    odp, arc, ests, y0, truth_at, cap = _two_body_case(4, nb.MODE_STRICT, nb.KalmanVariant.DeviationTracking, [np.zeros(3)] * 4)
    sol = odp.process_arcs(ests, arc, estimates_capacity=cap)
    assert (sol.status == 0).all() and sol.records["count"].max() <= cap
    for i in range(4):
        L = sol.n_estimates(i)
        ep = sol.records["epoch"][:L, i]
        assert (np.diff(ep[1:]) >= 0).all()
        assert (sol.records["covar"][1:L, ::10, i][:, :6] >= 0.0).all()
        assert np.linalg.norm(sol.records["deviation"][:L, :, i], axis=1).max() < 1e-12
        for r in sol.residuals(i):
            if r is not None:
                assert np.linalg.norm(r[0]) < 1e-12 and np.linalg.norm(r[1]) < 1e-12
    sm = sol.smooth()
    for i in range(4):
        assert sm.error(i) is None
        est = sm.estimate(sm.n_estimates(i) - 1, i)
        assert np.linalg.norm(est.state_deviation) < 1e-12
        assert np.linalg.norm(np.diag(est.covar)) < 1e-4
        y, yf = est.state().to_vector(), truth_at[est.nominal_state.epoch()]
        assert np.linalg.norm(y[:3] - yf[:3]) < 1e-9 and np.linalg.norm(y[3:6] - yf[3:6]) < 1e-9, (i, y[:6] - yf[:6])


def test_per_estimate_parquet_export(tmp_path):
    """ODSolution.to_parquet with records: one row per estimate, the covariance, RIC sigma and filter-smoother columns."""
    import pyarrow.parquet as pq

    prop = om.propagator("field", nb.MODE_FAST)
    odp = om.od_process(prop, "field", "ckf_reject")
    epochs, schedule, obs, dev = om.arc("field", "regular")
    odp.devices = dict(dev)
    st, cs, ep, cov = om.filters("field")
    tmpl = nb.Spacecraft(orbit=om.truth_orbit("field"))
    ests = [nb.KfEstimate(tmpl.with_vector(int(ep[i]), st[:, i]), cov[:, i].reshape(9, 9).T.copy()) for i in range(om.N_F)]
    sol = odp.process_arcs(ests, nb.TrackingDataArc(epochs, list(schedule), obs), estimates_capacity=300)
    sm = sol.smooth()
    i = 3
    L = sol.n_estimates(i)
    for s_, name in ((sol, "filter.parquet"), (sm, "smoothed.parquet")):
        t = pq.read_table(s_.to_parquet(tmp_path / name, index=i))
        assert t.num_rows == L
        names = t.column_names
        assert "Covariance X*Y (Earth J2000) (km^2)" in names and "Sigma X (RIC) (km)" in names and "Filter-smoother ratio X (km^2)" in names
        P = np.stack([s_.estimate(k, i).covar for k in range(L)])
        assert np.array_equal(t.column("Covariance X*Vy (Earth J2000) (km^2/s)").to_numpy(), P[:, 0, 4])
        fs = t.column("Filter-smoother ratio X (km^2)")
        if s_ is sm:
            assert fs.null_count == 1 and not fs[L - 1].is_valid
            assert np.array_equal(fs.to_numpy(zero_copy_only=False)[: L - 1], sm.filter_smoother_ratios(i)[: L - 1, 0], equal_nan=True)
        else:
            assert fs.null_count == L
        tu = sum(r is None for r in s_.residuals(i))
        assert t.column("Tracker").null_count == tu
