"""Angle tracking (nyxb_od_aer_batch, nyxb_od_aer_smooth_batch) on the GPU: the three kernel families against the restatement
(tests/aer_oracle.py), range/Doppler-only stations against nyxb_od_ekf_batch, the argument checks, and the reference's
od_tb_val_az_el_ckf_fixed_step_perfect_stations restated with its smoothing."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import aer_oracle as ao
from tests.aer_util import ALL, dsn, oracle_run, scenario

pytestmark = pytest.mark.gpu
S = 10**9
FAMILIES = ("STRICT", "FAST-thread", "FAST-coop")
TOL = {"STRICT": (1e-9, 1e-12), "FAST-thread": (1e-6, 1e-9), "FAST-coop": (1e-6, 1e-9)}   # km, km/s (the position tests' bounds)
ANG = (MT.Azimuth, MT.Elevation)
ELRAZ = (MT.Elevation, MT.Range, MT.Azimuth)
RC_BAD_ARG = -1   # NYXB_RC_BAD_ARG


def _prop(sc, family):
    mode = nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST
    prop = nb.Propagator.new(sc["dyn"], nb.IntegratorMethod.DormandPrince78, sc["opts"], mode=mode)
    prop.engine(sc["frame"], None).set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    return prop


def process(sc, family, variant=nb.KalmanVariant.ReferenceUpdate, msr_size=2, reject=None, snc=None, cap=None, devices=None):
    odp = nb.KalmanODProcess(_prop(sc, family), variant, nb.SigmaRejection(reject) if reject else None, devices or sc["devices"], None,
                             msr_size=msr_size)
    if snc is not None:
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12] * 3, 10 * nb.Unit.Minute, snc))
    return odp, odp.process_arcs(sc["ests"], sc["arc"], estimates_capacity=cap)


# Bounds of the residuals per type of the output slot (km, km/s, deg, deg) and of the residual ratio: 10 x the largest difference over
# this file's cases, prefit and postfit alike, measured on an H100 80GB HBM3 (700 W), rounded up.  Range 2.1e-9 km (STRICT, the postfit
# of the short-window case) and 6.2e-10 km (FAST), Doppler 3.5e-14 / 5.2e-14 km/s, azimuth 6.1e-12 / 1.9e-12 deg, elevation 2.0e-13 /
# 2.8e-13 deg, ratio 1.0e-5 (STRICT, the short-window case) / 3.2e-6.  tests/test_gpu_aer_matrix.py pins the same kernels to the restatement's own spread.
SLOT_TOL = {"STRICT": {MT.Range: 3e-8, MT.Doppler: 4e-13, MT.Azimuth: 7e-11, MT.Elevation: 3e-12, "ratio": 1e-4},
            "FAST-thread": {MT.Range: 7e-9, MT.Doppler: 6e-13, MT.Azimuth: 2e-11, MT.Elevation: 3e-12, "ratio": 4e-5},
            "FAST-coop": {MT.Range: 7e-9, MT.Doppler: 6e-13, MT.Azimuth: 2e-11, MT.Elevation: 3e-12, "ratio": 4e-5}}


def slot_types(sc, odp):
    """[m][4]: the type at each output slot (the list position in the measurement's station), None where there is none."""
    out = []
    for nm in sc["arc"].tracker:
        types = list(odp.devices[nm].measurement_types) if nm in odp.devices else []
        out.append([MT(t) for t in types] + [None] * (4 - len(types)))
    return out


def check_residuals(types, family, got, ref, stop=None):
    """prefit and postfit per slot type, the ratio on its own bound: the NaN patterns equal, the differences within SLOT_TOL."""
    tol = SLOT_TOL[family]
    for f in ("prefit", "postfit", "resid_ratio"):
        g, r = got[f][:stop], ref[f][:stop]
        assert np.array_equal(np.isnan(g), np.isnan(r)), f
        d = np.abs(np.nan_to_num(g) - np.nan_to_num(r))
        worst = {}
        for k in range(d.shape[0]):
            for q in range(4):
                key = "ratio" if f == "resid_ratio" else types[k][q]
                if key is not None:
                    worst[key] = max(worst.get(key, 0.0), float(d[k, q]))
        print(f"AERSLOT {family} {f} " + " ".join(f"{getattr(k, 'name', k)}={v:.1e}" for k, v in worst.items()))
        assert all(v <= tol[k] for k, v in worst.items()), (f, worst)


def check(sc, odp, sol, family, filters=None):
    tr, tv = TOL[family]
    types = slot_types(sc, odp)
    for i in (filters if filters is not None else range(len(sc["ests"]))):
        ref = oracle_run(sc, odp, i)
        assert sol.status[i] == ref["status"]
        if family == "STRICT":
            assert sol.details["n_steps"][i] == ref["n_steps"]
        assert np.abs(sol.final_state_soa[:3, i] - ref["state"][:3]).max() < tr
        assert np.abs(sol.final_state_soa[3:6, i] - ref["state"][3:6]).max() < tv
        assert np.allclose(sol.covar[i], ref["covar"], rtol=1e-6, atol=1e-15)
        assert np.array_equal(sol.msr_flags[:, i], ref["flags"])
        check_residuals(types, family, {f: getattr(sol, f)[:, :, i] for f in ("prefit", "postfit", "resid_ratio")}, ref)


VARIANTS = {
    "ekf-m2": dict(),
    "ckf-m2": dict(variant=nb.KalmanVariant.DeviationTracking),
    "ekf-m1-snc-ric": dict(msr_size=1, snc=nb.LocalFrame.RIC),
    "ckf-m1": dict(variant=nb.KalmanVariant.DeviationTracking, msr_size=1),
    "ekf-m2-reject": dict(reject=2.0),
}


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("name", list(VARIANTS))
def test_parity(family, name):
    sc = scenario()
    odp, sol = process(sc, family, **VARIANTS[name])
    assert (sol.status == 0).all()
    if name == "ekf-m2-reject":
        assert (sol.msr_flags & abi.MSRF_REJECTED).any()
    check(sc, odp, sol, family)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("types", [ANG, ELRAZ], ids=["angles-only", "el-r-az"])
@pytest.mark.parametrize("msr_size", [1, 2])
def test_parity_type_lists(family, types, msr_size):
    """Angles only, and [El, R, Az], with a 10 deg mask (invisible passes), absent types, an all-absent measurement and an unknown
    tracker.  [El, R, Az] at msr_size 2 ends each measurement with the short window [Az]: its identity row with a zero R entry collapses
    the covariance along that row, and a later window ends the filter with SingularNoiseRk (status 1), as in the restatement.  Which
    measurement fails is decided by a pivot at the rounding level, so that case compares every measurement before the first one that
    fails on either side (several of them through the short window) and the status."""
    sc = scenario(types=types, fixed=True, seed=2, n_msr=40, cadence_s=120, orbit=nb.Orbit.keplerian(
        26000.0, 0.02, 40.0, 30.0, 40.0, 10.0, 0, nb.EARTH_J2000))
    sc["devices"] = dsn(10.0, types)          # data simulated without a mask, processed with one
    sc["arc"].obs[3, int(MT.Azimuth), :] = np.nan
    sc["arc"].obs[5, :, 1] = np.nan
    sc["arc"].tracker[7] = "nobody"
    odp, sol = process(sc, family, variant=nb.KalmanVariant.DeviationTracking, msr_size=msr_size)
    singular = types == ELRAZ and msr_size == 2
    assert (sol.status == (1 if singular else 0)).all()
    if singular:
        for i in range(len(sc["ests"])):
            ref = oracle_run(sc, odp, i)
            assert ref["status"] == 1
            stop = min(np.nonzero(sol.msr_flags[:, i])[0][-1], np.nonzero(ref["flags"])[0][-1])   # the failing measurement
            assert stop >= 20 and np.isfinite(ref["resid_ratio"][:stop, 1]).sum() >= 4     # short windows [Az] before it
            assert np.array_equal(sol.msr_flags[:stop, i], ref["flags"][:stop])
            check_residuals(slot_types(sc, odp), family, {f: getattr(sol, f)[:, :, i] for f in ("prefit", "postfit", "resid_ratio")}, ref,
                            stop)
            assert np.isnan(sol.prefit[:stop, 3, i]).all() and np.isfinite(sol.prefit[:stop, 2, i]).sum() >= 4
        return
    assert (sol.msr_flags & abi.MSRF_NOT_VISIBLE).any() and (sol.msr_flags & abi.MSRF_PROCESSED).any()
    assert sol.msr_flags[5, 1] == abi.MSRF_ABSENT and sol.msr_flags[7, 0] == 0
    check(sc, odp, sol, family)


@pytest.mark.parametrize("family", FAMILIES)
def test_records_null_outputs_and_batch_invariance(family):
    """Records on or off and NULL optional outputs leave `out` bit-identical; each filter of a batch equals the same filter alone;
    the records equal the restatement's stream."""
    sc = scenario(n=5, seed=3)
    odp, plain = process(sc, family, msr_size=1)
    _, rec = process(sc, family, msr_size=1, cap=200)
    for f in ("final_state_soa", "covar", "state_deviation", "resid_ratio", "prefit", "postfit", "msr_flags"):
        assert np.array_equal(getattr(plain, f), getattr(rec, f), equal_nan=True), f
    names, st_c = odp.aer_stations_c(sc["frame"])
    tracker = np.array([names.index(t) for t in sc["arc"].tracker], dtype=np.int32)
    st, cs, ep = nb.pack_spacecraft(e.nominal_state for e in sc["ests"])
    cov0 = np.stack([np.asarray(e.covar).T.reshape(81) for e in sc["ests"]], axis=1)
    n = len(sc["ests"])
    m = len(sc["arc"])
    out_state, out_epoch, out_cov, status = np.empty((9, n)), np.empty(n, dtype=np.int64), np.empty((81, n)), np.zeros(n, dtype=np.int32)
    out = abi.OdOutputsC(out_state.ctypes.data, out_epoch.ctypes.data, out_cov.ctypes.data, None, None, None, None, None, None, None, None,
                         status.ctypes.data)
    obs = np.ascontiguousarray(sc["arc"].obs)
    arc_c = abi.TrackingArcC(m, sc["arc"].epoch_ns.ctypes.data, tracker.ctypes.data, obs.ctypes.data)
    eng = odp.prop.engine(sc["frame"], None)
    rc = eng._lib.nyxb_od_aer_batch(eng._h, C.byref(odp.config_c()), len(names), st_c, C.byref(arc_c), n, st.ctypes.data, cs.ctypes.data,
                                    ep.ctypes.data, cov0.ctypes.data, C.byref(out), None)
    assert rc == 0 and np.array_equal(out_state, plain.final_state_soa) and (status == plain.status).all()
    alone = odp.process_arcs([sc["ests"][3]], nb.TrackingDataArc(sc["arc"].epoch_ns, sc["arc"].tracker, sc["arc"].obs[:, :, 3:4], ALL))
    assert np.array_equal(alone.final_state_soa[:, 0], plain.final_state_soa[:, 3])
    assert np.array_equal(alone.prefit[:, :, 0], plain.prefit[:, :, 3], equal_nan=True)
    sink = []
    oracle_run(sc, odp, 1, sink=sink)
    L = rec.n_estimates(1)
    assert L == len(sink)
    assert [int(t) for t in rec.records["tag"][:L, 1]] == [s["tag"] for s in sink]
    assert max(abs(int(x) >> 3 & 3) for x in rec.records["tag"][:L, 1] if x >= 0) == 3       # window 3 at msr_size 1
    for k in range(L):
        assert np.abs(rec.records["nominal"][k, :3, 1] - sink[k]["nominal"][:3]).max() < 10 * TOL[family][0]


def _rd_only():
    """Range/Doppler-only stations, the arc padded to four slots (NaN angles)."""
    sc = scenario(types=(MT.Range, MT.Doppler), seed=8)
    arc = sc["arc"]
    arc.obs[4, 1, :] = np.nan
    pad = np.full((len(arc), 2, arc.n), np.nan)
    sc["arc"] = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, np.concatenate([arc.obs, pad], axis=1), ALL)
    return sc


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("msr_size", [1, 2])
def test_range_doppler_stations_match_the_ground_path(family, msr_size):
    """Range/Doppler-only stations through nyxb_od_aer_batch against the same arc through nyxb_od_ekf_batch: bit-identical on
    STRICT (state, covariance, prefit, postfit, ratio in its slot, flags, records), the FAST filter tolerance otherwise."""
    sc = _rd_only()
    arc4 = sc["arc"]
    arc2 = nb.TrackingDataArc(arc4.epoch_ns, arc4.tracker, arc4.obs[:, :2, :])
    outs = []
    for arc in (arc4, arc2):
        odp = nb.KalmanODProcess(_prop(sc, family), nb.KalmanVariant.ReferenceUpdate, nb.SigmaRejection(3.0), sc["devices"], None,
                                 msr_size=msr_size)
        outs.append(odp.process_arcs(sc["ests"], arc, estimates_capacity=300))
    a, g = outs
    assert (a.status == 0).all() and (g.status == 0).all()
    slot = [0, 1] if msr_size == 1 else [0, 0]
    ratio_a = np.stack([a.resid_ratio[:, w, :] for w in range(2 if msr_size == 1 else 1)], axis=1)
    ratio_g = np.stack([g.resid_ratio[:, slot[w], :] for w in range(2 if msr_size == 1 else 1)], axis=1)
    assert np.isnan(a.prefit[:, 2:, :]).all() and np.isnan(a.resid_ratio[:, 2:, :]).all()
    if family == "STRICT":
        for f in ("final_state_soa", "covar", "state_deviation", "msr_flags"):
            assert np.array_equal(getattr(a, f), getattr(g, f)), f
        for f in ("prefit", "postfit"):
            assert np.array_equal(getattr(a, f)[:, :2, :], getattr(g, f), equal_nan=True), f
        assert np.array_equal(ratio_a, ratio_g, equal_nan=True)
        ra, rg = a.records, g.records
        assert np.array_equal(ra["count"], rg["count"])
        for k in ("epoch", "nominal", "deviation", "covar", "stm"):
            assert np.array_equal(ra[k], rg[k], equal_nan=True), k
        tags_a = [abi.od_pos_tag_fields(int(x)) if x >= 0 else x for x in ra["tag"].ravel()]
        tags_g = [abi.od_tag_fields(int(x)) if x >= 0 else x for x in rg["tag"].ravel()]
        assert tags_a == tags_g
    else:
        tr, tv = TOL[family]
        assert np.abs(a.final_state_soa[:3] - g.final_state_soa[:3]).max() < tr
        assert np.abs(a.final_state_soa[3:6] - g.final_state_soa[3:6]).max() < tv
        assert np.array_equal(a.msr_flags, g.msr_flags)
        assert np.allclose(np.nan_to_num(a.prefit[:, :2]), np.nan_to_num(g.prefit), rtol=1e-5, atol=10 * tr)


@pytest.mark.parametrize("family", FAMILIES)
def test_zero_variance_is_singular_noise(family):
    """msr_size 1, a zero azimuth variance and a zero initial covariance: S is zero, the fallback to R finds R singular too, so the
    first azimuth window ends the filter with SingularNoiseRk (status 1), as the restatement."""
    sc = scenario(types=ANG, sigma={MT.Range: 1.0, MT.Doppler: 1.0, MT.Azimuth: 0.0, MT.Elevation: 1e-3}, seed=9, n_msr=8)
    for e in sc["ests"]:
        e.covar[:] = 0.0
    odp, sol = process(sc, family, msr_size=1)
    assert (sol.status == 1).all()
    check(sc, odp, sol, family)


def test_argument_checks():
    """BAD_ARG for a type outside 0..3, a duplicate type, n_types outside 1..4 and msr_size outside 1..2, before any launch."""
    sc = scenario(n=1, n_msr=4)
    odp = nb.KalmanODProcess(_prop(sc, "STRICT"), nb.KalmanVariant.ReferenceUpdate, None, sc["devices"], None, msr_size=2)
    eng = odp.prop.engine(sc["frame"], None)
    names, st_c = odp.aer_stations_c(sc["frame"])
    st, cs, ep = nb.pack_spacecraft(e.nominal_state for e in sc["ests"])
    cov0 = np.asarray(sc["ests"][0].covar).T.reshape(81, 1).copy()
    tracker = np.zeros(4, dtype=np.int32)
    obs = np.ascontiguousarray(sc["arc"].obs)
    arc_c = abi.TrackingArcC(4, sc["arc"].epoch_ns.ctypes.data, tracker.ctypes.data, obs.ctypes.data)
    o_st, o_ep, o_cov, o_s = np.empty((9, 1)), np.empty(1, dtype=np.int64), np.empty((81, 1)), np.zeros(1, dtype=np.int32)
    out = abi.OdOutputsC(o_st.ctypes.data, o_ep.ctypes.data, o_cov.ctypes.data, None, None, None, None, None, None, None, None, o_s.ctypes.data)

    def call(stations, cfg=None):
        return eng._lib.nyxb_od_aer_batch(eng._h, C.byref(cfg or odp.config_c()), len(names), stations, C.byref(arc_c), 1, st.ctypes.data,
                                          cs.ctypes.data, ep.ctypes.data, cov0.ctypes.data, C.byref(out), None)

    assert call(st_c) == 0 and o_s[0] == 0
    launches = eng._lib.nyxb_engine_launch_count(eng._h)
    bad = [("types", 0, 4), ("types", 1, -1), ("types", 1, 0), ("n_types", None, 0), ("n_types", None, 5)]
    for field, idx, val in bad:
        arr = (abi.AerStationC * len(names))()
        C.memmove(arr, st_c, C.sizeof(arr))
        if idx is None:
            setattr(arr[0], field, val)
        else:
            getattr(arr[0], field)[idx] = val
        assert call(arr) == RC_BAD_ARG, (field, idx, val)
    for M in (0, 3):
        cfg = odp.config_c()
        cfg.msr_size = M
        assert call(st_c, cfg) == RC_BAD_ARG
        assert b"msr_size" in abi.load_library().nyxb_last_error()
    assert eng._lib.nyxb_engine_launch_count(eng._h) == launches        # rejected before any device work
    # the types of a station with angles are refused by the range/Doppler entry point, and an angle station needs a 4-slot arc
    with pytest.raises(nb.ODError):
        odp.process_arcs(sc["ests"], nb.TrackingDataArc(sc["arc"].epoch_ns, sc["arc"].tracker, sc["arc"].obs[:, :2]))


def test_smoother_against_restatement_and_failed_filters():
    """nyxb_od_aer_smooth_batch against the restated smoother (states, covariances, four-slot postfits through the AER window); a filter
    with a nonzero status is not smoothed and has NaN outputs."""
    from dataclasses import replace

    sc = scenario(n=3, seed=12, fixed=True)
    sc["devices"] = dsn(types=ANG)
    odp, sol = process(sc, "STRICT", msr_size=1, cap=400)
    assert (sol.status == 0).all()
    sol = replace(sol, status=np.array([0, 0, 1], dtype=np.int32))
    sm = sol.smooth()
    names, st_c = odp.aer_stations_c(sc["frame"])
    tracker = np.array([names.index(t) for t in sc["arc"].tracker], dtype=np.int32)
    for i in (0, 1):
        want = ao.smooth_restated(sol.records, i, st_c, None, 1, sc["arc"].obs, tracker)
        for k, (ys, Ps, post) in enumerate(want):
            assert np.abs(sm.smoother["state"][k, :3, i] - ys[:3]).max() < 1e-7
            assert np.allclose(sm.smoother["covar"][k, :, i].reshape(9, 9).T, Ps, rtol=1e-6, atol=1e-14)
            g = sm.smoother["postfit"][k, :, i]
            assert np.array_equal(np.isnan(g), np.isnan(post)) and np.allclose(np.nan_to_num(g), np.nan_to_num(post), rtol=1e-6, atol=1e-9)
        assert np.isfinite(sm.rms_postfit_residuals(i))
    assert sm.error(2) is not None and np.isnan(sm.smoother["state"][:, :, 2]).all() and np.isnan(sm.smoother["postfit"][:, :, 2]).all()


def _perfect_stations(n):
    """od_tb_val_az_el_ckf_fixed_step_perfect_stations (tests/orbit_determination/two_body.rs:599-856): 22 000 km orbit, two-body, RK4
    at a fixed 10 s, 1 day; Madrid, Canberra and Goldstone at a 0 deg mask with azimuth and elevation only, noise-free tracking every
    10 s from every station that sees the spacecraft, processed with sigma 1e-6 by a CKF started on the truth.  As in the test for
    range and Doppler (tests/test_gpu_smooth.py), the observations are the filter's own computed values: obs - prefit of a first run."""
    frame = nb.EARTH_J2000
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    prop = nb.Propagator.new(dyn, nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=nb.MODE_STRICT)
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0, 0.01, 30.0, 80.0, 40.0, 0.0, 0, frame))
    day = 86400 * S
    st1, cs1, ep1 = nb.pack_spacecraft([truth0])
    _, _, _, tst, (t_ep, t_st, t_cnt) = prop.engine(frame, None).propagate_batch(st1, cs1, ep1, day, traj_capacity=8700)
    assert tst[0] == 0 and t_ep[t_cnt[0] - 1, 0] == day
    ep_all, st_all = t_ep[: t_cnt[0], 0], t_st[:, : t_cnt[0], 0].T
    zero = {t: 0.0 for t in ALL}
    sim = dsn(0.0, ANG, zero)
    epochs, names, obs = [], [], []
    for name in sim:
        a = nb.simulate_tracking(ep_all, st_all[:, :6, None], sim, [name] * len(ep_all), frame, None, None)
        vis = ~np.isnan(a.obs[:, int(MT.Azimuth), 0])
        epochs.append(ep_all[vis]); names += [name] * int(vis.sum()); obs.append(a.obs[vis])
    epochs = np.concatenate(epochs); obs = np.concatenate(obs)
    order = np.argsort(epochs, kind="stable")
    epochs, names, obs = epochs[order], [names[j] for j in order], obs[order]
    proc = dsn(0.0, ANG, {t: 1e-6 for t in ALL})
    cov = np.diag([1e-3, 1e-3, 1e-3, 1e-6, 1e-6, 1e-6, 0.0, 0.0, 0.0])
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.DeviationTracking, None, proc, None, msr_size=2)
    cap = len(ep_all) + len(epochs)
    first = odp.process_arcs([nb.KfEstimate.from_covar(truth0, cov)], nb.TrackingDataArc(epochs, names, obs, ALL), estimates_capacity=cap)
    assert first.status[0] == 0 and (first.msr_flags[:, 0] == abi.MSRF_PROCESSED).all()
    obs = obs.copy()
    obs[:, 2:, :] = obs[:, 2:, :] - first.prefit[:, :2, :]
    L = first.n_estimates(0)
    truth_at = {int(e): first.records["nominal"][k, :, 0].copy() for k, e in enumerate(first.records["epoch"][:L, 0])}
    arc = nb.TrackingDataArc(epochs, names, np.repeat(obs, n, axis=2), ALL)
    ests = [nb.KfEstimate.from_covar(truth0, cov) for _ in range(n)]
    return odp, arc, ests, truth_at, cap


def test_od_tb_val_az_el_ckf_fixed_step_perfect_stations():
    """The reference's bounds on STRICT: deviation, prefit and postfit below 1e-12, covariance diagonal norm below 1e-6, final state
    equal to the truth; after smooth(): deviation below 1e-12, covariance below 1e-4, within 1e-9 km and 1e-9 km/s of the truth."""
    odp, arc, ests, truth_at, cap = _perfect_stations(4)
    sol = odp.process_arcs(ests, arc, estimates_capacity=cap)
    assert (sol.status == 0).all() and sol.records["count"].max() <= cap
    for i in range(4):
        L = sol.n_estimates(i)
        assert np.linalg.norm(sol.records["deviation"][:L, :, i], axis=1).max() < 1e-12
        for r in sol.residuals(i):
            if r is not None:
                assert np.linalg.norm(r[0]) < 1e-12 and np.linalg.norm(r[1]) < 1e-12
        last = sol.estimate(L - 1, i)
        assert np.linalg.norm(np.diag(last.covar)) < 1e-6
        yf = truth_at[last.nominal_state.epoch()]
        assert np.abs(last.state().to_vector()[:6] - yf[:6]).max() <= 2 * np.finfo(float).eps * np.abs(yf[:6]).max()
    sm = sol.smooth()
    for i in range(4):
        assert sm.error(i) is None
        est = sm.estimate(sm.n_estimates(i) - 1, i)
        assert np.linalg.norm(est.state_deviation) < 1e-12
        assert np.linalg.norm(np.diag(est.covar)) < 1e-4
        y, yf = est.state().to_vector(), truth_at[est.nominal_state.epoch()]
        assert np.linalg.norm(y[:3] - yf[:3]) < 1e-9 and np.linalg.norm(y[3:6] - yf[3:6]) < 1e-9
    print(f"AZ-EL-CKF: {len(arc)} measurements, final covariance diagonal norm "
          f"{np.linalg.norm(np.diag(sol.estimate(sol.n_estimates(0) - 1, 0).covar)):.3e}")
