"""The position-fix filter (nyxb_od_position_batch) and its smoother on the GPU, against the restatement (tests/position_oracle.py),
on the three kernel families; the reference's GPS test restated; a consistency check of the filter without an oracle."""
import numpy as np
import pytest
from scipy import stats

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import position_oracle as po
from tests.position_util import gps_scenario, oracle_run, ric_error_m, scenario

pytestmark = pytest.mark.gpu
S = 10**9
FAMILIES = ("STRICT", "FAST-thread", "FAST-coop")
TOL = {"STRICT": (1e-9, 1e-12), "FAST-thread": (1e-6, 1e-9), "FAST-coop": (1e-6, 1e-9)}   # km, km/s


def process(sc, family, variant=nb.KalmanVariant.ReferenceUpdate, msr_size=3, reject=None, snc=None, method=None, cap=None):
    mode = nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST
    prop = nb.Propagator.new(sc["dyn"], method or nb.IntegratorMethod.DormandPrince78, sc["opts"], mode=mode)
    prop.engine(sc["frame"], None).set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    odp = nb.KalmanODProcess(prop, variant, nb.SigmaRejection(reject) if reject else None, sc["devices"], None, msr_size=msr_size)
    if snc is not None:
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12] * 3, 10 * nb.Unit.Minute, snc))
    return odp, odp.process_arcs(sc["ests"], sc["arc"], estimates_capacity=cap)


def check(sc, odp, sol, family, filters=None, rel=False):
    """Parity with the restatement.  STRICT also needs equal step counts.  rel: bounds relative to the state's size (for the
    inconsistent [Y, X, Z] model, whose updates are large)."""
    tr, tv = TOL[family]
    for i in (filters if filters is not None else range(len(sc["ests"]))):
        ref = oracle_run(sc, odp, i)
        sr, sv = (tr * np.abs(ref["state"][:3]).max(), tv * np.abs(ref["state"][3:6]).max()) if rel else (tr, tv)
        assert sol.status[i] == ref["status"]
        if family == "STRICT":
            assert sol.details["n_steps"][i] == ref["n_steps"]
        assert np.abs(sol.final_state_soa[:3, i] - ref["state"][:3]).max() < sr
        assert np.abs(sol.final_state_soa[3:6, i] - ref["state"][3:6]).max() < sv
        assert np.allclose(sol.covar[i], ref["covar"], rtol=1e-6, atol=1e-15)
        assert np.array_equal(sol.msr_flags[:, i], ref["flags"])
        for f in ("prefit", "postfit", "resid_ratio"):
            g, r = getattr(sol, f)[:, :, i], ref[f]
            assert np.array_equal(np.isnan(g), np.isnan(r)), f
            assert np.allclose(np.nan_to_num(g), np.nan_to_num(r), rtol=1e-5, atol=10 * sr), f


VARIANTS = {
    "ekf-m3": dict(),
    "ckf-m3-ric": dict(variant=nb.KalmanVariant.DeviationTracking, snc=nb.LocalFrame.RIC),
    "ekf-m1-inertial": dict(msr_size=1, snc=nb.LocalFrame.Inertial),
    "ckf-m1": dict(variant=nb.KalmanVariant.DeviationTracking, msr_size=1),
    "ekf-m3-reject": dict(reject=3.0),
}


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("name", list(VARIANTS))
def test_parity(family, name):
    sc = scenario()
    odp, sol = process(sc, family, **VARIANTS[name])
    assert sol.status.tolist() == [0] * 4
    check(sc, odp, sol, family)


@pytest.mark.parametrize("family", FAMILIES)
def test_parity_edges(family):
    """a constant bias (stays in the prefit), absent components, an unknown tracker, two devices, fixed steps, at msr_size 1.  At
    msr_size 3 the second device, which carries two types, leaves a zero row and a zero R entry: SingularNoiseRk at its first fix."""
    sc = scenario(bias=0.05, two_devices=True, fixed=True, seed=4)
    sc["arc"].obs[3, 1, :] = np.nan
    sc["arc"].obs[5, :, 1] = np.nan
    sc["arc"].tracker[7] = "nobody"
    for M in (1, 3):
        odp, sol = process(sc, family, msr_size=M, reject=200.0)
        check(sc, odp, sol, family)
        if M == 3:
            assert (sol.status == 1).all()
        else:
            assert (sol.status == 0).all()
            assert sol.msr_flags[5, 1] == abi.MSRF_ABSENT and sol.msr_flags[7, 0] == 0


@pytest.mark.parametrize("family", FAMILIES)
def test_parity_edges_msr_size_3(family):
    """msr_size 3 with one device: a bias that stays in the prefit, an absent component (zero H row, R kept, prefit minus the
    computed observation), an all-absent fix and an unknown tracker, all updates accepted; then the [Y, X, Z] order, whose computed
    observation disagrees with H."""
    sc = scenario(bias=0.02, fixed=True, seed=6)
    sc["arc"].obs[2, 1, :] = np.nan
    sc["arc"].obs[4, :, 0] = np.nan
    sc["arc"].tracker[6] = "nobody"
    odp, sol = process(sc, family)
    check(sc, odp, sol, family)
    assert (sol.status == 0).all() and not (sol.msr_flags & abi.MSRF_REJECTED).any()
    assert sol.msr_flags[4, 0] == abi.MSRF_ABSENT and sol.msr_flags[6, 0] == 0
    # the absent Y of fix 2: zero H row and zero real observation, so its prefit is minus the computed observation (the nominal y)
    assert (np.abs(sol.prefit[2, 1, :]) > 1000.0).all() and np.isfinite(sol.postfit[2, 1, :]).all()
    scy = scenario(types=(MT.Y, MT.X, MT.Z), n_msr=4, seed=7)
    odp, sol = process(scy, family)
    check(scy, odp, sol, family, rel=True)


def _smooth_restated(rec, i, dev_c, M, arc_obs, tracker):
    """ODSolution::smooth of filter i from its records (smooth.rs:104-249), and its recomputed postfit through the position window."""
    L = int(rec["count"][i])
    out = []
    for k in range(L - 1):
        phi = rec["stm"][k + 1, :, i].reshape(9, 9).T
        Pi = np.linalg.inv(phi)
        xs = Pi @ rec["deviation"][k + 1, :, i]
        Ps = Pi @ rec["covar"][k + 1, :, i].reshape(9, 9).T @ Pi.T
        ys = rec["nominal"][k, :, i] + xs
        ys[6] = min(max(ys[6], 0.0), 2.0)
        post = np.full(3, np.nan)
        tg = int(rec["tag"][k + 1, i])
        if tg >= 0:
            mk, w, _, _ = abi.od_pos_tag_fields(tg)
            win = po.window(dev_c[tracker[mk]], M, w, arc_obs[mk, :, i], ys)
            cur, _, real, _, _, comp = win
            for q in range(len(cur)):
                post[w * M + q] = real[q] - comp[q]
        out.append((ys, Ps, post))
    return out


@pytest.mark.parametrize("family", FAMILIES)
def test_records_smoothing_and_batch_invariance(family):
    sc = scenario()
    for M in (3, 1):
        odp, plain = process(sc, family, msr_size=M)
        _, rec = process(sc, family, msr_size=M, cap=200)
        for f in ("final_state_soa", "covar", "prefit", "postfit", "resid_ratio", "msr_flags", "status"):
            assert np.array_equal(getattr(plain, f), getattr(rec, f), equal_nan=True), f
        R = rec.records
        tr = TOL[family][0]
        for i in range(2):
            sink = []
            oracle_run(sc, odp, i, sink=sink)
            L = len(sink)
            assert R["count"][i] == L
            assert [int(t) for t in R["tag"][:L, i]] == [e["tag"] for e in sink]
            assert [int(t) for t in R["epoch"][:L, i]] == [e["epoch"] for e in sink]
            for k, e in enumerate(sink):
                assert np.abs(R["nominal"][k, :3, i] - e["nominal"][:3]).max() < tr
                assert np.abs(R["deviation"][k, :3, i] - e["deviation"][:3]).max() < tr
                assert np.allclose(R["covar"][k, :, i].reshape(9, 9).T, e["covar"], rtol=1e-6, atol=1e-15)
                stm = R["stm"][k, :, i].reshape(9, 9).T
                assert np.abs(stm - e["stm"]).max() < 1e-7 * np.abs(e["stm"]).max()
        sm = rec.smooth()
        assert (sm.smoother["status"] == 0).all()
        _, dev_c = odp.position_devices_c()
        tracker = np.zeros(len(sc["arc"]), dtype=np.int32)
        for i in range(2):
            want = _smooth_restated(R, i, dev_c, M, sc["arc"].obs, tracker)
            for k, (ys, Ps, post) in enumerate(want):
                assert np.abs(sm.smoother["state"][k, :3, i] - ys[:3]).max() < 1e-7
                assert np.allclose(sm.smoother["covar"][k, :, i].reshape(9, 9).T, Ps, rtol=1e-6, atol=1e-14)
                g = sm.smoother["postfit"][k, :, i]
                assert np.array_equal(np.isnan(g), np.isnan(post)), (k, g, post)
                assert np.allclose(np.nan_to_num(g), np.nan_to_num(post), rtol=1e-6, atol=1e-9)
    # one filter alone gives the same bits as in the batch (plain: the msr_size 1 run of the last pass)
    sc1 = dict(sc, ests=sc["ests"][2:3], arc=nb.TrackingDataArc(sc["arc"].epoch_ns, sc["arc"].tracker, sc["arc"].obs[:, :, 2:3],
                                                                 sc["arc"].types))
    _, one = process(sc1, family, msr_size=1)
    assert np.array_equal(one.final_state_soa[:, 0], plain.final_state_soa[:, 2])
    assert np.array_equal(one.covar[0], plain.covar[2])


def test_null_optional_outputs():
    """ratio, prefit, postfit, flags, state_dev, details NULL: the required outputs are the same bits."""
    import ctypes as C

    sc = scenario()
    odp, full = process(sc, "STRICT")
    eng = odp.prop.engine(sc["frame"], None)
    names, dev_c = odp.position_devices_c()
    from nyx_b200.cosmic import pack_spacecraft
    st, cs, ep = pack_spacecraft([e.nominal_state for e in sc["ests"]])
    n, arc = len(sc["ests"]), sc["arc"]
    cov = np.empty((81, n))
    for i, e in enumerate(sc["ests"]):
        cov[:, i] = np.asarray(e.covar).reshape(9, 9).T.reshape(81)
    tr = np.zeros(len(arc), dtype=np.int32)
    obs = np.ascontiguousarray(arc.obs)
    carc = abi.PositionArcC(len(arc), arc.epoch_ns.ctypes.data, tr.ctypes.data, obs.ctypes.data)
    out_state, out_epoch, out_cov = np.empty((9, n)), np.empty(n, dtype=np.int64), np.empty((81, n))
    status = np.zeros(n, dtype=np.int32)
    out = abi.OdOutputsC(out_state.ctypes.data, out_epoch.ctypes.data, out_cov.ctypes.data, None, None, None, None, None, None, None,
                         None, status.ctypes.data)
    rc = eng._lib.nyxb_od_position_batch(eng._h, C.byref(odp.config_c()), 1, dev_c, C.byref(carc), n, st.ctypes.data, cs.ctypes.data,
                                         ep.ctypes.data, cov.ctypes.data, C.byref(out), None)
    assert rc == 0
    assert np.array_equal(out_state, full.final_state_soa) and np.array_equal(status, full.status)
    assert np.array_equal(out_cov.T.reshape(n, 9, 9).transpose(0, 2, 1), full.covar)


def test_msr_size_2_is_singular_noise():
    sc = scenario()
    _, sol = process(sc, "STRICT", msr_size=2)
    assert (sol.status == 1).all()


def test_argument_checks():
    sc = scenario(n=1)
    prop = nb.Propagator.new(sc["dyn"], nb.IntegratorMethod.DormandPrince78, sc["opts"], mode=nb.MODE_STRICT)
    eng = prop.engine(sc["frame"], None)
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, sc["devices"], None, msr_size=3)
    names, dev_c = odp.position_devices_c()
    from nyx_b200.cosmic import pack_spacecraft
    st, cs, ep = pack_spacecraft([e.nominal_state for e in sc["ests"]])
    cov = np.asarray(sc["ests"][0].covar).reshape(81, 1)
    arc = sc["arc"]
    tr = np.zeros(len(arc), dtype=np.int32)

    def run(cfg, devs):
        return eng.od_position_batch(cfg, 1, devs, arc.epoch_ns, tr, arc.obs, st, cs, ep, cov)
    for bad in ([abi.MSR_RANGE, abi.MSR_Y, abi.MSR_Z], [abi.MSR_X, abi.MSR_X, abi.MSR_Z]):
        d = (abi.PositionDeviceC * 1)(); d[0] = dev_c[0]
        for q in range(3):
            d[0].types[q] = bad[q]
        with pytest.raises(nb.PropagationError, match="rc=-1"):
            run(odp.config_c(), d)
    d = (abi.PositionDeviceC * 1)(); d[0] = dev_c[0]; d[0].n_types = 4
    with pytest.raises(nb.PropagationError, match="rc=-1"):
        run(odp.config_c(), d)
    cfg = odp.config_c(); cfg.msr_size = 4
    with pytest.raises(nb.PropagationError, match="rc=-1"):
        run(cfg, dev_c)
    with pytest.raises(nb.ODError):
        nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None,
                           dict(sc["devices"], dss=nb.GroundStation.dss65_madrid(0.0, nb.StochasticNoise(1e-3), nb.StochasticNoise(1e-6))),
                           None, msr_size=3).process_arcs(sc["ests"], arc)


def test_reference_gps_position_filtering():
    """gps_position.rs restated over 16 noise streams (the reference's stream, seed 12345 of its own generator, cannot be reproduced).
    As the reference, the error is that of the LAST ESTIMATE's nominal state (the pre-update nominal of the last fix) against the
    truth, in RIC.  The reference asserts < 0.1 m for its one stream.  At the end of the arc the per-axis sigma is about
    1 m x 2 / sqrt(360) = 0.1 m, so a 3-D error below 0.1 m is roughly a one-in-five draw; over these streams the errors spread
    from 0.1 to 0.35 m, consistent with the filter's own covariance (test_consistency_mean_nees), so the spread is asserted:
    median below 0.25 m and every stream below 0.5 m.  The same scenario runs on the CPU restatement (tests/test_host_position.py)."""
    sc = gps_scenario(16)
    _, sol = process(sc, "STRICT", method=nb.IntegratorMethod.RungeKutta89, cap=800)
    assert (sol.status == 0).all()
    truth = sc["truth"][-1, :3, 0]
    errs = [ric_error_m(sc, sol.records["nominal"][sol.n_estimates(i) - 1, :, i], truth) for i in range(16)]
    print("GPS final RIC position error over 16 noise seeds [m]: min %.4f median %.4f max %.4f" % (min(errs), np.median(errs), max(errs)))
    assert np.median(errs) < 0.25 and max(errs) < 0.5


def test_consistency_mean_nees():
    """1 024 filters, initial errors drawn from P0, independent noise: the mean NEES of the final position must lie in the two-sided
    99.9 % interval of chi2(3 * 1024) / 1024."""
    n = 1024
    sc = scenario(n=n, n_msr=60, degree=0, seed=11)
    _, sol = process(sc, "FAST-thread")
    assert (sol.status == 0).all()
    truth = sc["truth"][-1, :3, 0]
    e = sol.final_state_soa[:3, :] - truth[:, None]
    nees = np.array([e[:, i] @ np.linalg.solve(sol.covar[i][:3, :3], e[:, i]) for i in range(n)])
    lo, hi = stats.chi2.ppf(0.0005, 3 * n) / n, stats.chi2.ppf(0.9995, 3 * n) / n
    print(f"mean NEES {nees.mean():.4f} in [{lo:.4f}, {hi:.4f}]")
    assert lo <= nees.mean() <= hi
