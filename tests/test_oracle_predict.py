"""Covariance mapping (`KalmanODProcess::predict_until`, od/process/mod.rs:440-486) without a GPU: the oracle restatement
(tests/predict_oracle.py) reproduces the reference's quirks and an independent chain of per-chunk STM propagations; the host
mirror (`predict_*`, `PredictionSolution`, `to_parquet`) runs on an oracle-backed stand-in of the engine; the C ABI rejects bad
arguments before any device work."""
import ctypes as C
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi

from .od_util import S

MS = 60 * S   # KalmanODProcess.max_step default


@pytest.fixture(scope="module")
def po(oracle):
    from . import predict_oracle

    return predict_oracle


def _setup(stepping="fixed", degree=4):
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    if stepping == "fixed":
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(10.0))
    else:   # adaptive, starting from a 5 s step (not max_step): predict_until does not call set_step
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions(init_step=5 * S))
    orbit = nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame)
    sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    est = nb.KfEstimate.from_diag(sc, [1.0, 0.5, 0.25, 1e-6, 2e-6, 3e-6, 0.0, 0.0, 0.0])
    est.covar[0, 4] = est.covar[4, 0] = 1e-4
    return dict(frame=frame, dyn=dyn, prop=prop, sc=sc, est=est, dyn_c=dyn.pack(frame, None).c, opts_c=prop.opts.to_c(prop.method))


def _consts(sc):
    return np.array([sc.mass.dry_mass_kg, sc.mass.extra_mass_kg, sc.srp.area_m2, sc.drag.area_m2])


def _cfg(prop, variant=nb.KalmanVariant.DeviationTracking, snc=None, max_step=MS):
    odp = nb.KalmanODProcess(prop, variant, None, {}, None)
    odp.max_step = max_step
    if snc is not None:
        odp.with_process_noise(snc)
    return odp, odp.config_c()


def _run(po, s, cfg, end, dev0=None):
    e = s["est"]
    return po.predict_until(s["dyn_c"], s["opts_c"], cfg, e.nominal_state.to_vector(), _consts(e.nominal_state), e.nominal_state.epoch(),
                            e.covar, end, dev0)


@pytest.mark.parametrize("end_s,count,last_s", [(600, 11, 600), (630, 12, 660), (0, 2, 60), (-5, 2, 60), (1e-9, 2, 60), (59, 2, 60),
                                                (61, 3, 120)])
def test_record_count_epochs_and_overshoot(po, end_s, count, last_s):
    s = _setup()
    _, cfg = _cfg(s["prop"])
    end = int(round(end_s * S))
    r = _run(po, s, cfg, end)
    assert r["status"] == 0 and r["count"] == count == 1 + max(1, math.ceil(end / MS))
    assert np.array_equal(r["rec_epoch"], np.arange(count, dtype=np.int64) * MS)   # record k at epoch0 + k max_step, exactly
    assert r["epoch"] == last_s * S and 0 <= r["epoch"] - max(end, 0) < MS or end <= 0
    assert np.array_equal(r["rec_covar"][0], s["est"].covar)                          # record 0 = the initial estimate
    assert np.array_equal(r["rec_state"][0], s["est"].nominal_state.to_vector())


def test_no_set_step_first_chunk_starts_from_init_step(po, oracle):
    s = _setup("adaptive")
    _, cfg = _cfg(s["prop"])
    e = s["est"].nominal_state
    r = _run(po, s, cfg, 10 * MS)

    def chain(set_step):
        inst = oracle.Inst(s["dyn_c"], s["opts_c"], e.to_vector(), _consts(e), 0)
        if set_step:
            inst.set_step(MS, False)
        for _ in range(10):
            assert inst.for_duration(MS) == 0
            y, ep, *_ = inst.get()
            y[9:] = np.eye(9).reshape(81)
            inst.set(y, ep)
        y, ep, _, _, det = inst.get()
        return y[:9], int(det["n_steps"])

    y0, n0 = chain(False)
    y1, n1 = chain(True)
    assert np.array_equal(r["state"], y0) and r["n_steps"] == n0
    assert n1 != n0   # process_arc's set_step(max_step) would have changed the step sequence


def _snc_q(dt_s, diag):
    g = np.zeros((9, 3))
    for i in range(3):
        g[i, i] = dt_s ** 2 / 2.0
        g[i + 3, i] = dt_s
    return g @ np.diag(diag) @ g.T


def test_chain_of_oracle_stm_propagations(po, oracle):
    """Record k = an independent numpy chain over per-chunk STM propagations of the oracle: P <- Phi P Phi^T + Q, x <- Phi x."""
    s = _setup()
    q = np.array([1e-10, 2e-10, 3e-10])
    _, cfg = _cfg(s["prop"], snc=nb.ProcessNoise3D.from_diagonal(q, 3600 * S))
    dev0 = np.array([0.1, -0.2, 0.05, 1e-4, 0.0, -1e-4, 0.0, 0.0, 0.0])
    r = _run(po, s, cfg, 5 * MS, dev0)
    e = s["est"].nominal_state
    st, cs, ep = nb.pack_spacecraft([e])
    P, x = s["est"].covar.copy(), dev0.copy()
    for k in range(1, r["count"]):
        st, ep, stm, _, status = oracle.propagate_batch_stm(s["dyn_c"], s["opts_c"], st, cs, ep, int(ep[0]) + MS)
        assert status[0] == 0 and ep[0] == k * MS
        Phi = stm[:, 0].reshape(9, 9).T
        P = Phi @ P @ Phi.T + _snc_q(60.0, q)
        x = Phi @ x
        assert np.allclose(r["rec_covar"][k], P, rtol=1e-12, atol=1e-14 * np.abs(P).max())
        want = st[:, 0] + x
        assert np.allclose(r["rec_state"][k], want, rtol=1e-14, atol=1e-12)


@pytest.mark.parametrize("frame", [None, nb.LocalFrame.RIC])
@pytest.mark.parametrize("disable_s", [3600, 30])
def test_snc_frames_and_disable_time(po, frame, disable_s):
    s = _setup()
    q = np.array([1e-8, 4e-8, 9e-8])
    _, cfg0 = _cfg(s["prop"])
    _, cfg = _cfg(s["prop"], snc=nb.ProcessNoise3D.from_diagonal(q, disable_s * S, frame))
    r0, r = _run(po, s, cfg0, 2 * MS), _run(po, s, cfg, 2 * MS)
    dq = r["rec_covar"][1] - r0["rec_covar"][1]
    if disable_s < 60:
        assert np.array_equal(dq, np.zeros((9, 9)))     # the time since the previous estimate exceeds disable_time: no SNC
        return
    qq = q
    if frame == nb.LocalFrame.RIC:                     # snc.rs:226-247: rotate, keep the diagonal only
        y = r0["rec_state"][1]                          # the nominal state of the first time update (zero deviation)
        D = nb.od.dcm_ric_to_inertial(nb.Orbit(*y[:6], 0, s["frame"]))
        qq = np.diag(D @ np.diag(q) @ D.T)
    assert np.allclose(dq, _snc_q(60.0, qq), rtol=1e-9, atol=1e-20)


def test_ckf_deviation_is_mapped_and_ekf_deviation_is_zero(po, oracle):
    s = _setup()
    dev0 = np.array([0.1, -0.2, 0.05, 1e-4, 0.0, -1e-4, 0.0, 0.0, 0.0])
    _, ckf = _cfg(s["prop"], nb.KalmanVariant.DeviationTracking)
    _, ekf = _cfg(s["prop"], nb.KalmanVariant.ReferenceUpdate)
    rc, re = _run(po, s, ckf, MS, dev0), _run(po, s, ekf, MS, dev0)
    e = s["est"].nominal_state
    st, cs, ep = nb.pack_spacecraft([e])
    _, _, stm, _, _ = oracle.propagate_batch_stm(s["dyn_c"], s["opts_c"], st, cs, ep, MS)
    Phi = stm[:, 0].reshape(9, 9).T
    assert np.allclose(rc["state_dev"], Phi @ dev0, rtol=1e-14, atol=1e-16)
    assert np.array_equal(re["state_dev"], np.zeros(9))
    assert np.array_equal(re["rec_state"][1], re["state"])
    assert np.array_equal(rc["rec_state"][0], e.to_vector() + dev0) and np.array_equal(re["rec_state"][0], e.to_vector() + dev0)
    assert np.array_equal(rc["rec_covar"][1], re["rec_covar"][1])


def test_cr_is_clamped_in_the_records(po):
    s = _setup()
    _, cfg = _cfg(s["prop"])
    dev0 = np.zeros(9)
    dev0[6] = 5.0
    r = _run(po, s, cfg, MS, dev0)
    assert r["rec_state"][0][6] == 2.0 and r["rec_state"][1][6] == 2.0


# --------------------------------------------------------------------------- host mirror on an oracle-backed engine
class _OracleEngine:
    """Stands in for nyx_b200.Engine: `od_predict_batch` runs the oracle restatement run by run and packs what the C ABI returns."""

    def __init__(self, po, dyn_c, opts_c):
        self.po, self.dyn_c, self.opts_c = po, dyn_c, opts_c
        self.calls = []

    def od_predict_batch(self, cfg, st, cs, ep, end, cov0, dev0=None, capacity=0, record_states=True, record_covars=True):
        n = st.shape[1]
        self.calls.append(dict(end=end.copy(), dev0=None if dev0 is None else dev0.copy(), capacity=capacity))
        K = int(capacity)
        out = dict(state=np.empty((9, n)), epoch=np.empty(n, dtype=np.int64), covar=np.empty((n, 9, 9)), dev=np.empty((9, n)),
                   count=np.empty(n, dtype=np.int64), rs=np.full((K, 9, n), np.nan), rc=np.full((K, 81, n), np.nan))
        for i in range(n):
            r = self.po.predict_until(self.dyn_c, self.opts_c, cfg, st[:, i], cs[:, i], ep[i], cov0[:, i].reshape(9, 9).T, end[i],
                                      None if dev0 is None else dev0[:, i])
            out["state"][:, i], out["epoch"][i], out["covar"][i], out["dev"][:, i] = r["state"], r["epoch"], r["covar"], r["state_dev"]
            out["count"][i] = r["count"]
            k = min(K, r["count"])
            out["rs"][:k, :, i] = r["rec_state"][:k]
            out["rc"][:k, :, i] = r["rec_covar"][:k].transpose(0, 2, 1).reshape(k, 81)
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        return nb.PredictionSolution(out["state"], out["epoch"], out["covar"], out["dev"], details, np.zeros(n, dtype=np.int32),
                                     out["count"], out["rs"] if record_states else None, out["rc"] if record_covars else None,
                                     np.asarray(ep, dtype=np.int64).copy(), int(cfg.max_step_ns))


class _OracleProp:
    def __init__(self, eng):
        self.eng = eng

    def engine(self, frame, almanac):
        return self.eng


def _mirror(po, variant=nb.KalmanVariant.DeviationTracking):
    s = _setup()
    eng = _OracleEngine(po, s["dyn_c"], s["opts_c"])
    odp = nb.KalmanODProcess(_OracleProp(eng), variant, None, {}, None)
    odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-10, 1e-10, 1e-10], 3600 * S, nb.LocalFrame.RIC))
    return s, eng, odp


def test_predict_methods_pack_the_ensemble(po):
    s, eng, odp = _mirror(po)
    e0 = s["est"]
    e1 = nb.KfEstimate(e0.nominal_state.with_vector(30 * S, e0.nominal_state.to_vector()), e0.covar * 2.0, np.arange(9) * 1e-3)
    sol = odp.predict_ensemble_for([e0, e1], 5 * MS + 1)
    call = eng.calls[-1]
    assert call["end"].tolist() == [5 * MS + 1, 30 * S + 5 * MS + 1]       # end_i = epoch0_i + duration
    assert np.array_equal(call["dev0"][:, 1], np.arange(9) * 1e-3) and call["capacity"] == 7
    assert sol.rec_count.tolist() == [7, 7] and sol.final_epoch_ns.tolist() == [6 * MS, 30 * S + 6 * MS]
    assert np.array_equal(sol.record_epochs(1), 30 * S + np.arange(7) * MS)
    assert np.array_equal(sol.record_covar(0, 1), e1.covar)
    fe = sol.final_estimate(1)
    assert fe.nominal_state.epoch() == 30 * S + 6 * MS and np.array_equal(fe.covar, sol.covar[1])
    assert np.array_equal(fe.state_deviation, sol.state_deviation[:, 1])
    # the single-estimate forms
    one = odp.predict_until(e0, 2 * MS)
    assert one.rec_count.tolist() == [3] and np.array_equal(one.rec_state[:, :, 0], sol.rec_state[:3, :, 0])
    assert odp.predict_for(e1, 2 * MS).final_epoch_ns[0] == 30 * S + 2 * MS
    few = odp.predict_until(e0, 5 * MS, capacity=2)
    assert few.rec_count[0] == 6 and few.stored(0) == 2 and few.record_epochs(0).tolist() == [0, MS]


def test_to_parquet_columns_and_values(po, tmp_path):
    pq = pytest.importorskip("pyarrow.parquet")
    s, eng, odp = _mirror(po)
    sol = odp.predict_until(s["est"], 3 * MS)
    path = sol.to_parquet(tmp_path / "pred.parquet")
    tab = pq.read_table(str(path))
    names = tab.column_names
    fr = s["frame"].name
    assert names[0] == "Epoch (UTC)" and tab.num_rows == 4
    cov_cols = [c for c in names if c.startswith("Covariance ")]
    assert len(cov_cols) == 45 and cov_cols[0] == f"Covariance X*X ({fr}) (km^2)" and f"Covariance X*Vy ({fr}) (km^2/s)" in cov_cols
    assert f"Covariance Vx*Mass ({fr}) (km/s*kg)" in cov_cols and f"Covariance Cr*Cd ({fr}) (unitless)" in cov_cols
    sig = [f"Sigma {it} ({fr}) ({u})" for it, u in zip(("X", "Y", "Z", "Vx", "Vy", "Vz", "Cr", "Cd", "Mass"),
                                                          ("km", "km", "km", "km/s", "km/s", "km/s", "unitless", "unitless", "kg"))]
    ric = ["Sigma X (RIC) (km)", "Sigma Y (RIC) (km)", "Sigma Z (RIC) (km)", "Sigma Vx (RIC) (km/s)", "Sigma Vy (RIC) (km/s)",
           "Sigma Vz (RIC) (km/s)"]
    for c in sig + ric + ["Whitened residual #0", "Whitened residual #1", "Residual ratio", "Residual Rejected", "Tracker",
                          "Gain X*[0]", "Gain Mass*[1]", "Filter-smoother ratio X (km^2)", "Filter-smoother ratio Mass (km*kg)"]:
        assert c in names, c
    assert names.index(sig[0]) > names.index(cov_cols[-1]) and names.index(ric[0]) == names.index(sig[-1]) + 1
    for c in ("Residual ratio", "Tracker", "Gain X*[0]", "Filter-smoother ratio Vz (km^2/s)"):
        assert tab[c].null_count == 4
    # one covariance entry and one RIC sigma by hand, at record 2
    P2 = sol.record_covar(2, 0)
    assert tab[f"Covariance X*Vy ({fr}) (km^2/s)"].to_pylist()[2] == P2[0, 4]
    assert tab[sig[1]].to_pylist()[2] == math.sqrt(P2[1, 1])
    y = sol.rec_state[2, :, 0]
    r, v = y[:3], y[3:6]
    rh = r / np.linalg.norm(r)
    ch = np.cross(r, v) / np.linalg.norm(np.cross(r, v))
    ih = np.cross(ch, rh)
    D = np.column_stack([rh, ih, ch])                                # RIC -> inertial
    want = math.sqrt((D @ P2[3:6, 3:6] @ D.T)[1, 1])                  # as coded: D C D^T, rate block zero
    assert tab["Sigma Vy (RIC) (km/s)"].to_pylist()[2] == pytest.approx(want, rel=1e-13)
    # state columns: the estimate's state (nominal + deviation)
    assert tab["X (km)"].to_pylist()[2] == y[0] and tab["VX (km/s)"].to_pylist()[2] == y[3]


def test_to_random_variable():
    sc = nb.Spacecraft(orbit=nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, nb.EARTH_J2000))
    cov = np.diag([1.0, 2.0, 3.0, 1e-6, 2e-6, 3e-6, 0.0, 0.0, 0.0])
    est = nb.KfEstimate(sc, cov, np.arange(9) * 0.01)
    mvn = est.to_random_variable()
    assert isinstance(mvn, nb.MvnSpacecraft) and mvn.template is sc
    assert np.array_equal(mvn.mean, np.arange(9) * 0.01)
    ss = mvn.sqrt_s_v
    assert np.allclose(ss @ ss.T, cov, atol=1e-15)


def test_abi_rejects_bad_arguments():
    lib = abi.load_library()
    assert lib.nyxb_od_predict_batch(None, None, 1, None, None, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
    cfg = abi.OdConfigC()
    cfg.variant = abi.KF_DEVIATION_TRACKING
    for bad in (0, -MS):
        cfg.max_step_ns = bad
        assert lib.nyxb_od_predict_batch(None, C.byref(cfg), 1, None, None, None, None, None, None, None) == -1
        assert b"max_step" in lib.nyxb_last_error()
    cfg.max_step_ns = MS
    cfg.variant = 7
    assert lib.nyxb_od_predict_batch(None, C.byref(cfg), 1, None, None, None, None, None, None, None) == -1
    assert b"variant" in lib.nyxb_last_error()
    cfg.variant = abi.KF_REFERENCE_UPDATE
    st = np.zeros((9, 1)); cs = np.zeros((4, 1)); ep = np.zeros(1, dtype=np.int64); cov = np.zeros((81, 1))
    assert lib.nyxb_od_predict_batch(None, C.byref(cfg), 1, st.ctypes.data, cs.ctypes.data, ep.ctypes.data, ep.ctypes.data,
                                     cov.ctypes.data, None, None) == -1                      # NULL outputs
    assert b"null" in lib.nyxb_last_error()


def test_predict_outputs_layout():
    assert C.sizeof(abi.PredictOutputsC) == 80
    assert abi.PredictOutputsC.capacity.offset == 48
