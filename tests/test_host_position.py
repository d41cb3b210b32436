"""The Python host layer of the position-fix filter on the CPU: KalmanODProcess.process_arcs with position devices, the per-estimate
accessors (residuals, RMS statistics), record_estimates, and the parquet export / round trip, on an oracle-backed engine stand-in
whose od_position_batch runs the restatement (tests/position_oracle.py) one filter after the other."""
import numpy as np
import pyarrow.parquet as pq
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import position_oracle as po
from tests.util import OracleEngine

S = 10**9


class PositionOracleEngine(OracleEngine):
    def od_position_batch(self, cfg_c, n_devices, devices_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns, covar0_soa,
                          record_estimates=False, estimates_capacity=None):
        from nyx_b200.od import ODSolution

        self.launches += 1
        n, m = state_soa.shape[1], len(msr_epoch_ns)
        out_state = np.empty((9, n)); out_epoch = np.empty(n, dtype=np.int64); covar = np.empty((n, 9, 9)); dev = np.empty((9, n))
        ratio = np.full((m, 3, n), np.nan); prefit = np.full((m, 3, n), np.nan); postfit = np.full((m, 3, n), np.nan)
        flags = np.zeros((m, n), dtype=np.int32)
        est_state = np.full((m, 9, n), np.nan) if record_estimates else None
        est_cov = np.full((m, 9, n), np.nan) if record_estimates else None
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE); status = np.zeros(n, dtype=np.int32)
        streams = []
        for i in range(n):
            sink = []
            r = po.process_arc(self.packed.c, self.opts, cfg_c, list(devices_c)[:n_devices], msr_epoch_ns, np.asarray(msr_tracker),
                               np.ascontiguousarray(obs[:, :, i]), state_soa[:, i].copy(), consts_soa[:, i].copy(), int(epoch0_ns[i]),
                               covar0_soa[:, i].reshape(9, 9).T, sink=sink)
            streams.append(sink)
            out_state[:, i], out_epoch[i], covar[i], dev[:, i] = r["state"], r["epoch"], r["covar"], r["state_dev"]
            ratio[:, :, i], prefit[:, :, i], postfit[:, :, i], flags[:, i] = r["resid_ratio"], r["prefit"], r["postfit"], r["flags"]
            if record_estimates:
                est_state[:, :, i], est_cov[:, :, i] = r["est_state"], r["est_covar_diag"]
            details["n_steps"][i], status[i] = r["n_steps"], r["status"]
        records = None if estimates_capacity is None else stack(streams, int(estimates_capacity))
        return ODSolution(out_state, out_epoch, covar, dev, ratio, prefit, postfit, flags, est_state, est_cov, details, status,
                          records=records)


def stack(streams, cap):
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


def setup(oracle, monkeypatch, msr_size=3, types=(MT.Y, MT.X, MT.Z), n=2, n_msr=12):
    frame = nb.EARTH_J2000
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions.default(), mode=nb.MODE_STRICT)
    eng = {}

    def engine(fr, alm):
        return eng.setdefault(fr, PositionOracleEngine(oracle, prop, fr, alm))
    monkeypatch.setattr(prop, "engine", engine)
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame), mass=nb.Mass(500.0, 0.0, 0.0))
    epochs = (np.arange(1, n_msr + 1) * 60 * S).astype(np.int64)
    st, cs, ep = nb.pack_spacecraft([truth0])
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(dyn.pack(frame, None).c, nb.IntegratorOptions.with_fixed_step_s(10.0).to_c(
        nb.IntegratorMethod.RungeKutta89), st, cs, ep, int(epochs[-1]), traj_capacity=n_msr * 6 + 2)
    truth = np.repeat(t_st[:, np.searchsorted(t_ep[: t_cnt[0], 0], epochs), 0].T[:, :, None], n, axis=2)
    dev = nb.PositionDevice("gnss")
    for t in types:
        dev.with_noise(t, nb.StochasticNoise(1e-3))
    arc = nb.simulate_position_fixes(epochs, truth, {"gnss": dev}, ["gnss"] * n_msr, np.random.default_rng(1))
    rng = np.random.default_rng(2)
    ests = []
    for _ in range(n):
        v = truth0.to_vector()
        v[:3] += rng.normal(0, 0.1, 3)
        ests.append(nb.KfEstimate.from_diag(truth0.with_vector(0, v), [0.01] * 3 + [1e-8] * 3 + [0.0] * 3))
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, {"gnss": dev}, None, msr_size=msr_size)
    return odp, arc, ests


@pytest.mark.parametrize("msr_size", [1, 3])
def test_residuals_and_rms_decode_position_tags(oracle, monkeypatch, msr_size):
    odp, arc, ests = setup(oracle, monkeypatch, msr_size=msr_size, types=(MT.X, MT.Y, MT.Z))
    sol = odp.process_arcs(ests, arc, estimates_capacity=200)
    assert (sol.status == 0).all()
    for i in range(2):
        res = sol.residuals(i)
        assert len(res) == sol.n_estimates(i)
        got = [(r[0].copy(), r[1].copy(), r[2]) for r in res if r is not None]
        want = []
        for k in range(len(arc)):
            for w in range(3 // msr_size):
                sl = list(range(w * msr_size, (w + 1) * msr_size))
                want.append((sol.prefit[k, sl, i], sol.postfit[k, sl, i], sol.resid_ratio[k, w if msr_size == 1 else 0, i]))
        assert len(got) == len(want) == len(arc) * (3 // msr_size)
        for g, w in zip(got, want):
            assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]) and g[2] == w[2]
        L = sol.n_estimates(i)
        pre2 = sum(float(w[0] @ w[0]) for w in want)
        assert sol.rms_prefit_residuals(i) == pytest.approx(np.sqrt(pre2 / L), rel=1e-15)
        assert sol.rms_postfit_residuals(i) == pytest.approx(np.sqrt(sum(float(w[1] @ w[1]) for w in want) / L), rel=1e-15)
        assert sol.rms_residual_ratios(i) == pytest.approx(np.sqrt(sum(w[2] ** 2 for w in want) / L), rel=1e-15)


def test_record_estimates(oracle, monkeypatch):
    odp, arc, ests = setup(oracle, monkeypatch)
    sol = odp.process_arcs(ests, arc, record_estimates=True)
    assert np.isfinite(sol.est_state).all() and np.array_equal(sol.est_state[-1], sol.final_state_soa)


def test_tracking_arc_parquet_round_trip(oracle, monkeypatch, tmp_path):
    _, arc, _ = setup(oracle, monkeypatch, types=(MT.X, MT.Z))
    arc.obs[4, :, 0] = np.nan
    arc.to_parquet(tmp_path / "a.parquet")
    names = pq.read_table(str(tmp_path / "a.parquet")).column_names
    assert names == ["Epoch (UTC)", "Tracking device", "X (km)", "Z (km)"]
    back = nb.TrackingDataArc.from_parquet(tmp_path / "a.parquet")
    assert back.types == (MT.X, MT.Y, MT.Z) and back.obs.shape == (len(arc) - 1, 3, 1)
    keep = np.arange(len(arc)) != 4
    assert np.array_equal(back.epoch_ns, arc.epoch_ns[keep])
    assert np.array_equal(back.obs[:, :, 0], arc.obs[keep, :, 0], equal_nan=True)


def test_solution_parquet_position_columns(oracle, monkeypatch, tmp_path):
    odp, arc, ests = setup(oracle, monkeypatch)
    sol = odp.process_arcs(ests, arc, estimates_capacity=200)
    sol.to_parquet(tmp_path / "s.parquet", index=1)
    tab = pq.read_table(str(tmp_path / "s.parquet"))
    assert "Prefit residual: X (km)" in tab.column_names and "Prefit residual: Range (km)" not in tab.column_names
    res = [r for r in sol.residuals(1)]
    pre_y = np.array([np.nan if v is None else v for v in tab["Prefit residual: Y (km)"].to_pylist()])
    # device list [Y, X, Z]: the Y column holds slot 0 of every measurement update
    want = np.array([r[0][0] if r is not None else np.nan for r in res])
    assert np.array_equal(pre_y, want, equal_nan=True)
    sol2 = odp.process_arcs(ests, arc, record_estimates=True)
    sol2.to_parquet(tmp_path / "p.parquet", index=0)
    t2 = pq.read_table(str(tmp_path / "p.parquet"))
    z = np.array(t2["Postfit residual: Z (km)"].to_pylist(), dtype=float)
    assert np.array_equal(z, sol2.postfit[:, 2, 0])


def test_reference_gps_scenario_on_the_restatement(oracle):
    """The reference's gps_position.rs scenario on the CPU restatement over 16 noise streams, the last estimate's nominal state
    against the truth in RIC (the bound and why: tests/test_gpu_position.py::test_reference_gps_position_filtering)."""
    from tests.position_util import gps_errors_restatement

    errs = gps_errors_restatement(16)
    print("GPS on the restatement [m]:", np.round(sorted(errs), 3))
    assert np.median(errs) < 0.25 and max(errs) < 0.5, errs
