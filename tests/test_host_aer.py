"""The Python host layer of angle tracking on the CPU: KalmanODProcess.process_arcs over stations with azimuth and elevation, the
per-estimate accessors (residuals, RMS statistics), smooth(), the parquet export and round trip, and the dispatch and its errors, on an
oracle-backed engine stand-in whose od_aer_batch / od_aer_smooth_batch run the restatement (tests/aer_oracle.py) one filter after the
other."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import AER_TYPES
from nyx_b200.od import MeasurementType as MT
from tests import aer_oracle as ao
from tests.aer_util import dsn, truth_states
from tests.test_host_position import stack
from tests.util import OracleEngine

S = 10**9


class AerOracleEngine(OracleEngine):
    def od_aer_batch(self, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns, covar0_soa,
                     record_estimates=False, estimates_capacity=None):
        from nyx_b200.od import ODSolution

        self.launches += 1
        n, m = state_soa.shape[1], len(msr_epoch_ns)
        out_state = np.empty((9, n)); out_epoch = np.empty(n, dtype=np.int64); covar = np.empty((n, 9, 9)); dev = np.empty((9, n))
        ratio, prefit, postfit = (np.full((m, 4, n), np.nan) for _ in range(3))
        flags = np.zeros((m, n), dtype=np.int32)
        est_state = np.full((m, 9, n), np.nan) if record_estimates else None
        est_cov = np.full((m, 9, n), np.nan) if record_estimates else None
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE); status = np.zeros(n, dtype=np.int32)
        streams = []
        for i in range(n):
            sink = []
            r = ao.process_arc(self.packed.c, self.opts, cfg_c, list(stations_c)[:n_stations], msr_epoch_ns, np.asarray(msr_tracker),
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

    def od_aer_smooth_batch(self, cfg_c, n_stations, stations_c, msr_tracker, obs, records, filter_status, outputs=None):
        cap, n = records["epoch"].shape
        r = {k: np.full((cap, rows, n), np.nan) for k, rows in (("state", 9), ("deviation", 9), ("covar", 81), ("fs_ratio", 9), ("postfit", 4))}
        r["status"] = np.asarray(filter_status, dtype=np.int32).copy()
        for i in range(n):
            if r["status"][i]:
                continue
            for k, (ys, Ps, post) in enumerate(ao.smooth_restated(records, i, list(stations_c)[:n_stations], self.packed.c, cfg_c.msr_size,
                                                                  obs, np.asarray(msr_tracker))):
                r["state"][k, :, i], r["covar"][k, :, i], r["postfit"][k, :, i] = ys, Ps.T.reshape(81), post
        return r


def setup(oracle, monkeypatch, msr_size=2, types=(MT.Range, MT.Doppler, MT.Azimuth, MT.Elevation), n=2, n_msr=12):
    frame = nb.EARTH_J2000
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions.default(), mode=nb.MODE_STRICT)
    eng = {}

    def engine(fr, alm):
        return eng.setdefault(fr, AerOracleEngine(oracle, prop, fr, alm))
    monkeypatch.setattr(prop, "engine", engine)
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame), mass=nb.Mass(500.0, 0.0, 0.0))
    epochs = (np.arange(1, n_msr + 1) * 60 * S).astype(np.int64)
    truth = np.repeat(truth_states(dyn, frame, truth0, epochs)[:, :, None], n, axis=2)
    devices = dsn(-90.0, types)
    names = list(devices)
    arc = nb.simulate_tracking(epochs, truth, devices, [names[k % 3] for k in range(n_msr)], frame, None, np.random.default_rng(1))
    rng = np.random.default_rng(2)
    ests = []
    for _ in range(n):
        v = truth0.to_vector()
        v[:3] += rng.normal(0, 0.1, 3)
        ests.append(nb.KfEstimate.from_diag(truth0.with_vector(0, v), [0.01] * 3 + [1e-8] * 3 + [0.0] * 3))
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, devices, None, msr_size=msr_size)
    return odp, arc, ests


@pytest.mark.parametrize("msr_size", [1, 2])
def test_residuals_rms_and_smooth_decode_aer_tags(oracle, monkeypatch, msr_size):
    """Records carry NYXB_OD_POS_TAG; the ratio of window w is in slot w; smooth() puts each recomputed postfit at its measurement and
    window."""
    odp, arc, ests = setup(oracle, monkeypatch, msr_size=msr_size)
    assert arc.is_aer and arc.obs.shape == (12, 4, 2)
    sol = odp.process_arcs(ests, arc, estimates_capacity=200)
    assert (sol.status == 0).all()
    W = 4 // msr_size
    for i in range(2):
        got = [r for r in sol.residuals(i) if r is not None]
        want = [(sol.prefit[k, w * msr_size:(w + 1) * msr_size, i], sol.postfit[k, w * msr_size:(w + 1) * msr_size, i], sol.resid_ratio[k, w, i])
                for k in range(len(arc)) for w in range(W)]
        assert len(got) == len(want) == len(arc) * W
        for g, w in zip(got, want):
            assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]) and g[2] == w[2] and np.isfinite(g[2])
        L = sol.n_estimates(i)
        assert sol.rms_prefit_residuals(i) == pytest.approx(np.sqrt(sum(float(w[0] @ w[0]) for w in want) / L), rel=1e-15)
        assert sol.rms_residual_ratios(i) == pytest.approx(np.sqrt(sum(w[2] ** 2 for w in want) / L), rel=1e-15)
    sm = sol.smooth()
    for i in range(2):
        for p in range(sol.n_estimates(i) - 1):
            tag = int(sol.records["tag"][p + 1, i])
            if tag >= 0:
                mk, w, _, _ = abi.od_pos_tag_fields(tag)
                sl = slice(w * msr_size, (w + 1) * msr_size)
                assert np.array_equal(sm.postfit[mk, sl, i], sm.smoother["postfit"][p, sl, i], equal_nan=True)
        assert np.isfinite(sm.rms_postfit_residuals(i))


def test_tracking_arc_parquet_round_trip_and_default_reader(oracle, monkeypatch, tmp_path):
    _, arc, _ = setup(oracle, monkeypatch, n=1)
    arc.obs[4, :, 0] = np.nan
    arc.obs[6, int(MT.Doppler), 0] = np.nan
    arc.to_parquet(tmp_path / "a.parquet")
    names = pq.read_table(str(tmp_path / "a.parquet")).column_names
    assert names == ["Epoch (UTC)", "Tracking device", "Range (km)", "Doppler (km/s)", "Azimuth (deg)", "Elevation (deg)"]
    back = nb.TrackingDataArc.from_parquet(tmp_path / "a.parquet", types=AER_TYPES)
    keep = np.arange(len(arc)) != 4
    assert back.types == AER_TYPES and np.array_equal(back.epoch_ns, arc.epoch_ns[keep])
    assert np.array_equal(back.obs[:, :, 0], arc.obs[keep, :, 0], equal_nan=True)
    # the default reader keeps today's behaviour: range and Doppler only
    rd = nb.TrackingDataArc.from_parquet(tmp_path / "a.parquet")
    assert rd.types == (MT.Range, MT.Doppler) and np.array_equal(rd.obs[:, :, 0], arc.obs[keep, :2, 0], equal_nan=True)
    tab = pq.read_table(str(tmp_path / "a.parquet")).select(["Epoch (UTC)", "Tracking device", "Azimuth (deg)"])
    pq.write_table(tab, str(tmp_path / "az.parquet"))
    with pytest.raises(nb.ODError, match="Range"):
        nb.TrackingDataArc.from_parquet(tmp_path / "az.parquet")
    az = nb.TrackingDataArc.from_parquet(tmp_path / "az.parquet", types=AER_TYPES)
    assert np.isnan(az.obs[:, [0, 1, 3], 0]).all() and np.array_equal(az.obs[:, 2, 0], arc.obs[keep, 2, 0])
    pq.write_table(pa.table({"Epoch (UTC)": tab["Epoch (UTC)"], "Tracking device": tab["Tracking device"], "X (km)": tab["Azimuth (deg)"]}),
                   str(tmp_path / "x.parquet"))
    with pytest.raises(nb.ODError):
        nb.TrackingDataArc.from_parquet(tmp_path / "x.parquet", types=AER_TYPES)


def test_solution_parquet_angle_columns(oracle, monkeypatch, tmp_path):
    odp, arc, ests = setup(oracle, monkeypatch, types=(MT.Elevation, MT.Range, MT.Azimuth))
    sol = odp.process_arcs(ests, arc, estimates_capacity=200)
    tab = pq.read_table(str(sol.to_parquet(tmp_path / "s.parquet", index=1)))
    assert "Prefit residual: Azimuth (deg)" in tab.column_names and "Postfit residual: Elevation (deg)" in tab.column_names
    el = np.array([np.nan if v is None else v for v in tab["Prefit residual: Elevation (deg)"].to_pylist()])
    # list [El, R, Az] at msr_size 2: window 0 holds El in slot 0; window 1 holds Az alone
    want = np.array([r[0][0] if r is not None and int(sol.records["tag"][p, 1]) >> 3 & 3 == 0 else np.nan
                     for p, r in enumerate(sol.residuals(1))])
    assert np.array_equal(el, want, equal_nan=True)
    sol2 = odp.process_arcs(ests, arc, record_estimates=True)
    t2 = pq.read_table(str(sol2.to_parquet(tmp_path / "p.parquet", index=0)))
    rows = np.nonzero(sol2.msr_flags[:, 0] & abi.MSRF_PROCESSED)[0]
    assert np.array_equal(np.array(t2["Postfit residual: Azimuth (deg)"].to_pylist(), dtype=float), sol2.postfit[rows, 2, 0], equal_nan=True)


def test_dispatch_and_errors(oracle, monkeypatch):
    odp, arc, ests = setup(oracle, monkeypatch, n=1)
    eng = odp.prop.engine(nb.EARTH_J2000, None)
    odp.process_arcs(ests, arc)
    assert eng.launches == 1
    arc2 = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc.obs[:, :2])
    with pytest.raises(nb.ODError, match="AER_TYPES"):
        odp.process_arcs(ests, arc2)
    with pytest.raises(nb.ODError):
        nb.BatchLeastSquares(odp.prop, odp.devices, None)
    rd = dsn(-90.0, (MT.Range, MT.Doppler))
    with pytest.raises(nb.ODError):
        nb.BatchLeastSquares(odp.prop, rd, None).estimate(ests[0].nominal_state, arc)
    with pytest.raises(nb.ODError):
        nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc.obs[:, :3], AER_TYPES)
    with pytest.raises(nb.ODError):
        dsn(0.0)["Madrid"].with_msr_type(MT.X, nb.StochasticNoise(1.0)).to_aer_c(nb.EARTH_J2000, None)


def test_simulate_tracking_slots():
    """Without angles the simulator's arc is unchanged (two slots); with them it has four, slot = type."""
    frame = nb.EARTH_J2000
    y = np.zeros((3, 6, 1))
    y[:, 0, 0], y[:, 4, 0] = 7000.0, 7.5
    ep = np.array([1, 2, 3], dtype=np.int64) * 60 * S
    a2 = nb.simulate_tracking(ep, y, dsn(-90.0, (MT.Range, MT.Doppler)), ["Madrid"] * 3, frame, None)
    a4 = nb.simulate_tracking(ep, y, dsn(-90.0, (MT.Elevation, MT.Range)), ["Madrid"] * 3, frame, None)
    assert a2.types == (MT.Range, MT.Doppler) and a2.obs.shape == (3, 2, 1)
    assert a4.types == AER_TYPES and a4.obs.shape == (3, 4, 1) and np.isnan(a4.obs[:, [1, 2], 0]).all()
    assert np.array_equal(a4.obs[:, 0, 0], a2.obs[:, 0, 0]) and (np.abs(a4.obs[:, 3, 0]) <= 90.0).all()
