"""The host layer of interlink tracking on the CPU: InterlinkTxSpacecraft, its packing and recordings, the ODErrors of the unsupported
options, the kind checks of KalmanODProcess and BatchLeastSquares, simulate_interlink, and the solution's "Tracker" names."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import interlink_oracle as io
from tests import interlink_util as iu

S = 10**9


@pytest.fixture(scope="module")
def traj():
    return iu.record(iu.dynamics(0), iu.nrho_orbit(), 30 * 60 * S, name="NRHO Tx SC")


def test_name(traj):
    assert iu.device(traj).name() == "NRHO Tx SC"
    anon = nb.Traj(traj.template, traj.epochs_ns, traj.states)
    assert iu.device(anon).name() == "unnamed"


def test_to_c_and_odeerrors(traj):
    d = iu.device(traj, (MT.Doppler, MT.Range), sigma=(2e-3, 3e-6), bias=0.25).to_c(3, iu.FRAME)
    assert (d.tx, d.n_types, list(d.types)) == (3, 2, [abi.MSR_DOPPLER, abi.MSR_RANGE])
    assert list(d.noise_var) == [3e-6 ** 2, 2e-3 ** 2] and list(d.bias) == [0.25, 0.25] and d.body_radius_km == 1737.4
    for kw in ({"integration_time": 60 * S}, {"ab_corr": "LT"}):
        dev = iu.device(traj)
        for k, v in kw.items():
            setattr(dev, k, v)
        with pytest.raises(nb.ODError):
            dev.to_c(0, iu.FRAME)
    with pytest.raises(nb.ODError, match="trajectory is in Moon J2000"):
        iu.device(traj).to_c(0, nb.EARTH_J2000)
    with pytest.raises(nb.ODError, match="NoiseNotConfigured"):
        nb.InterlinkTxSpacecraft(traj, [MT.Range], {}).to_c(0, iu.FRAME)


def test_sink_columns_shared(traj):
    other = iu.record(iu.dynamics(0), iu.llo_orbit(), 10 * 60 * S)
    devices = {"a": iu.device(traj), "b": iu.device(other), "c": iu.device(traj)}
    odp = nb.KalmanODProcess(nb.Propagator.default(iu.dynamics(0)), nb.KalmanVariant.ReferenceUpdate, None, devices, None)
    assert odp.is_interlink and not odp.is_position
    names, arr, (sink, n_tx, (ep, st, cnt)) = odp.interlink_c(iu.FRAME)
    assert names == ["a", "b", "c"] and [arr[i].tx for i in range(3)] == [0, 1, 0] and n_tx == 2
    assert sink.capacity == len(traj) and list(cnt) == [len(traj), len(other)]
    assert np.array_equal(ep[:len(other), 1], other.epochs_ns) and np.array_equal(st[:, :len(traj), 0], traj.states[:, :6].T)


def test_kinds_and_bls(traj):
    gs = nb.GroundStation.dss65_madrid(0.0, nb.StochasticNoise(1e-3), nb.StochasticNoise(1e-6))
    prop = nb.Propagator.default(iu.dynamics(0))
    mixed = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, {"tx": iu.device(traj), "gs": gs}, None)
    with pytest.raises(nb.ODError, match="mixed"):
        mixed.is_interlink
    with pytest.raises(nb.ODError, match="interlink"):
        nb.BatchLeastSquares(prop, {"tx": iu.device(traj)}, None)


def test_simulate_interlink_geometry(traj):
    """simulate_interlink's values are the restatement's computed observation plus the seeded noise, NaN where the Moon blocks."""
    truth_tr = iu.record(iu.dynamics(0), iu.llo_orbit(), 25 * 60 * S)
    epochs = (np.arange(1, 25) * 60 * S).astype(np.int64)
    truth = np.stack([truth_tr.at(int(e)).orbit.to_cartesian_pos_vel() for e in epochs])[:, :, None]
    dev = {"tx": iu.device(traj)}
    clean = nb.simulate_interlink(epochs, truth, dev, ["tx"] * len(epochs), iu.FRAME)
    assert clean.types == (MT.Range, MT.Doppler) and clean.obs.shape == (24, 2, 1)
    for k, e in enumerate(epochs):
        tx = io.tx_state(traj, int(e))
        if io.obstructed(tx, truth[k, :, 0], 1737.4):
            assert np.isnan(clean.obs[k, :, 0]).all()
        else:
            assert tuple(clean.obs[k, :, 0]) == pytest.approx(io.computed(tx, truth[k, :, 0]), rel=1e-14, abs=1e-16)
    noisy = nb.simulate_interlink(epochs, truth, dev, ["tx"] * len(epochs), iu.FRAME, np.random.default_rng(0))
    vis = ~np.isnan(clean.obs[:, 0, 0])
    assert np.abs(noisy.obs[vis, 0, 0] - clean.obs[vis, 0, 0]).max() < 6e-3


def test_tracker_name_is_device_name(traj):
    sol = nb.ODSolution(*([None] * 12), devices={"key": iu.device(traj)})
    assert sol._tracker_name("key") == "NRHO Tx SC" and sol._tracker_name("other") == "other"
    assert "ODTrajError" in nb.ODSolution(*([None] * 11), np.array([abi.ERR_TX_NO_DATA])).error(0)
    assert "Range" in nb.ODSolution(*([None] * 11), np.array([abi.ERR_NO_RANGE])).error(0)
