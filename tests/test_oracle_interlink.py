"""The interlink restatement (tests/interlink_oracle.py) on the CPU: the reference's as-coded quirks, the window's outcomes and the C
ABI's struct and argument checks (no launch is reached)."""
import ctypes as C
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import interlink_oracle as io
from tests import interlink_util as iu

S = 10**9


@pytest.fixture(scope="module")
def sc():
    return iu.scenario(n=2, n_msr=120, degree=0)


def _dev(sc, types=(MT.Range, MT.Doppler), radius=None):
    d = iu.device(sc["traj"], types).to_c(0, iu.FRAME)
    if radius is not None:
        d.body_radius_km = radius
    return d


def _visible_k(sc):
    return [k for k in range(len(sc["arc"])) if not np.isnan(sc["arc"].obs[k, 0, 0])]


def test_doppler_ignores_transmitter_velocity(sc):
    """The computed Doppler is rho . v_rx / |rho|, against an independent formula; the true range rate (v_rx - v_tx) differs."""
    for k in _visible_k(sc)[::7]:
        t = int(sc["arc"].epoch_ns[k])
        y = sc["truth"][k, :, 0]
        tx = io.tx_state(sc["traj"], t)
        rng, rr = io.computed(tx, y)
        u = (y[:3] - tx[:3]) / np.linalg.norm(y[:3] - tx[:3])
        assert rng == pytest.approx(np.linalg.norm(y[:3] - tx[:3]), rel=1e-14)
        assert rr == pytest.approx(float(u @ y[3:6]), rel=1e-12, abs=1e-15)
        assert abs(rr - float(u @ (y[3:6] - tx[3:6]))) > 1e-4          # the transmitter's velocity matters, and is left out


def _true(tx, y):
    d, dv = y[:3] - tx[:3], y[3:6] - tx[3:6]
    r = np.linalg.norm(d)
    return r, float(d @ dv) / r


def test_rows_against_central_differences(sc):
    """At the observed values equal to the true ones, the rows are the central differences of the true range and range rate; the
    Doppler row differs from the differences of the as-coded computed Doppler by the v_tx / rho terms."""
    k = _visible_k(sc)[3]
    t = int(sc["arc"].epoch_ns[k])
    y = np.concatenate([sc["truth"][k, :, 0], [1.0, 0.0, 50.0]])
    tx = io.tx_state(sc["traj"], t)
    rng, rr = _true(tx, y)
    o = np.array([rng, rr])
    hr, hd = np.array(io.h_row(abi.MSR_RANGE, tx, y, o)), np.array(io.h_row(abi.MSR_DOPPLER, tx, y, o))
    fr, fd, fc = np.zeros(9), np.zeros(9), np.zeros(9)
    for j in range(6):
        h = 1e-3 if j < 3 else 1e-6
        yp, ym = y.copy(), y.copy()
        yp[j] += h
        ym[j] -= h
        fr[j] = (_true(tx, yp)[0] - _true(tx, ym)[0]) / (2 * h)
        fd[j] = (_true(tx, yp)[1] - _true(tx, ym)[1]) / (2 * h)
        fc[j] = (io.computed(tx, yp)[1] - io.computed(tx, ym)[1]) / (2 * h)
    assert np.allclose(hr, fr, rtol=0, atol=1e-8)            # the differences of a 40 000 km range round at about 1e-9
    assert np.allclose(hd, fd, rtol=0, atol=1e-9)
    rho = y[:3] - tx[:3]
    gap = hd[:3] - fc[:3]
    assert np.abs(gap).max() > 1e-6
    assert np.allclose(gap, -(tx[3:6] - (float(rho @ tx[3:6]) / rng ** 2) * rho) / rng, rtol=0, atol=1e-9)


def test_windows_msr_size_1_and_2(sc):
    k = _visible_k(sc)[0]
    t = int(sc["arc"].epoch_ns[k])
    o, y = sc["arc"].obs[k, :, 0], sc["truth"][k, :, 0]
    d = _dev(sc)
    w2 = io.window(d, sc["traj"], 2, 0, o, t, t, y)
    assert w2[0] == [abi.MSR_RANGE, abi.MSR_DOPPLER] and io.window(d, sc["traj"], 2, 1, o, t, t, y) == "empty"
    for wno, typ in ((0, abi.MSR_RANGE), (1, abi.MSR_DOPPLER)):
        w1 = io.window(d, sc["traj"], 1, wno, o, t, t, y)
        assert w1[0] == [typ] and np.array_equal(w1[3][0], w2[3][wno]) and w1[5][0] == w2[5][wno]
    assert io.window(d, sc["traj"], 1, 2, o, t, t, y) == "empty"
    short = _dev(sc, (MT.Doppler,))                          # one type at msr_size 2: an identity row and a zero R entry
    ws = io.window(short, sc["traj"], 2, 0, o, t, t, y)
    assert ws[0] == [abi.MSR_DOPPLER] and np.array_equal(ws[3][1], np.eye(2, 9)[1]) and ws[4][1] == 0.0


def test_outside_recording_is_a_status_and_precedes_obstruction(sc):
    """An epoch outside the recording is TX_NO_DATA, not 'not visible', even when the Moon blocks the link; a missing range for a
    Doppler row is NO_RANGE, also when blocked: h_tilde runs first."""
    blocked = [k for k in range(len(sc["arc"])) if np.isnan(sc["arc"].obs[k, 0, 0])]
    assert blocked
    k = blocked[0]
    t = int(sc["arc"].epoch_ns[k])
    y = sc["truth"][k, :, 0]
    tx = io.tx_state(sc["traj"], t)
    o = np.array(io.computed(tx, y))
    d = _dev(sc)
    assert io.window(d, sc["traj"], 2, 0, o, t, t, y) == "not_visible"
    late = int(sc["traj"].epochs_ns[-1]) + 1
    assert io.window(d, sc["traj"], 2, 0, o, late, late, y) == io.TX_NO_DATA
    assert io.window(d, sc["traj"], 2, 0, o, t, late, y) == io.TX_NO_DATA           # the computed observation's epoch alone
    assert io.window(d, sc["traj"], 2, 0, np.array([np.nan, o[1]]), t, t, y) == io.NO_RANGE


def test_obstruction_across_the_limb(sc):
    """Moving the receiver across the Moon's limb as seen from the transmitter flips the link at the radius."""
    t = int(sc["traj"].epochs_ns[5])
    tx = io.tx_state(sc["traj"], t)
    u = tx[:3] / np.linalg.norm(tx[:3])
    side = np.cross(u, [1.0, 0.0, 0.0])
    side /= np.linalg.norm(side)                             # the receiver at h from the centre, square to the transmitter's direction:
    R = 1737.4                                               # the link passes the centre at h (1 - h^2 / 2|r_tx|^2), within 1 km of h
    y_near = np.concatenate([(R + 2.0) * side, [0.0] * 3])
    y_far = np.concatenate([(R - 2.0) * side, [0.0] * 3])
    assert not io.obstructed(tx, y_near, R) and io.obstructed(tx, y_far, R)
    assert not io.obstructed(tx, y_far, -1.0)                # radius <= 0: no test


def test_filter_restatement_runs(sc):
    """The restated filter over the arc: exactly the measurements the Moon blocks are flagged, the others processed."""
    prop = nb.Propagator.new(sc["dyn"], nb.IntegratorMethod.DormandPrince78, sc["opts"])
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, sc["devices"], None)
    sc = dict(sc, arc=nb.TrackingDataArc(sc["arc"].epoch_ns, sc["arc"].tracker, sc["arc"].obs.copy()))
    arc = sc["arc"]
    blocked = np.isnan(arc.obs[:, 0, 0])
    for k in np.nonzero(blocked)[0]:                         # data where the Moon blocks the link: the filter's test flags them
        tx = io.tx_state(sc["traj"], int(arc.epoch_ns[k]))
        arc.obs[k, :, 0] = io.computed(tx, sc["truth"][k, :, 0])
    r = iu.oracle_run(sc, odp, 0)
    assert np.array_equal(r["flags"] == abi.MSRF_NOT_VISIBLE, blocked)
    assert r["status"] == 0
    assert (r["flags"] == abi.MSRF_NOT_VISIBLE).any() and (r["flags"] == abi.MSRF_PROCESSED).any()
    assert np.array_equal(r["flags"] == abi.MSRF_PROCESSED, ~blocked) and np.isfinite(r["state"]).all()


def test_struct_size_and_null_arguments():
    assert C.sizeof(abi.InterlinkTxC) == 56
    lib = abi.load_library()
    cfg = abi.OdConfigC(variant=0, msr_size=2, max_step_ns=60 * S, epoch_precision_ns=1000)
    dev = (abi.InterlinkTxC * 1)()
    dev[0].n_types, dev[0].types[0], dev[0].types[1] = 2, abi.MSR_RANGE, abi.MSR_DOPPLER
    ep = np.array([1, 2], dtype=np.int64) * S
    trk = np.zeros(2, dtype=np.int32)
    obs = np.zeros((2, 2, 1))
    arc = abi.TrackingArcC(2, ep.ctypes.data, trk.ctypes.data, obs.ctypes.data)
    x = np.zeros(81)
    out = abi.OdOutputsC(x.ctypes.data, x.ctypes.data, x.ctypes.data, None, None, None, None, None, None, None, None, x.ctypes.data)
    tep, tst, tcnt = np.zeros(3, dtype=np.int64), np.zeros(18), np.array([3], dtype=np.int64)
    sink = abi.TrajSink(3, tep.ctypes.data, tst.ctypes.data, tcnt.ctypes.data)
    call = lambda eng=None, s=C.byref(sink), n_tx=1, d=dev: lib.nyxb_od_interlink_batch(  # noqa: E731
        eng, C.byref(cfg), 1, d, n_tx, s, C.byref(arc), 1, x.ctypes.data, x.ctypes.data, x.ctypes.data, x.ctypes.data, C.byref(out), None)
    assert call() == -1                                      # NULL engine (the other refusals need an engine: tests/test_gpu_interlink.py)
    smooth = lib.nyxb_od_interlink_smooth_batch(None, C.byref(cfg), 1, dev, 1, C.byref(sink), C.byref(arc), 1, None, None, None)
    assert smooth == -1


def test_interlink_c_refusals_need_no_engine(sc):
    """The packing checks of the host layer that mirror NYXB_RC_BAD_ARG."""
    with pytest.raises(nb.ODError):
        iu.device(sc["traj"], (MT.Range, MT.Range)).to_c(0, iu.FRAME)
    with pytest.raises(nb.ODError):
        iu.device(sc["traj"], (MT.Azimuth,)).to_c(0, iu.FRAME)
    assert math.isclose(_dev(sc).body_radius_km, 1737.4)
