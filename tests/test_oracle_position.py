"""CPU checks of the position-fix filter (PositionDevice): the reference's quirks as the restatement (tests/position_oracle.py) codes
them, the 3x3 ratio and gain against numpy, record tags, the host-side types and the C ABI's argument checks."""
import ctypes as C
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import PositionDevice, StochasticNoise, TrackingDataArc, simulate_position_fixes
from tests import position_oracle as po

X, Y, Z = nb.od.MeasurementType.X, nb.od.MeasurementType.Y, nb.od.MeasurementType.Z
Y9 = np.array([7000.0, -1200.0, 300.0, 1.0, 7.2, 0.3, 1.8, 2.2, 50.0])


def dev(types, sig=1e-3, bias=0.0):
    d = PositionDevice("gnss")
    for t in types:
        d.with_noise(t, StochasticNoise(sig, bias))
    return d.to_c()


def test_computed_observation_is_the_list_position_and_the_bias_cancels():
    d = dev([Y, X, Z], bias=0.25)
    cur, avail, real, H, Rk, comp = po.window(d, 3, 0, np.array([1.0, 2.0, 3.0]), Y9)
    assert cur == [abi.MSR_Y, abi.MSR_X, abi.MSR_Z] and all(avail)
    assert np.array_equal(comp, [((Y9[i] + 0.0) + 0.25) - 0.25 for i in range(3)])   # list position ii -> component ii
    assert np.array_equal(real, [2.0, 1.0, 3.0])                                       # observation by type
    # H by type: the Y row differentiates component 1 although comp[0] is component 0
    assert np.array_equal(H[:, :3], [[0, 1, 0], [1, 0, 0], [0, 0, 1]]) and not H[:, 3:].any()
    assert np.array_equal(Rk, [1e-6] * 3)


def test_absent_type_keeps_zero_row_and_its_variance():
    d = dev([X, Y, Z])
    cur, avail, real, H, Rk, comp = po.window(d, 3, 0, np.array([1.0, np.nan, 3.0]), Y9)
    assert avail == [True, False, True]
    assert not H[1].any() and real[1] == 0.0 and Rk[1] == 1e-6
    assert real[1] - comp[1] == -Y9[1]
    assert po.window(d, 3, 0, np.array([np.nan] * 3), Y9) == "unavailable"


@pytest.mark.parametrize("M,n_types,windows", [(3, 3, 1), (1, 3, 3), (2, 3, 2), (1, 2, 2), (3, 2, 1)])
def test_window_counts(M, n_types, windows):
    d = dev([X, Y, Z][:n_types])
    got = 0
    for wno in range(n_types // M + 1):
        w = po.window(d, M, wno, np.array([1.0, 2.0, 3.0]), Y9)
        if w == "empty":
            break
        got += 1
    assert got == windows


def test_msr_size_2_second_window_is_singular():
    d = dev([X, Y, Z])
    _, _, real, H, Rk, comp = po.window(d, 2, 1, np.array([1.0, 2.0, 3.0]), Y9)
    assert not H[1].any() and Rk[1] == 0.0
    P = np.eye(9)
    S = H @ P @ H.T + np.diag(Rk)
    assert po.ratio(2, S, Rk, real - comp) is None                     # SingularNoiseRk


def test_zero_variance_is_singular():
    d = dev([X, Y, Z], sig=0.0)
    _, _, real, H, Rk, comp = po.window(d, 3, 0, np.array([1.0, 2.0, 3.0]), Y9)
    S = H @ np.zeros((9, 9)) @ H.T + np.diag(Rk)
    assert po.ratio(3, S, Rk, real - comp) is None


def test_ratio_and_gain_3x3_against_numpy():
    rng = np.random.default_rng(3)
    for _ in range(50):
        A = rng.normal(size=(9, 9))
        P = A @ A.T
        H = np.zeros((3, 9)); H[0, 1] = H[1, 0] = H[2, 2] = 1.0
        Rk = rng.uniform(1e-4, 1e-2, 3)
        S = H @ P @ H.T + np.diag(Rk)
        pre = rng.normal(size=3)
        L = np.linalg.cholesky(S)
        want = math.sqrt(float(np.linalg.solve(L, pre) @ np.linalg.solve(L, pre)) / 3)
        assert po.ratio(3, S, Rk, pre) == pytest.approx(want, rel=1e-12)
        K = po.gain(3, S, P @ H.T)
        assert np.allclose(K, P @ H.T @ np.linalg.inv(S), rtol=1e-10, atol=1e-12)
    # not positive definite: ratio from R, gain from the closed-form inverse
    S = np.array([[1.0, 2.0, 0.0], [2.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    assert po.chol3(S) is None
    Rk = np.array([4.0, 9.0, 1.0])
    assert po.ratio(3, S, Rk, np.array([2.0, 3.0, 1.0])) == pytest.approx(1.0)
    assert np.allclose(po.gain(3, S, np.eye(9, 3)), np.eye(9, 3) @ np.linalg.inv(S))
    assert po.gain(3, np.zeros((3, 3)), np.eye(9, 3)) is None


def test_pos_tags_round_trip():
    for k, w, rej, M in [(0, 0, 0, 1), (5, 2, 1, 1), (123456, 1, 0, 2), (7, 0, 1, 3)]:
        t = abi.od_pos_tag(k, w, rej, M)
        assert abi.od_pos_tag_fields(t) == (k, w, rej, M)


def test_simulator_value_is_list_position_plus_bias():
    d = PositionDevice("gnss").with_noise(Y, StochasticNoise(0.0, 0.5)).with_noise(X, StochasticNoise(0.0, 0.0))
    truth = np.array([[[1.0], [2.0], [3.0], [0.0], [0.0], [0.0]]])
    arc = simulate_position_fixes([10], truth, {"gnss": d}, ["gnss"])
    assert arc.types == (X, Y, Z) and arc.obs.shape == (1, 3, 1)
    assert arc.obs[0, 1, 0] == 1.5 and arc.obs[0, 0, 0] == 2.0 and np.isnan(arc.obs[0, 2, 0])


def test_host_types():
    with pytest.raises(nb.od.ODError):
        PositionDevice("a").to_c()
    with pytest.raises(nb.od.ODError):
        TrackingDataArc(np.array([0, 1]), ["a", "a"], np.zeros((2, 2, 1)), (X, Y, Z))
    arc = TrackingDataArc(np.array([0, 1, 2]), ["a", "b", "a"], np.zeros((3, 3, 2)), (X, Y, Z))
    assert arc.filter_by_offset(0, 2).types == arc.types
    assert TrackingDataArc.stack([arc, arc]).obs.shape == (3, 3, 4)
    with pytest.raises(nb.od.ODError):
        nb.BatchLeastSquares(None, {"a": PositionDevice("a").with_noise(X, StochasticNoise(1e-3))}, None)


def test_abi_null_arguments():
    lib = abi.load_library()
    assert C.sizeof(abi.PositionDeviceC) == 64 and C.sizeof(abi.PositionArcC) == 32
    assert lib.nyxb_od_position_batch(None, None, 0, None, None, 1, None, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
    assert lib.nyxb_od_position_smooth_batch(None, None, 0, None, None, 1, None, None, None) == -1
