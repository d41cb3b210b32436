"""The Python targeting layer (nyx_b200/targeter.py) on the CPU: an engine stand-in whose `target_batch` / `propagate_batch` call the
oracle and the restatement (tests/target_oracle.py) instead of libnyxb.so.  Errors, decoding, `apply`, and the VNC refusal of
ProcessNoise3D."""
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from oracle import pyoracle
from tests import target_oracle as T

S = 10**9
FRAME = nb.EARTH_J2000
MU = FRAME.mu_km3_s2()


class OracleEngine:
    def __init__(self, prop):
        self.dyn_c = prop.dynamics.pack(FRAME, None).c
        self.opts_c = prop.opts.to_c(prop.method)

    def target_batch(self, cfg, st, cs, ep, t_c, t_f):
        out = T.target_batch(self.dyn_c, self.opts_c, cfg, st, cs, ep, t_c, t_f)
        out.pop("xi")
        return out

    def propagate_batch(self, st, cs, ep, end):
        return pyoracle.propagate_batch(self.dyn_c, self.opts_c, st, cs, ep, end)


@pytest.fixture
def prop(monkeypatch):
    p = nb.Propagator.default_dp78(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body()))
    eng = OracleEngine(p)
    monkeypatch.setattr(p, "engine", lambda frame, almanac=None: eng)
    return p


def sc(ta=180.0, epoch=0):
    return nb.Spacecraft(orbit=nb.Orbit.keplerian(8000.0, 0.2, 30.0, 60.0, 60.0, ta, epoch, FRAME), mass=nb.Mass(100.0, 0.0, 0.0))


HALF = int(round(math.pi * math.sqrt(8000.0**3 / MU) * S))


def test_defaults_match_the_reference():
    v = nb.Variable.from_vary(nb.Vary.VelocityY)
    assert (v.perturbation, v.init_guess, v.max_step, v.max_value, v.min_value) == (0.0001, 0.0, 0.2, 5.0, -5.0)
    assert nb.Objective.new(nb.StateParameter.SemiMajorAxis, 1.0).tolerance == 1e-3
    assert nb.Objective.new(nb.StateParameter.Period, 1.0).tolerance == 0.1
    t = nb.Targeter.delta_v(None, [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 1.0)])
    assert t.iterations == 100 and t.correction_frame is None and [x.component for x in t.variables] == [3, 4, 5]
    assert nb.Targeter.vnc(None, t.objectives).correction_frame == nb.LocalFrame.VNC
    assert [x.component for x in nb.Targeter.delta_r(None, t.objectives).variables] == [0, 1, 2]


def test_solution_decoding_and_apply(prop):
    tgt = nb.Targeter.delta_v(prop, [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 8100.0)])
    sol = tgt.try_achieve_from(sc(), 0, HALF)
    assert abs(np.linalg.norm(sol.correction) - 0.05312024615278713) < 1e-6
    assert sol.corrected_state.epoch() == 0 and sol.achieved_state.epoch() == HALF
    assert sol.corrected_state.mass == sc().mass
    final = tgt.apply(sol)
    assert abs(nb.param.evaluate(nb.StateParameter.SemiMajorAxis, final.orbit.to_cartesian_pos_vel(), MU) - 8100.0) <= 1e-3


def test_ensemble_errors_and_apply_many(prop):
    tgt = nb.Targeter.delta_v(prop, [nb.Objective.within_tolerance(nb.StateParameter.SemiMajorAxis, 8100.0, 1e-9)])
    tgt.iterations = 2
    ens = tgt.try_achieve_from_many([sc(), sc(170.0)], 0, HALF)
    assert len(ens) == 2
    for i in range(2):
        e = ens.error(i)
        assert isinstance(e, nb.TargetingError) and e.variant == "TooManyIterations"
        with pytest.raises(nb.TargetingError):
            ens.solution(i)
    tgt2 = nb.Targeter.delta_v(prop, [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 8100.0)])
    ens2 = tgt2.try_achieve_from_many([sc(), sc(170.0)], 0, HALF)
    assert [ens2.error(i) for i in range(2)] == [None, None]
    assert len(tgt2.apply_many(ens2)) == 2


def test_verification_error(prop):
    tgt = nb.Targeter.delta_v(prop, [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 8100.0)])
    sol = tgt.try_achieve_from(sc(), 0, HALF)
    sol.corrected_state = sc()
    with pytest.raises(nb.TargetingError) as e:
        tgt.apply(sol)
    assert e.value.variant == "Verification"


def test_refusals(prop):
    obj = [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 8100.0)]
    with pytest.raises(nb.TargetingError, match="UnsupportedVariable"):
        nb.Variable.from_vary(nb.Vary.ThrustX)
    with pytest.raises(nb.TargetingError, match="UnsupportedVariable"):
        nb.Targeter.new(prop, [nb.Variable(component=nb.Vary.Duration)], obj).try_achieve_from(sc(), 0, HALF)
    with pytest.raises(nb.TargetingError, match="UnsupportedObjectiveFrame"):
        nb.Targeter.in_frame(prop, [nb.Variable()], obj, nb.MOON_J2000).try_achieve_from(sc(), 0, HALF)
    with pytest.raises(nb.TargetingError, match="UnsupportedObjective"):
        nb.Targeter.delta_v(prop, [nb.Objective.new(nb.StateParameter.Cr, 1.0)]).try_achieve_from(sc(), 0, HALF)
    with pytest.raises(nb.TargetingError, match="FrameError"):
        nb.Targeter.vnc_with_components(prop, [nb.Variable(component=nb.Vary.PositionX)], obj).try_achieve_from(sc(), 0, HALF)
    with pytest.raises(nb.TargetingError, match="VariableError"):
        nb.Targeter.new(prop, [nb.Variable(max_step=-1.0)], obj).try_achieve_from(sc(), 0, HALF)
    with pytest.raises(nb.TargetingError, match="UnderdeterminedProblem"):
        nb.Targeter.delta_v(prop, []).try_achieve_from(sc(), 0, HALF)


def test_status_decoding_of_a_singular_jacobian(prop):
    tgt = nb.Targeter.new(prop, [nb.Variable(component=nb.Vary.VelocityX)], [nb.Objective.new(nb.StateParameter.Z, 1.0)])
    with pytest.raises(nb.TargetingError) as e:
        tgt.try_achieve_from(sc(), 0, 0)
    assert e.value.variant == "SingularJacobian"


def test_c3_and_declination_are_evaluated():
    rv = sc(0.0).orbit.to_cartesian_pos_vel()
    sma = nb.param.evaluate(nb.StateParameter.SemiMajorAxis, rv, MU)
    assert nb.param.evaluate(nb.StateParameter.C3, rv, MU) == pytest.approx(-MU / sma, rel=1e-15)
    assert nb.param.evaluate(nb.StateParameter.Declination, rv, MU) == pytest.approx(math.degrees(math.asin(rv[2] / np.linalg.norm(rv[:3]))))


def test_process_noise_refuses_vnc():
    with pytest.raises(nb.ODError):
        nb.ProcessNoise3D.from_diagonal([1e-12] * 3, 0, nb.LocalFrame.VNC)
    nb.ProcessNoise3D.from_diagonal([1e-12] * 3, 0, nb.LocalFrame.RIC)
    assert abi.TGT_FRAME_VNC == 1


def test_spacecraft_uncertainty_rotates_a_vnc_covariance():
    """sc_uncertainty.rs:100-102: the diagonal is rotated by the VNC -> inertial DCM (columns v^, h^, v^ x h^), not taken as inertial"""
    s = sc(40.0)
    u = nb.SpacecraftUncertainty(s, frame=nb.LocalFrame.VNC, x_km=1.0, y_km=0.1, z_km=0.01, vx_km_s=1e-3, vy_km_s=1e-4, vz_km_s=1e-5)
    cov = u.to_estimate().covar
    r, v = s.orbit.radius_km, s.orbit.velocity_km_s
    vh = v / np.linalg.norm(v)
    nh = np.cross(r, v) / np.linalg.norm(np.cross(r, v))
    D = np.column_stack([vh, nh, np.cross(vh, nh)])
    np.testing.assert_allclose(cov[:3, :3], D.T @ np.diag([1.0, 0.01, 1e-4]) @ D, rtol=0, atol=1e-15)
    np.testing.assert_allclose(cov[3:6, 3:6], D.T @ np.diag([1e-6, 1e-8, 1e-10]) @ D, rtol=0, atol=1e-21)
    # the same DCM as the targeter's correction frame
    assert np.allclose(D.ravel(), T.dcm(T.FRAME_VNC, s.orbit.to_cartesian_pos_vel()), rtol=0, atol=1e-15)
    inertial = nb.SpacecraftUncertainty(s, x_km=1.0, y_km=0.1, z_km=0.01, vx_km_s=1e-3, vy_km_s=1e-4, vz_km_s=1e-5).to_estimate().covar
    assert not np.allclose(cov, inertial)
