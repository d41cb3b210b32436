"""The targeter restatement (tests/target_oracle.py) on the reference's own two-body targeter tests, with their GMAT bounds, plus the
pins of what nyxb_target_batch computes: the pseudo-inverse, the clamp order, the stop conditions, the corrected-state quirk, the
per-objective perturbations, the host build of nyxb_target.h, and the argument checks of the C ABI.  CPU only."""
import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import target_oracle as T

ROOT = Path(__file__).resolve().parents[1]
S = 10**9
FRAME = nb.EARTH_J2000
MU = FRAME.mu_km3_s2()
VX, VY, VZ = 3, 4, 5


def two_body(prop_ctor=nb.Propagator.default_dp78):
    prop = prop_ctor(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body()))
    return prop.dynamics.pack(FRAME, None).c, prop.opts.to_c(prop.method)


def ref_orbit(ta_deg):
    """the reference tests' orbit: SMA 8 000 km, ECC 0.2, INC 30, RAAN 60, AoP 60"""
    o = nb.Orbit.keplerian(8000.0, 0.2, 30.0, 60.0, 60.0, ta_deg, 0, FRAME)
    sc = nb.Spacecraft(orbit=o, mass=nb.Mass(100.0, 0.0, 0.0))
    half = int(round(math.pi * math.sqrt(8000.0**3 / MU) * S))   # period / 2
    return nb.pack_spacecraft([sc]), half


def run(cfg, ta_deg=180.0, prop_ctor=nb.Propagator.default_dp78, t_c=0, span=None, **kw):
    dyn_c, opts_c = two_body(prop_ctor)
    (st, cs, ep), half = ref_orbit(ta_deg)
    t_f = t_c + (half if span is None else span)
    return T.target_batch(dyn_c, opts_c, cfg, st, cs, ep, t_c, t_f, **kw)


def dv(*max_step):
    return [(c, 1e-4, 0.0, m, 5.0, -5.0) for c, m in zip((VX, VY, VZ), max_step or (0.2, 0.2, 0.2))]


# ---- the reference's two-body tests (tests/mission_design/targeter single_oe.rs, multi_oe.rs, multi_oe_vnc.rs): |correction| against
# GMAT.  (variables, objectives, true anomaly, propagator, correction frame, GMAT |correction|, bound); a bound of None is the reference's
# "within 1e-6 of GMAT, or smaller"
C3_DECL = [(T.DECL, 5.0, 0.1), (T.C3, -5.0, 0.5)]
SMA_ECC = [(T.ECC, 0.4, 1e-5), (T.SMA, 8100.0, 0.1)]
DP78, RK89 = nb.Propagator.default_dp78, nb.Propagator.default
REFERENCE_CASES = {
    "tgt_sma_from_apo": (dv(), [(T.SMA, 8100.0, 1e-3)], 180.0, DP78, T.FRAME_NONE, 0.05312024615278713, 1e-6),
    "tgt_ecc_from_apo": (dv(5.0, 5.0, 5.0), [(T.ECC, 0.4, 1e-3)], 180.0, DP78, T.FRAME_NONE, 0.7721483022815125, 1e-3),
    "tgt_raan_from_apo": (dv(), [(T.RAAN, 65.0, 1e-3)], 180.0, DP78, T.FRAME_NONE, 0.30344716711198855, 1.5e-3),
    "tgt_raan_from_peri": (dv(0.5, 0.5, 0.5), [(T.RAAN, 65.0, 1e-3)], 0.0, DP78, T.FRAME_NONE, 0.45110541873478793, 6e-3),
    "tgt_aop_from_apo": (dv(), [(T.AOP, 65.0, 1e-3)], 180.0, DP78, T.FRAME_NONE, 0.11772316331182386, 1e-3),
    "tgt_aop_from_peri": (dv(), [(T.AOP, 65.0, 1e-3)], 0.0, DP78, T.FRAME_NONE, 0.12197875695918228, 6e-3),
    "tgt_c3_decl": (dv(), C3_DECL, 0.0, RK89, T.FRAME_NONE, 2.385704523944014, 6e-3),
    "conv_tgt_sma_ecc": (dv(0.5, 0.5, 0.5), SMA_ECC, 0.0, RK89, T.FRAME_NONE, 3.1160765514523914, None),
    "tgt_vnc_c3_decl": (dv(), C3_DECL, 0.0, RK89, T.FRAME_VNC, 2.385704523944014, 6e-3),
    "tgt_vnc_sma_ecc": (dv(0.5, 0.5, 0.5), SMA_ECC, 0.0, RK89, T.FRAME_VNC, 3.1160765514523914, None),
}


def meets_gmat(norm, gmat, bound):
    return abs(norm - gmat) < 1e-6 or norm < gmat if bound is None else abs(norm - gmat) < bound


@pytest.mark.parametrize("name", sorted(REFERENCE_CASES))
def test_reference_case_meets_its_gmat_bound(name):
    variables, objectives, ta, ctor, frame, gmat, bound = REFERENCE_CASES[name]
    out = run(T.config(variables, objectives, frame=frame), ta, prop_ctor=ctor)
    assert out["status"][0] == 0, out["status"]
    norm = float(np.linalg.norm(out["correction"][:, 0]))
    assert meets_gmat(norm, gmat, bound), (name, norm, gmat)


def test_per_objective_perturbations_equal_the_per_variable_ones():
    cfg = T.config(dv(), [(T.DECL, 5.0, 0.1), (T.C3, -5.0, 0.5)])
    a = run(cfg, 0.0, prop_ctor=nb.Propagator.default)
    b = run(cfg, 0.0, prop_ctor=nb.Propagator.default, per_objective=True)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


# ---- the pseudo-inverse, both branches, against numpy
@pytest.mark.parametrize("O,V", [(1, 3), (2, 3), (3, 3), (3, 2), (6, 6), (2, 6)])
def test_pseudo_inverse_matches_numpy(O, V):
    rng = np.random.default_rng(O * 10 + V)
    J = rng.normal(size=(O, V))
    P = np.array(T.pinv(list(J.ravel()), O, V)).reshape(V, O)
    np.testing.assert_allclose(P, np.linalg.pinv(J), rtol=0, atol=1e-10)


def test_pseudo_inverse_singular_on_a_zero_column():
    J = [1.0, 0.0, 2.0, 0.0]   # 2 x 2, second column zero
    assert T.pinv(J, 2, 2) is None


def test_clamp_order_is_step_first_then_bounds_on_the_step():
    var = abi.TgtVariableC(VX, 0, 1e-4, 0.0, 0.2, 0.1, -0.05)
    assert T.clamp(var, 0.3) == 0.2          # |d| > max_step: clipped to the step, the max value is not applied
    assert T.clamp(var, -0.3) == -0.2
    assert T.clamp(var, 0.15) == 0.1         # within the step: bounded by max_value
    assert T.clamp(var, -0.15) == -0.05      # and by min_value
    assert T.clamp(var, 0.01) == 0.01


# ---- stop conditions
def test_converged_at_iteration_zero():
    (st, cs, ep), half = ref_orbit(180.0)
    dyn_c, opts_c = two_body()
    end, _, _, _ = T.pyoracle.propagate_batch(dyn_c, opts_c, st, cs, ep, half)
    sma = T.evaluate(T.SMA, end[:6, 0], MU)
    out = run(T.config(dv(), [(T.SMA, sma + 1e-4, 1e-3)]))
    assert out["status"][0] == 0 and out["iterations"][0] == 0
    assert np.array_equal(out["correction"][:, 0], np.zeros(3))


def test_too_many_iterations_after_iterations_plus_one_evaluations():
    trace = []
    out = run(T.config(dv(), [(T.SMA, 8100.0, 1e-9)], iterations=2), trace=trace)
    assert out["status"][0] == abi.ERR_TGT_TOO_MANY_ITERATIONS and out["iterations"][0] == 2
    assert [t[0] for t in trace] == [0, 1, 2]


def test_correction_ineffective_when_the_step_is_clipped_to_zero():
    out = run(T.config([(c, 1e-4, 0.0, 0.0, 5.0, -5.0) for c in (VX, VY, VZ)], [(T.SMA, 8100.0, 1e-3)]))
    assert out["status"][0] == abi.ERR_TGT_CORRECTION_INEFFECTIVE and out["iterations"][0] == 1


def test_singular_jacobian_on_an_exactly_zero_column():
    out = run(T.config([(VX, 1e-4, 0.0, 0.2, 5.0, -5.0)], [(T.Z, 1.0, 1e-3)]), span=0)
    assert out["status"][0] == abi.ERR_TGT_SINGULAR_JACOBIAN and out["iterations"][0] == 0


def test_corrected_state_applies_the_total_once_with_the_start_dcm():
    cfg = T.config(dv(), [(T.DECL, 5.0, 0.1), (T.C3, -5.0, 0.5)], frame=T.FRAME_VNC)
    trace = []
    out = run(cfg, 0.0, prop_ctor=nb.Propagator.default, trace=trace)
    assert out["status"][0] == 0 and out["iterations"][0] >= 2
    dyn_c, opts_c = two_body(nb.Propagator.default)
    (st, cs, ep), _ = ref_orbit(0.0)
    start, _, _, _ = T.pyoracle.propagate_batch(dyn_c, opts_c, st, cs, ep, 0)
    once = T.apply_vars(cfg, list(out["correction"][:, 0]), start[:6, 0])
    assert np.array_equal(out["corrected"][:6, 0], once)
    # the iterated state (each step applied with the DCM of the state it is applied to) is not the corrected state
    assert not np.array_equal(np.array(once), np.array(out["xi"][:, 0]))
    assert np.abs(np.array(once)[3:] - out["xi"][3:, 0]).max() > 1e-12


# ---- the host build of nyxb_target.h
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so_path = tmp_path_factory.mktemp("shim") / "target_core_shim.so"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                    str(ROOT / "tests" / "cpp" / "target_core_shim.cpp"), "-o", str(so_path)], check=True, capture_output=True)
    lib = C.CDLL(str(so_path))
    lib.shim_tgt_eval.restype = C.c_double
    lib.shim_tgt_eval.argtypes = [C.c_int, C.c_void_p, C.c_double]
    lib.shim_tgt_step.restype = C.c_int
    lib.shim_tgt_step.argtypes = [C.POINTER(abi.TargetConfigC), C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.shim_tgt_perturbed.restype = None
    lib.shim_tgt_perturbed.argtypes = [C.POINTER(abi.TargetConfigC), C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _states(rng, k):
    out = []
    for _ in range(k):
        o = nb.Orbit.keplerian(rng.uniform(6800, 42000), rng.uniform(0.001, 0.7), rng.uniform(0.5, 179), rng.uniform(0, 360),
                               rng.uniform(0, 360), rng.uniform(0, 360), 0, FRAME)
        out.append(o.to_cartesian_pos_vel())
    return out


def test_host_build_of_the_header_matches_the_restatement(shim):
    rng = np.random.default_rng(7)
    states = _states(rng, 40)
    # degenerate states where the header's angles have nothing to guard them: equatorial (no node), circular (no periapsis),
    # radial (no angular momentum), at rest (zero energy divides), and non-finite
    degenerate = [np.array([7000.0, 0, 0, 0, 7.5, 0]), np.array([7000.0, 0, 0, 0, math.sqrt(MU / 7000.0), 0]),
                  np.array([7000.0, 0, 0, 1.0, 0, 0]), np.array([0.0, 0, 7000.0, 0, 0, 0]), np.array([7000.0, 0, 0, 0, 0, 0]),
                  np.array([0.0, 0, 0, 0, 7.5, 0]), np.array([7000.0, 0, np.nan, 0, 7.5, 0]), np.array([7000.0, 0, 0, np.inf, 7.5, 0])]
    n_nan = 0
    for rv in states + degenerate:
        rv = np.ascontiguousarray(rv, dtype=np.float64)
        for p in range(abi_n_params()):
            got, want = shim.shim_tgt_eval(p, rv.ctypes.data, MU), T.evaluate(p, rv, MU)
            assert got == want or (math.isnan(got) and math.isnan(want)), (p, rv, got, want)
            n_nan += math.isnan(want)
    assert n_nan > 20
    n_steps = 0
    for frame in (T.FRAME_NONE, T.FRAME_VNC, T.FRAME_RIC):
        for O, V in ((1, 3), (2, 3), (3, 3), (3, 2), (2, 1)):
            comps = [VX, VY, VZ][:V] if frame else [0, VY, VZ][:V]
            cfg = T.config([(c, 1e-3 * (j + 1), 0.0, 0.05, 5.0, -5.0) for j, c in enumerate(comps)],
                           [(p, rng.uniform(0, 1) * 10, 1e-6) for p in (T.SMA, T.INC, T.ECC)[:O]], frame=frame, iterations=3)
            for rv in states[:10]:
                xi = list(rv)
                for j in range(V):
                    out = np.empty(6)
                    shim.shim_tgt_perturbed(C.byref(cfg), j, np.ascontiguousarray(rv).ctypes.data, out.ctypes.data)
                    assert np.array_equal(out, T.perturbed(cfg, j, xi))
                xf = np.ascontiguousarray(np.stack([np.asarray(rv) * (1 + 1e-3 * k) for k in range(V + 1)]))
                xi_c, tot_c, err_c, prev_c = np.ascontiguousarray(rv, dtype=np.float64).copy(), np.full(6, 0.01), np.empty(6), np.array([math.inf])
                rc = shim.shim_tgt_step(C.byref(cfg), MU, 1, xf.ctypes.data, xi_c.ctypes.data, tot_c.ctypes.data, err_c.ctypes.data, prev_c.ctypes.data)
                rc_p, xi_p, tot_p, err_p, prev_p, _ = T.step(cfg, MU, 1, [list(x) for x in xf], xi, [0.01] * V, math.inf)
                assert rc == rc_p
                assert np.array_equal(xi_c, xi_p) and np.array_equal(tot_c[:V], tot_p) and prev_c[0] == prev_p
                assert np.array_equal(err_c[:O], err_p)
                n_steps += 1
    assert n_steps == 150


def abi_n_params():
    return 23


# ---- the C ABI: layouts and argument checks (no device is reached)
def test_struct_sizes():
    assert C.sizeof(abi.TgtVariableC) == 48 and C.sizeof(abi.TgtObjectiveC) == 40 and C.sizeof(abi.TargetConfigC) == 544


def _bad(cfg, **over):
    lib = abi.load_library()
    fake = C.create_string_buffer(64)   # never dereferenced: every check below happens before the engine is read
    d = np.zeros(64)
    i32 = np.zeros(8, dtype=np.int32)
    args = dict(eng=C.cast(fake, C.c_void_p), state=d.ctypes.data, consts=d.ctypes.data, epoch=d.ctypes.data)
    args.update(over)
    return lib.nyxb_target_batch(args["eng"], C.byref(cfg), 1, args["state"], args["consts"], args["epoch"], 0, 1, d.ctypes.data,
                                 d.ctypes.data, d.ctypes.data, d.ctypes.data, i32.ctypes.data, i32.ctypes.data)


def good():
    return T.config(dv(), [(T.SMA, 8100.0, 1e-3)])


def test_too_many_problems_are_rejected_before_any_launch():
    lib = abi.load_library()
    fake = C.create_string_buffer(64)
    d = np.zeros(64)
    i32 = np.zeros(8, dtype=np.int32)
    rc = lib.nyxb_target_batch(C.cast(fake, C.c_void_p), C.byref(good()), 2**31 // 7 + 1, d.ctypes.data, d.ctypes.data, d.ctypes.data, 0, 1,
                               d.ctypes.data, d.ctypes.data, d.ctypes.data, d.ctypes.data, i32.ctypes.data, i32.ctypes.data)
    assert rc == -1 and b"too many" in lib.nyxb_last_error()


@pytest.mark.parametrize("mutate", [
    lambda c: setattr(c, "n_vars", 0), lambda c: setattr(c, "n_vars", 7), lambda c: setattr(c, "n_objs", 0),
    lambda c: setattr(c, "n_objs", 7), lambda c: setattr(c, "correction_frame", 3), lambda c: setattr(c, "iterations", -1),
    lambda c: setattr(c.vars[0], "component", 6), lambda c: setattr(c.vars[0], "component", -1),
    lambda c: setattr(c.objs[0], "parameter", 23), lambda c: setattr(c.objs[0], "parameter", -1),
    lambda c: (setattr(c, "correction_frame", T.FRAME_VNC), setattr(c.vars[0], "component", 0)),
    lambda c: setattr(c.vars[1], "max_step", -0.1), lambda c: setattr(c.vars[1], "max_value", -0.1),
    lambda c: setattr(c.vars[1], "min_value", 5.5), lambda c: setattr(c.vars[2], "perturbation", 0.0),
    lambda c: setattr(c.vars[2], "perturbation", math.inf), lambda c: setattr(c.vars[2], "perturbation", math.nan),
])
def test_bad_config_is_rejected_before_any_launch(mutate):
    cfg = good()
    mutate(cfg)
    assert _bad(cfg) == -1


def test_null_pointers_are_rejected():
    assert _bad(good(), eng=None) == -1
    assert _bad(good(), state=None) == -1
    assert _bad(good(), epoch=None) == -1
    lib = abi.load_library()
    assert lib.nyxb_target_batch(None, None, 1, None, None, None, 0, 1, None, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
