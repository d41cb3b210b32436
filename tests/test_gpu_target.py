"""nyxb_target_batch on the GPU against the restatement (tests/target_oracle.py), JGM-3 8x8 LEO, start epochs that differ per problem.

Families: per-thread STRICT and FAST, warp-cooperative STRICT and FAST, transposed FAST, each forced with nyxb_engine_set_kernel.
STRICT must give the restatement's status and iteration count for every problem and corrections within 1e-9 relative; FAST the same
statuses, corrections within FAST_REL of STRICT's, and converged problems whose corrected states, re-propagated by the oracle, meet
their tolerances.  The fixtures keep every error of every iteration away from its tolerance (test_fixture_errors_are_clear_of_tolerances,
on the CPU), so that FAST's perturbation of the propagation cannot flip a convergence test.
"""
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from oracle import pyoracle
from tests import target_oracle as T
from tests.test_oracle_target import REFERENCE_CASES, meets_gmat

S = 10**9
FRAME = nb.EARTH_J2000
MU = FRAME.mu_km3_s2()
VX, VY, VZ = 3, 4, 5
T_C = 600 * S
T_F = T_C + 2700 * S
FAST_REL = 1e-7   # relative |correction| FAST vs STRICT; an H100 (700 W) measured at most 3.4e-9 (backward, transposed); printed by the test
FAMILIES = [(nb.MODE_STRICT, abi.KERNEL_THREAD), (nb.MODE_FAST, abi.KERNEL_THREAD), (nb.MODE_STRICT, abi.KERNEL_COOP),
            (nb.MODE_FAST, abi.KERNEL_COOP), (nb.MODE_FAST, abi.KERNEL_TRANSPOSED)]
FAM_IDS = ["strict-thread", "fast-thread", "strict-coop", "fast-coop", "fast-transposed"]


def dynamics():
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", 8, 8, nb.IAU_EARTH_FRAME)
    return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))


DYN = dynamics()


def prop(mode):
    return nb.Propagator.default(DYN, mode=mode)


def states(sma_offsets, nan_at=()):
    scs = []
    for k, d in enumerate(sma_offsets):
        o = nb.Orbit.keplerian(6878.0 + d, 0.01 + 0.001 * k, 51.6, 30.0 + k, 40.0, 10.0 * k, -60 * S * k, FRAME)
        scs.append(nb.Spacecraft(orbit=o, mass=nb.Mass(100.0, 10.0, 0.0)))
    st, cs, ep = nb.pack_spacecraft(scs)
    for k in nan_at:
        st[0, k] = np.nan
    return st, cs, ep


def oracle_args():
    p = prop(nb.MODE_STRICT)
    return DYN.pack(FRAME, None).c, p.opts.to_c(p.method)


def _nominal_sma(st, cs, ep, k):
    dyn_c, opts_c = oracle_args()
    a, aep, _, _ = pyoracle.propagate_batch(dyn_c, opts_c, st[:, k:k + 1], cs[:, k:k + 1], ep[k:k + 1], T_C)
    b, _, _, _ = pyoracle.propagate_batch(dyn_c, opts_c, a, cs[:, k:k + 1], aep, T_F)
    return T.evaluate(T.SMA, b[:6, 0], MU)


def scenarios():
    """name -> (cfg, state, consts, epoch0, t_c, t_f)"""
    st, cs, ep = states([0.0, 3.0, -4.0, 7.0, 900.0, 0.0, 2.0], nan_at=(5,))
    desired = _nominal_sma(st, cs, ep, 0) + 2e-4   # problem 0 converges at iteration 0
    inertial = T.config([(c, 1e-4, 0.0, 0.2, 5.0, -5.0) for c in (VX, VY, VZ)], [(T.SMA, desired, 1e-3)], iterations=2)
    rows = ([(c, 1e-4, 0.0, 0.2, 5.0, -5.0) for c in (VX, VY, VZ)], [(T.SMA, 6893.0, 1e-3), (T.ECC, 0.013, 1e-5)])
    two = T.config(*rows, iterations=6)
    st2, cs2, ep2 = states([0.0, 4.0, 9.0])
    return {
        "inertial": (inertial, st, cs, ep, T_C, T_F),
        "vnc": (T.config(*rows, frame=T.FRAME_VNC, iterations=6), st2, cs2, ep2, T_C, T_F),
        "ric": (T.config(*rows, frame=T.FRAME_RIC, iterations=6), st2, cs2, ep2, T_C, T_F),
        "backward": (two, st2, cs2, ep2, -T_C, -T_C - 2700 * S),
        "singular": (T.config([(VX, 1e-4, 0.0, 0.2, 5.0, -5.0)], [(T.Z, 1.0, 1e-3)]), st2, cs2, ep2, T_C, T_C),
    }


SCEN = scenarios()


@pytest.fixture(scope="module")
def restated():
    dyn_c, opts_c = oracle_args()
    out = {}
    for name, (cfg, st, cs, ep, tc, tf) in SCEN.items():
        trace = []
        out[name] = (T.target_batch(dyn_c, opts_c, cfg, st, cs, ep, tc, tf, trace=trace), trace)
    return out


def test_fixture_errors_are_clear_of_tolerances(restated):
    """every error of every evaluation is more than 20 % away from its tolerance, and the set holds every outcome"""
    for name, (out, trace) in restated.items():
        cfg = SCEN[name][0]
        for it, p, err, _ in trace:
            for i, e in enumerate(err):
                if math.isfinite(e):
                    tol = cfg.objs[i].tolerance
                    assert not 0.8 * tol < abs(e) < 1.2 * tol, (name, it, p, i, e, tol)
    st = restated["inertial"][0]["status"].tolist()
    it = restated["inertial"][0]["iterations"].tolist()
    assert st[0] == 0 and it[0] == 0
    assert any(s == 0 and i > 0 for s, i in zip(st, it))
    assert abi.ERR_TGT_TOO_MANY_ITERATIONS in st and abi.ERR_PROP_MATH in [s & 0xFF for s in st]
    assert (restated["singular"][0]["status"] == abi.ERR_TGT_SINGULAR_JACOBIAN).all()
    for name in ("vnc", "ric", "backward"):
        assert (restated[name][0]["status"] == 0).all(), (name, restated[name][0]["status"])


def engine(mode, kernel):
    eng = prop(mode).engine(FRAME, None)
    eng.set_kernel(kernel)
    return eng


def call(eng, name, sl=slice(None)):
    cfg, st, cs, ep, tc, tf = SCEN[name]
    return eng.target_batch(cfg, st[:, sl], cs[:, sl], ep[sl], tc, tf)


@pytest.fixture(scope="module")
def strict_runs():
    return {name: call(engine(nb.MODE_STRICT, abi.KERNEL_THREAD), name) for name in SCEN}


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES, ids=FAM_IDS)
@pytest.mark.parametrize("name", sorted(SCEN))
def test_family_against_restatement(fam, name, restated, strict_runs):
    mode, kernel = fam
    eng = engine(mode, kernel)
    got = call(eng, name)
    ref = restated[name][0]
    assert got["status"].tolist() == ref["status"].tolist(), (got["status"], ref["status"])
    ok = (ref["status"] & 0xFF) != abi.ERR_PROP_MATH
    if mode == nb.MODE_STRICT:
        assert got["iterations"].tolist() == ref["iterations"].tolist()
        d = np.abs(got["correction"][:, ok] - ref["correction"][:, ok]).max() / max(np.abs(ref["correction"][:, ok]).max(), 1e-12)
        assert d < 1e-9, d
        return
    s = strict_runs[name]
    scale = max(np.abs(s["correction"][:, ok]).max(), 1e-12)
    d = np.abs(got["correction"][:, ok] - s["correction"][:, ok]).max() / scale
    print(f"{name} {FAM_IDS[FAMILIES.index(fam)]}: max relative |correction| FAST vs STRICT = {d:.3e}")
    assert d < FAST_REL, d
    # converged problems without a local frame: the oracle re-propagates the corrected state and meets every tolerance
    cfg, st, cs, ep, tc, tf = SCEN[name]
    if cfg.correction_frame == T.FRAME_NONE and name != "singular":
        dyn_c, opts_c = oracle_args()
        conv = np.flatnonzero(got["status"] == 0)
        fin, _, _, _ = pyoracle.propagate_batch(dyn_c, opts_c, got["corrected"][:, conv], cs[:, conv], np.full(len(conv), tc, dtype=np.int64), tf)
        for k in range(len(conv)):
            for i in range(cfg.n_objs):
                o = cfg.objs[i]
                assert abs(o.desired - T.evaluate(o.parameter, fin[:6, k], MU)) <= o.tolerance


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES, ids=FAM_IDS)
def test_alone_equals_batch_and_calls_repeat(fam):
    eng = engine(*fam)
    full = call(eng, "inertial")
    again = call(eng, "inertial")
    for k in full:
        assert np.array_equal(full[k], again[k], equal_nan=True), k
    for p in (0, 2, 4):
        one = call(eng, "inertial", slice(p, p + 1))
        for k in full:
            assert np.array_equal(one[k][..., 0], full[k][..., p], equal_nan=True), (p, k)


@pytest.mark.gpu
def test_launch_count_grows_by_four_per_iteration():
    eng = engine(nb.MODE_STRICT, abi.KERNEL_THREAD)
    for name in ("inertial", "singular"):
        c0 = eng.launch_count()
        out = call(eng, name)
        live = out["status"] & 0xFF != abi.ERR_PROP_MATH
        rounds = int(out["iterations"][live].max()) + 1
        assert eng.launch_count() - c0 == 3 + 4 * rounds + 1, (name, eng.launch_count() - c0, rounds)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [nb.MODE_STRICT, nb.MODE_FAST], ids=["strict", "fast"])
@pytest.mark.parametrize("name", sorted(REFERENCE_CASES))
def test_reference_cases(mode, name):
    """the reference's cases with their GMAT bounds (tests/test_oracle_target.py).  They are two-body, which only the per-thread kernel
    runs (the lane-cooperative and transposed kernels split a harmonic field)"""
    variables, objectives, ta, ctor, frame, gmat, bound = REFERENCE_CASES[name]
    p = ctor(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body()), mode=mode)
    eng = p.engine(FRAME, None)
    eng.set_kernel(abi.KERNEL_THREAD)
    o = nb.Orbit.keplerian(8000.0, 0.2, 30.0, 60.0, 60.0, ta, 0, FRAME)
    st, cs, ep = nb.pack_spacecraft([nb.Spacecraft(orbit=o, mass=nb.Mass(100.0, 0.0, 0.0))])
    half = int(round(math.pi * math.sqrt(8000.0**3 / MU) * S))
    out = eng.target_batch(T.config(variables, objectives, frame=frame), st, cs, ep, 0, half)
    assert out["status"][0] == 0
    norm = float(np.linalg.norm(out["correction"][:, 0]))
    print(f"{name}: |correction| = {norm!r}")
    assert meets_gmat(norm, gmat, bound), (name, norm, gmat)


@pytest.mark.gpu
def test_states_outside_the_integration_frame_are_unsupported():
    alm = nb.Almanac.synthetic(nb.EARTH_J2000, 0, 3.0, bodies=(nb.MOON, nb.SUN))
    p = nb.Propagator.default(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.point_masses([nb.MOON, nb.SUN])))
    p.opts.integration_frame = nb.EARTH_J2000
    eng = p.engine(nb.MOON_J2000, alm)
    cfg, st, cs, ep, tc, tf = SCEN["vnc"]
    c0 = eng.launch_count()
    with pytest.raises(nb.PropagationError, match="rc=-4"):
        eng.target_batch(cfg, st, cs, ep, tc, tf)
    assert eng.launch_count() == c0


@pytest.mark.gpu
def test_python_layer_on_the_gpu():
    p = prop(nb.MODE_STRICT)
    o = nb.Orbit.keplerian(6878.0, 0.01, 51.6, 30.0, 40.0, 0.0, 0, FRAME)
    sc = nb.Spacecraft(orbit=o, mass=nb.Mass(100.0, 10.0, 0.0))
    tgt = nb.Targeter.delta_v(p, [nb.Objective.new(nb.StateParameter.SemiMajorAxis, 6890.0)])
    sol = tgt.try_achieve_from(sc, T_C, T_F)
    assert sol.iterations >= 1
    final = tgt.apply(sol)
    assert abs(nb.param.evaluate(nb.StateParameter.SemiMajorAxis, final.orbit.to_cartesian_pos_vel(), MU) - 6890.0) <= 1e-3
