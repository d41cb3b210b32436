"""Every kernel family against the CPU oracle for gravity fields of degree 71..96, the top of the range the C ABI accepts.

Inputs: tests/high_degree.py (degree-96 Earth and Moon fields: the fixtures continued by seeded draws on a fitted power law; 40 low
lunar orbits with periapses at 30..60 km and 24 LEO orbits at 250..300 km, polar and near-polar ones among them; RK89 at a fixed
60 s over 3 h).  Families are forced as in tests/test_gpu_fast_matrix.py and checked with `last_kernel()`:
  K1       per-thread kernel (FAST: column walk; STRICT: grav_accel_rows, whose Legendre rows are sized for degree 96)
  K2-G*    lane-cooperative FAST kernel at 8 / 16 / 32 lanes: 3-4 columns per lane at 32 lanes, record table in global memory
  K3-G*    lane-cooperative STRICT kernel (K2-G* in STRICT mode) at each lane count's largest fitting degree (32: 96, 16: 75, 8: 50)

FAST fixed step: status, epochs, n_steps, n_rhs and step_ns equal; |dr| and |dv| below max(5e-9 km, 10 x the spread of the
oracle against its FMA build) and max(5e-12 km/s, 10 x that spread).  STRICT fixed step: bit-equal.  STRICT adaptive (RK89,
default controller): the rule of tests/test_gpu_fuzz.py.  Exactly polar start states (x = y = 0 in the body frame, identity
rotation) through one 1 ms RK4 step.  The dispatch and refusals at the edges of the range: degree 97, the transposed kernel
above degree 70, forced STRICT lane counts whose shared-memory slab does not fit.  STM and filter kernels through the machinery
of tests/test_gpu_od_matrix.py with the degree-96 fields (tests/od_matrix.gravity).

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), FAST fixed step, |dr| km / |dv| km/s over every lunar shape (71x71 to
96x96, 96x0, 96x1, 96x48) and for the Earth 96x96 field; K2 gives the same numbers at 8, 16 and 32 lanes:
  family   lunar shapes         earth 96x96
  K1       1.4e-10 / 1.2e-13    3.7e-10 / 4.0e-13
  K2-G*    1.3e-10 / 1.2e-13    5.0e-10 / 5.9e-13
STRICT: bit-equal at fixed step, and every trajectory bit-equal in the adaptive runs.  STM and filters, largest ratio of the GPU
difference to the oracle's spread (the bound is 10): STM STRICT (lunar, with SRP) 0.98, FAST 1.5; filters FAST-coop 1.9,
FAST-thread 1.8, STRICT 1.6, coop against per-thread 1.3 (bound 3).  This file found that K2 at 32 lanes returned NaN at 95x95
(a recursion left running through a lane's 62-entry idle gap overflowed near the lunar surface); it takes about 4 min on that
card, most of it in the oracle's filters."""
import ctypes as C
import functools

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import high_degree as hd
from tests import od_matrix as om
from tests.test_gpu_fast_matrix import KERNEL, assert_fixed_parity, force_family
from tests.test_gpu_od_matrix import (COOP_VS_THREAD, MODES, SHAPE_CASES, assert_filter_parity, assert_stm_parity, check, run_filters,
                                      run_stm)
from tests.util import S, max_dr_dv

pytestmark = pytest.mark.gpu

RC_UNSUPPORTED = -4


def run(body, mode, family, degree=hd.TOP, order=None, opts=None, st=None, ep=None, end=hd.END):
    prop = hd.propagator(body, mode, degree, order, opts=opts)
    eng = force_family(nb.Engine(*prop.lower(hd.FRAME[body], None), mode, 0), family)
    st0, cs, ep0 = hd.ensemble(body)
    got = eng.propagate_batch(st0 if st is None else st, cs, ep0 if ep is None else ep, end)
    assert eng.last_kernel() == KERNEL[family[:2]], (family, eng.last_kernel())
    return eng, got


# ---- FAST, fixed step: K1 and K2 at every lane count x the shapes of the top of the range
FAST_FAMILIES = ("K1", "K2-G8", "K2-G16", "K2-G32")
FAST_SHAPES = [("moon", 71, 71), ("moon", 80, 80), ("moon", 95, 95), ("moon", 96, 96), ("moon", 96, 0), ("moon", 96, 1),
               ("moon", 96, 48), ("earth", 96, 96)]


@pytest.mark.parametrize("body,degree,order", FAST_SHAPES, ids=[f"{b}-{d}x{o}" for b, d, o in FAST_SHAPES])
@pytest.mark.parametrize("family", FAST_FAMILIES)
def test_fast_fixed_step(oracle, family, body, degree, order):
    _, got = run(body, nb.MODE_FAST, family, degree, order)
    assert_fixed_parity(got, hd.oracle_fixed(body, degree, order), hd.RK89, f"{family} {body} {degree}x{order}",
                        hd.fixed_bounds(body, degree, order))


# ---- STRICT: bit-equal at fixed step
STRICT_CASES = [("K1", "moon", 96), ("K1", "earth", 96), ("K2-G32", "moon", 96), ("K2-G32", "earth", 96), ("K2-G16", "moon", 75),
                ("K2-G8", "moon", 50)]


def assert_bit_equal(got, ref, tag):
    for k, name in enumerate(("state", "epoch")):
        assert np.array_equal(got[k], ref[k]), (tag, name, max_dr_dv(got[0], ref[0]))
    assert np.array_equal(got[3], ref[3]) and (got[3] == 0).all(), tag
    for f in ("n_steps", "n_rhs", "step_ns"):
        assert np.array_equal(got[2][f], ref[2][f]), (tag, f)


@pytest.mark.parametrize("family,body,degree", STRICT_CASES, ids=[f"{'K3' + f[2:] if f != 'K1' else f}-{b}-{d}" for f, b, d in STRICT_CASES])
def test_strict_fixed_step_bit_equal(oracle, family, body, degree):
    eng, got = run(body, nb.MODE_STRICT, family, degree)
    if family != "K1":
        assert eng.lanes() == int(family[4:])
    assert_bit_equal(got, hd.oracle_fixed(body, degree), f"STRICT {family} {body} {degree}")


@functools.lru_cache(maxsize=None)
def _oracle_adaptive(body):
    from oracle import pyoracle

    prop = hd.propagator(body, nb.MODE_STRICT, opts=nb.IntegratorOptions.default())
    st, cs, ep = hd.ensemble(body)
    return pyoracle.propagate_batch(prop.dynamics.pack(hd.FRAME[body], None).c, prop.opts.to_c(prop.method), st, cs, ep, hd.END)


@pytest.mark.parametrize("family", ("K1", "K2-G32"))
def test_strict_adaptive(oracle, family):
    """RK89 with the default controller (1e-12, RSSCartesianStep) at 96x96 on the lunar ensemble: status and epochs equal, at least
    90 % of the trajectories bit-equal (with equal step counts and next steps), the rest within 1e-6 km."""
    _, got = run("moon", nb.MODE_STRICT, family, opts=nb.IntegratorOptions.default())
    ref = _oracle_adaptive("moon")
    assert np.array_equal(got[3], ref[3]) and (got[3] == 0).all() and np.array_equal(got[1], ref[1])
    same = (got[0] == ref[0]).all(axis=0)
    print(f"STRICT adaptive {family}: {same.mean():.3f} bit-equal, max |dr| {max_dr_dv(got[0], ref[0])[0]:.2e}")
    assert same.mean() >= 0.9 and max_dr_dv(got[0], ref[0])[0] < 1e-6
    for f in ("n_steps", "step_ns"):
        assert np.array_equal(got[2][f][same], ref[2][f][same]), f


# ---- exactly polar start states
@pytest.mark.parametrize("family,mode", [("K1", "FAST"), ("K2-G32", "FAST"), ("K2-G8", "FAST"), ("K1", "STRICT"), ("K2-G32", "STRICT")],
                         ids=["K1-FAST", "K2-G32", "K2-G8", "K1-STRICT", "K3-G32"])
def test_exactly_polar_start_states(oracle, family, mode):
    """x = y = 0 in the body frame (identity rotation), at both poles, 30..300 km up, through one 1 ms RK4 step of the lunar 96x96
    field: STRICT bit-equal; FAST finite and within one or two ulps of the oracle's state (the harmonic part of the velocity change,
    ~1e-12 km/s, is a thousand times larger)."""
    m = MODES[mode]
    prop = nb.Propagator.new(hd.dynamics("moon"), nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(0.001), mode=m)
    packed, opts_c = prop.lower(nb.MOON_J2000, None)
    packed.c.gravity[0].rot.kind = 0
    eng = force_family(nb.Engine(packed, opts_c, m, 0), family)
    r_eq, mu = 1737.4, packed.c.mu_central_km3_s2
    st = np.zeros((9, 8))
    for i, (sign, alt, ang) in enumerate([(1, 30, 0), (-1, 30, 90), (1, 60, 45), (-1, 60, 200), (1, 100, 10), (-1, 150, 300),
                                          (1, 300, 135), (-1, 45, 270)]):
        r = r_eq + alt
        st[2, i] = sign * r
        st[3:5, i] = np.sqrt(mu / r) * np.array([np.cos(np.radians(ang)), np.sin(np.radians(ang))])
    cs = np.tile(np.array([[100.0], [0.0], [1.0], [1.0]]), (1, 8))
    ep = np.zeros(8, dtype=np.int64)
    got = eng.propagate_batch(st, cs, ep, 10**6)
    assert eng.last_kernel() == KERNEL[family[:2]]
    ref = oracle.propagate_batch(packed.c, opts_c, st, cs, ep, 10**6)
    assert np.isfinite(got[0]).all() and np.array_equal(got[1], ref[1]) and (got[3] == 0).all() and (ref[3] == 0).all()
    if mode == "STRICT":
        assert np.array_equal(got[0], ref[0]), max_dr_dv(got[0], ref[0])
    else:
        dr, dv = max_dr_dv(got[0], ref[0])
        assert dr < 1e-12 and dv < 1e-15, (dr, dv)


# ---- the edges of the range
def _field_engine(body, mode, degree, order=None):
    prop = hd.propagator(body, mode, degree, order)
    return nb.Engine(*prop.lower(hd.FRAME[body], None), mode, 0)


def test_degree_97_is_refused():
    c = np.zeros((98, 98))
    c[2, 0] = -2e-4
    gd = nb.GravityFieldData(97, 97, c, np.zeros((98, 98)), nb.IAU_MOON_FRAME)
    prop = nb.Propagator.new(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd))), hd.RK89,
                             nb.IntegratorOptions.with_fixed_step_s(60.0), mode=nb.MODE_FAST)
    packed, opts_c = prop.lower(nb.MOON_J2000, None)
    lib = abi.load_library()
    assert not lib.nyxb_engine_create(packed.byref(), C.byref(opts_c), nb.MODE_FAST, 0)
    assert "1..96" in abi.last_error()
    with pytest.raises(nb.PropagationError, match=r"1\.\.96"):
        nb.Engine(packed, opts_c, nb.MODE_FAST, 0)


def test_transposed_kernel_refused_above_degree_70():
    lib = abi.load_library()
    assert lib.nyxb_engine_set_kernel(_field_engine("moon", nb.MODE_FAST, 70).handle, nb.KERNEL_TRANSPOSED) == 0
    eng = _field_engine("moon", nb.MODE_FAST, 71)
    assert lib.nyxb_engine_set_kernel(eng.handle, nb.KERNEL_TRANSPOSED) == RC_UNSUPPORTED
    assert "8..70" in abi.last_error()


def test_auto_dispatch_at_degree_71_and_1024_trajectories():
    """1 024 trajectories would go to the transposed kernel up to degree 70; at 71 AUTO takes K2 at 32 lanes, and the result is
    the forced 32-lane run's bit for bit."""
    st, cs, ep = hd.ensemble("moon")
    idx = np.arange(1024) % st.shape[1]
    st, cs = st[:, idx].copy(), cs[:, idx].copy()
    st[:3] += np.random.default_rng(5).normal(0.0, 0.5, (3, 1024))
    ep = np.random.default_rng(6).integers(0, 600 * S, 1024).astype(np.int64)
    end = 1200 * S
    auto = _field_engine("moon", nb.MODE_FAST, 71)
    got = auto.propagate_batch(st, cs, ep, end)
    assert auto.last_kernel() == nb.KERNEL_COOP and auto.lanes() == 32
    forced = _field_engine("moon", nb.MODE_FAST, 71)
    forced.set_kernel(nb.KERNEL_COOP)
    forced.set_lanes(32)
    want = forced.propagate_batch(st, cs, ep, end)
    assert (got[3] == 0).all()
    for k in range(3):
        a, b = (got[k], want[k]) if k != 2 else (got[k].view(np.uint8), want[k].view(np.uint8))
        assert np.array_equal(a, b), k


@pytest.mark.parametrize("lanes,fits,refused", [(8, 50, 51), (16, 75, 76)])
def test_strict_lane_counts_whose_slab_does_not_fit_are_refused(lanes, fits, refused):
    """The STRICT cooperative kernel keeps each trajectory's Legendre triangle in shared memory: 8 lanes fit up to degree 50 and
    16 up to 75.  Above, nyxb_engine_set_lanes returns NYXB_RC_UNSUPPORTED with a message naming degree and lanes, before any
    launch, and leaves the setting alone; FAST (records in global memory) accepts them."""
    lib = abi.load_library()
    assert lib.nyxb_engine_set_lanes(_field_engine("moon", nb.MODE_STRICT, fits).handle, lanes) == 0
    eng = _field_engine("moon", nb.MODE_STRICT, refused)
    before = eng.lanes()
    assert lib.nyxb_engine_set_lanes(eng.handle, lanes) == RC_UNSUPPORTED
    msg = abi.last_error()
    assert f"degree-{refused}" in msg and f"{lanes} lanes" in msg, msg
    assert eng.lanes() == before == 32
    with pytest.raises(nb.PropagationError):
        eng.set_lanes(lanes)
    st, cs, ep = hd.ensemble("moon")
    got = eng.propagate_batch(st, cs, ep, 600 * S + int(ep.max()))
    assert (got[3] == 0).all() and eng.last_kernel() == nb.KERNEL_COOP
    assert lib.nyxb_engine_set_lanes(_field_engine("moon", nb.MODE_FAST, refused).handle, lanes) == 0


# ---- STM and filter kernels
STM_CASES = [("lunar", 96, 96), ("lunar", 96, 95), ("lunar", 81, 81), ("field", 96, 96)]


@pytest.mark.parametrize("config,degree,order", STM_CASES, ids=[f"{c}-{d}x{o}" for c, d, o in STM_CASES])
@pytest.mark.parametrize("mode", MODES)
def test_stm_high_degree(oracle, mode, config, degree, order):
    """STRICT without SRP ("field") bit-equal (assert_stm_parity)."""
    case = (config, om.METHOD, degree, order)
    assert_stm_parity(run_stm(mode, config, degree=degree, order=order), om.oracle_stm(*case), om.stm_bounds(*case),
                      f"{mode} {config} {degree}x{order}")


# (family, degree, order, columns per lane of the cooperative filter): 96x96 is the only four-column shape and takes four
# power-table passes; 96x95 has three columns and four passes; 95x95 three and three
FILTER_CASES = [("FAST-coop", 96, 96, 4), ("FAST-coop", 96, 95, 3), ("FAST-coop", 95, 95, 3), ("FAST-coop", 81, 81, 3),
                ("FAST-thread", 96, 96, None), ("STRICT", 96, 96, None)]


@pytest.mark.parametrize("family,degree,order,columns", FILTER_CASES, ids=[f"{f}-{d}x{o}" for f, d, o, _ in FILTER_CASES])
def test_filter_high_degree(oracle, family, degree, order, columns):
    if columns is not None:
        assert om.coop_columns_per_lane(degree, order) == columns
    check(family, "lunar", degree=degree, order=order)


def test_high_degree_shape_grid_covers_every_column_count():
    """With the shapes of tests/test_gpu_od_matrix.py, the cooperative filter runs one, two, three and four columns per lane."""
    coop = [(d, o) for f, _, d, o in SHAPE_CASES if f == "FAST-coop"] + [(d, o) for f, d, o, _ in FILTER_CASES if f == "FAST-coop"]
    assert {om.coop_columns_per_lane(d, o) for d, o in coop} == {1, 2, 3, 4}


def test_coop_against_per_thread_filter_at_degree_96(oracle):
    case = ("lunar", "ekf", "regular", 96, 96)
    coop = run_filters("FAST-coop", "lunar", degree=96, order=96)
    thread = run_filters("FAST-thread", "lunar", degree=96, order=96)
    as_ref = {"state": thread.final_state_soa, "covar": thread.covar, "state_dev": thread.state_deviation, "epoch": thread.final_epoch_ns,
              "resid_ratio": thread.resid_ratio, "prefit": thread.prefit, "postfit": thread.postfit, "msr_flags": thread.msr_flags,
              "est_state": thread.est_state, "est_covar_diag": thread.est_covar_diag, "n_steps": thread.details["n_steps"],
              "status": thread.status}
    tight = {k: v * COOP_VS_THREAD for k, v in om.filter_bounds(*case).items()}
    assert_filter_parity(coop, as_ref, tight, "coop-vs-thread lunar 96x96", om.SPREAD_FACTOR * COOP_VS_THREAD)
