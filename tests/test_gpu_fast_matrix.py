"""FAST-mode parity of every kernel family against the CPU oracle, force model by force model, integrator by integrator.

Families, each forced explicitly and checked with `last_kernel()`:
  K1          per-thread kernel, FAST column walk (grav_accel_cols)       set_kernel(KERNEL_THREAD)
  K2-G8/16/32 lane-cooperative kernel, 8 / 16 / 32 lanes per trajectory  set_lanes(G)
  K5-P8/10/16 transposed kernel, 8 / 10 / 16 walker positions per set    set_tx_positions(P)
  K5-sliced   transposed kernel, 5 attempts per time slice, one CTA (two set contexts for three sets): every set is parked and
              resumed many times                                           set_tx_tuning(5, 1)

Inputs: tests/fast_matrix.py (96 trajectories, per-lane constants and start epochs, JGM-3 21x21 in every configuration).

Fixed-step runs (part A): with a fixed step the step sequence cannot diverge, so the comparison measures the arithmetic.  Status,
epochs, n_steps, n_rhs and details.step_ns must be equal; |dr| < 5e-9 km and |dv| < 5e-12 km/s after 6 h (RK4 at 10 s:
5e-8 km, 5e-11 km/s).  The SRP and drag paths go through CUDA's acos / asin / exp / pow, which differ from glibc's in the last
ulp; the bounds hold with them.

Measured maxima on an H100 80GB HBM3 (SXM, 700 W power limit), RK89 at 60 s, |dr| km and |dv| km/s:

  family      field          third_body     srp            drag_constant  drag_exp.      drag_stdatm    all
  K1          2.0e-09 2e-12  1.5e-09 2e-12  2.6e-09 3e-12  1.6e-09 2e-12  1.7e-09 2e-12  2.1e-09 2e-12  3.1e-09 4e-12
  K2-G8       2.2e-09 3e-12  1.7e-09 2e-12  1.8e-09 2e-12  2.1e-09 2e-12  2.2e-09 3e-12  1.8e-09 2e-12  1.8e-09 2e-12
  K2-G16      2.2e-09 3e-12  1.7e-09 2e-12  1.8e-09 2e-12  2.1e-09 2e-12  1.9e-09 2e-12  1.8e-09 2e-12  1.8e-09 2e-12
  K2-G32      2.2e-09 3e-12  1.7e-09 2e-12  1.8e-09 2e-12  2.1e-09 2e-12  1.9e-09 2e-12  1.8e-09 2e-12  1.8e-09 2e-12
  K5-P8       1.9e-09 2e-12  1.7e-09 2e-12  1.6e-09 2e-12  1.7e-09 2e-12  2.0e-09 2e-12  1.7e-09 2e-12  1.9e-09 2e-12
  K5-P10      1.9e-09 2e-12  2.1e-09 2e-12  1.6e-09 2e-12  1.7e-09 2e-12  2.0e-09 2e-12  1.7e-09 2e-12  1.9e-09 2e-12
  K5-P16      1.9e-09 2e-12  1.8e-09 2e-12  1.6e-09 2e-12  1.7e-09 2e-12  2.0e-09 2e-12  1.7e-09 2e-12  1.9e-09 2e-12
  K5-sliced   1.9e-09 2e-12  1.7e-09 2e-12  1.6e-09 2e-12  1.7e-09 2e-12  2.0e-09 2e-12  1.7e-09 2e-12  1.9e-09 2e-12
Over every family: all methods at 45.5 s 3.5e-9 km / 4.1e-12 km/s, RK4 at 10 s 3.5e-9 / 3.9e-12, backward span 2.1e-9 / 2.5e-12,
field shapes 2.7e-9 / 3.2e-12, recorded states 3.1e-9 / 3.6e-12.  The whole file takes about 40 s on that card.

Adaptive runs (part C): the step sequences of GPU and oracle drift apart by the controller's rounding noise, so the bounds come from
the oracle's own sensitivity to that noise, computed on the same inputs:
    spread = max |oracle probe - oracle| over four probes: every error norm x (1 + 2^-52), x (1 - 2^-53), x (1 + 2^-50), and
             the oracle's speed build (FMA contraction)
    bound  = max(8 x spread, 10 x 5e-9 km)
The north-star cap of 1e-6 km is not applied: on this SRP + eclipse + StdAtm drag ensemble the oracle's spread alone reaches
1e-5 to 2e-4 km (a step boundary that moves across a shadow edge or the StdAtm branch altitude changes the step sequence that
follows), so a 1e-6 km cap would fail the reference algorithm against itself.  The GPU run is one more draw from the same
distribution as the probes: over the 126 cases x 4 calls, the largest GPU |dr| measured on the H100 above was 5.8 x the
four-probe spread (DP78, RSSCartesianStep, third call), hence the factor 8.
Status and epochs must be equal.  The step counts drift by the same noise: against its probes the oracle moves n_steps by up to
15 and n_rejected by up to 16 per trajectory (DP78 / RK89, LargestError, 1e-13 tolerance), so n_steps and n_rejected must agree
within max(1, 3 x the oracle's largest probe difference) of the same case (largest measured GPU difference: 2.2 x).

RK4 has no embedded error estimate (its error norm is 0): every attempt is accepted at the maximum step, so its runs use a 30 s
maximum step and cannot reject.  The controller powers x^(1/n) of the transposed kernel (tx_pow_inv_int) run for n = 9, 8, 6
and 5 on accepted steps and n = 8, 7, 5 and 4 on rejected ones."""
import functools

import numpy as np
import pytest

import nyx_b200 as nb
from tests import fast_matrix as fm
from tests.util import S, max_dr_dv

pytestmark = pytest.mark.gpu

RK89 = nb.IntegratorMethod.RungeKutta89
FAMILIES = ("K1", "K2-G8", "K2-G16", "K2-G32", "K5-P8", "K5-P10", "K5-P16", "K5-sliced")
KERNEL = {"K1": nb.KERNEL_THREAD, "K2": nb.KERNEL_COOP, "K5": nb.KERNEL_TRANSPOSED}


def family_engine(prop, family, alm=None):
    """A fresh engine of `prop` with the family forced."""
    return force_family(prop.engine(nb.EARTH_J2000, alm if alm is not None else fm.almanac()), family)


def force_family(eng, family):
    kind, _, arg = family.partition("-")
    if kind == "K1":
        eng.set_kernel(nb.KERNEL_THREAD)
    elif kind == "K2":
        eng.set_kernel(nb.KERNEL_COOP)
        if arg:
            eng.set_lanes(int(arg[1:]))
    else:
        eng.set_kernel(nb.KERNEL_TRANSPOSED)
        if arg == "sliced":
            eng.set_tx_tuning(5, 1)
        elif arg:
            eng.set_tx_positions(int(arg[1:]))
    return eng


def run_family(prop, family, st, cs, ep, end, **kw):
    eng = family_engine(prop, family)
    got = eng.propagate_batch(st, cs, ep, end, **kw)
    assert eng.last_kernel() == KERNEL[family[:2]], (family, eng.last_kernel())
    return eng, got


def assert_fixed_parity(got, ref, method, tag, bounds=None):
    out, out_ep, det, status = got[:4]
    r, r_ep, r_det, r_status = ref[:4]
    assert np.array_equal(status, r_status) and (status == 0).all(), (tag, status)
    assert np.array_equal(out_ep, r_ep), tag
    for f in ("n_steps", "n_rhs", "step_ns"):
        assert np.array_equal(det[f], r_det[f]), (tag, f)
    dr, dv = max_dr_dv(out, r)
    print(f"FASTMATRIX {tag} dr={dr:.3e} dv={dv:.3e}")
    bdr, bdv = bounds or fm.bounds(method)
    assert dr < bdr and dv < bdv, (tag, dr, dv)
    return dr, dv


# ---- A: every family x every configuration, RK89 at 60 s
@pytest.mark.parametrize("config", fm.CONFIGS)
@pytest.mark.parametrize("family", FAMILIES)
def test_fixed_step_configurations(oracle, family, config):
    st, cs, ep = fm.ensemble()
    ref = fm.oracle_fixed(config)
    _, got = run_family(fm.propagator(config), family, st, cs, ep, fm.END)
    assert_fixed_parity(got, ref, RK89, f"{family} {config}")


# ---- A: every family x every method on the full configuration (short final step), plus a backward span
@pytest.mark.parametrize("method", fm.METHODS, ids=lambda m: m.name)
@pytest.mark.parametrize("family", FAMILIES)
def test_fixed_step_methods(oracle, family, method):
    st, cs, ep = fm.ensemble()
    step = fm.method_step_s(method)
    ref = fm.oracle_fixed("all", method, step)
    prop = fm.propagator("all", method, nb.IntegratorOptions.with_fixed_step_s(step))
    _, got = run_family(prop, family, st, cs, ep, fm.END)
    assert_fixed_parity(got, ref, method, f"{family} all {method.name}")


@pytest.mark.parametrize("family", FAMILIES)
def test_fixed_step_backward(oracle, family):
    """From the oracle's 6 h state back to epoch 0 (a span of 5.3 - 6 h, negative fixed steps, a short final step)."""
    fwd = ("all", RK89, 60.0)
    ref = fm.oracle_fixed("all", RK89, 60.0, start=fwd, end=0)
    st0, ep0 = fm.oracle_fixed(*fwd)[:2]
    _, got = run_family(fm.propagator("all"), family, st0, fm.ensemble()[1], ep0, 0)
    assert (got[1] == 0).all()
    assert_fixed_parity(got, ref, RK89, f"{family} all backward")


# ---- A: field shapes where the kernels switch code paths (configuration "third_body")
SHAPES = [("K1", 6, 6), ("K1", 7, 7), ("K1", 21, 21),
          ("K2-G8", 8, 0), ("K2-G8", 8, 1), ("K2", 29, 29), ("K2", 30, 30), ("K2", 47, 47), ("K2", 48, 48), ("K2-G32", 70, 70),
          ("K5-P8", 8, 0), ("K5-P8", 8, 1), ("K5-P8", 40, 40), ("K5-P16", 41, 41), ("K5", 40, 40), ("K5", 41, 41), ("K5", 70, 70)]


@pytest.mark.parametrize("family,degree,order", SHAPES, ids=[f"{f}-{d}x{o}" for f, d, o in SHAPES])
def test_fixed_step_field_shapes(oracle, family, degree, order):
    """"K2" / "K5" without a suffix: the family's own choice of lanes (8 below degree 30, 16 below 48, 32 from 48; K2 at 70x70
    keeps its record table in global memory) or walker positions (8 up to degree 40, 16 above)."""
    st, cs, ep = fm.ensemble()
    ref = fm.oracle_fixed("third_body", degree=degree, order=order)
    eng, got = run_family(fm.propagator("third_body", degree=degree, order=order), family, st, cs, ep, fm.END)
    if family == "K2":
        assert eng.lanes() == (8 if degree < 30 else 16 if degree < 48 else 32)
    assert_fixed_parity(got, ref, RK89, f"{family} {degree}x{order}")


# ---- D: fixed-step recordings, every family
@pytest.mark.parametrize("family", FAMILIES)
def test_fixed_step_recording(oracle, family):
    """Record counts and epochs equal to the oracle's; every recorded state within the fixed-step bound (pins that the transposed
    kernel's controller, which writes the epochs, and its component warps, which write the states, agree on the index)."""
    cap = 400
    st, cs, ep = fm.ensemble()
    ref = fm.oracle_fixed("all", traj_capacity=cap)
    _, got = run_family(fm.propagator("all"), family, st, cs, ep, fm.END, traj_capacity=cap)
    assert_fixed_parity(got, ref, RK89, f"{family} all recording")
    (g_ep, g_st, g_cnt), (o_ep, o_st, o_cnt) = got[4], ref[4]
    assert np.array_equal(g_cnt, o_cnt) and np.array_equal(g_cnt, got[2]["n_steps"] + 1)
    assert np.array_equal(g_ep, o_ep)
    d = g_st - o_st
    dr = np.sqrt((d[:3] ** 2).sum(0)).max()
    dv = np.sqrt((d[3:6] ** 2).sum(0)).max()
    print(f"FASTMATRIX {family} all records dr={dr:.3e} dv={dv:.3e}")
    assert dr < fm.FIXED_DR and dv < fm.FIXED_DV, (dr, dv)


def test_transposed_recording_overflow_under_time_slicing(oracle):
    """Capacity overflow on the transposed kernel while sets are parked and resumed: the head of the stream is kept, the count is
    the capacity, the final states are those of the run that recorded everything."""
    st, cs, ep = fm.ensemble()
    eng, full = run_family(fm.propagator("all"), "K5-sliced", st, cs, ep, fm.END, traj_capacity=400)
    small = eng.propagate_batch(st, cs, ep, fm.END, traj_capacity=37)
    assert eng.last_kernel() == nb.KERNEL_TRANSPOSED
    assert (small[4][2] == 37).all()
    assert np.array_equal(small[4][0], full[4][0][:37]) and np.array_equal(small[4][1], full[4][1][:, :37])
    assert np.array_equal(small[0], full[0]) and np.array_equal(small[1], full[1]) and np.array_equal(small[3], full[3])


# ---- C: adaptive sweep, methods x error controls x families
ADAPTIVE_N = 48
SPANS = (5400 * S, 1800 * S, 7200 * S)
ERROR_SCALES = (1.0 + 2.0**-52, 1.0 - 2.0**-53, 1.0 + 2.0**-50)   # one-ulp-sized perturbations of every error norm    # forward, backward, forward again, the adapted step carried between the calls


def _adaptive_cases(method, ctrl):
    """(options, targets) of the two runs of one case: a chained forward / backward / forward run, and a one-hour run that starts
    with a 600 s step at a 1e-13 tolerance, so that the first attempts are rejected."""
    chained = nb.IntegratorOptions.with_adaptive_step_s(0.1, 120.0, 1e-10, ctrl)
    chained.init_step = 30 * nb.Unit.Second
    rejecting = nb.IntegratorOptions(init_step=600 * nb.Unit.Second, tolerance=1e-13, error_ctrl=ctrl)
    if method == nb.IntegratorMethod.RungeKutta4:
        chained.max_step = rejecting.max_step = rejecting.init_step = 30 * nb.Unit.Second
    return ((chained, SPANS), (rejecting, (3600 * S,)))


def _adaptive_inputs():
    st, cs, ep = fm.ensemble()
    idx = np.r_[0:32, 64:80]   # 32 LEO + 16 eccentric
    return st[:, idx].copy(), cs[:, idx].copy(), ep[idx].copy()


def _chain(run, st, cs, ep, targets, step0):
    """[(state, epoch, details, status, step)] after every call of a chained run"""
    step = np.full(st.shape[1], step0, dtype=np.int64)
    res, cur, cep = [], st, ep
    for t in targets:
        cur, cep, det, status = run(cur, cs, cep, t, step)[:4]
        res.append((cur, cep, det, status, step.copy()))
    return res


@functools.lru_cache(maxsize=None)
def _adaptive_reference(method, ctrl):
    """Per run: the oracle's chain and, per call, the position bound and the step-count bound from the oracle's own step-sequence
    sensitivity (module header)."""
    from oracle import pyoracle

    st, cs, ep = _adaptive_inputs()
    alm = fm.almanac()
    out = []
    for opts, targets in _adaptive_cases(method, ctrl):
        prop = nb.Propagator.new(fm.dynamics("all"), method, opts, mode=nb.MODE_FAST)
        packed, oc = prop.dynamics.pack(nb.EARTH_J2000, alm), opts.to_c(method)

        def orun(speed=False):
            return lambda a, b, c, t, step: pyoracle.propagate_batch(packed.c, oc, a, b, c, t, step, speed_build=speed)

        plain = _chain(orun(), st, cs, ep, targets, opts.init_step)
        probes = [_chain(orun(True), st, cs, ep, targets, opts.init_step)]
        for scale in ERROR_SCALES:
            pyoracle.set_error_scale(scale)
            try:
                probes.append(_chain(orun(), st, cs, ep, targets, opts.init_step))
            finally:
                pyoracle.set_error_scale(1.0)
        bounds = []
        for k, p in enumerate(plain):
            spread = max(max_dr_dv(p[0], q[k][0])[0] for q in probes)
            counts = {f: max(1, 3 * max(int(np.abs(p[2][f] - q[k][2][f]).max()) for q in probes)) for f in ("n_steps", "n_rejected")}
            bounds.append((max(8.0 * spread, 10 * fm.FIXED_DR), counts))
        out.append((plain, bounds))
    return out


@pytest.mark.parametrize("ctrl", list(nb.ErrorControl), ids=lambda c: c.name)
@pytest.mark.parametrize("method", fm.METHODS, ids=lambda m: m.name)
@pytest.mark.parametrize("family", ("K1", "K2-G8", "K5-P8"))
def test_adaptive_methods_and_error_controls(oracle, family, method, ctrl):
    st, cs, ep = _adaptive_inputs()
    for (opts, targets), (ref, bounds) in zip(_adaptive_cases(method, ctrl), _adaptive_reference(method, ctrl)):
        prop = nb.Propagator.new(fm.dynamics("all"), method, opts, mode=nb.MODE_FAST)
        eng = family_engine(prop, family)
        got = _chain(eng.propagate_batch, st, cs, ep, targets, opts.init_step)
        assert eng.last_kernel() == KERNEL[family[:2]]
        for k, (g, r, (bound, counts)) in enumerate(zip(got, ref, bounds)):
            tag = f"{family} {method.name} {ctrl.name} opts{opts.init_step // S}s call{k}"
            assert np.array_equal(g[3], r[3]) and (g[3] == 0).all(), (tag, g[3])
            assert np.array_equal(g[1], r[1]), tag
            for f in ("n_steps", "n_rejected"):
                assert np.abs(g[2][f] - r[2][f]).max() <= counts[f], (tag, f, np.abs(g[2][f] - r[2][f]).max(), counts[f])
            dr = max_dr_dv(g[0], r[0])[0]
            print(f"FASTMATRIX adaptive {tag} dr={dr:.3e} bound={bound:.3e} ratio={dr / bound:.3f} "
                  f"dsteps={int(np.abs(g[2]['n_steps'] - r[2]['n_steps']).max())}/{counts['n_steps']} "
                  f"drej={int(np.abs(g[2]['n_rejected'] - r[2]['n_rejected']).max())}/{counts['n_rejected']}")
            assert dr < bound, (tag, dr, bound)
        if opts.tolerance == 1e-13 and method != nb.IntegratorMethod.RungeKutta4:
            assert got[0][2]["n_rejected"].sum() > 0
