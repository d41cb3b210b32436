"""Parity of the STM propagation kernel and of both Kalman-filter kernels against the CPU oracle at fixed step, per output the C ABI
returns (oracle/pyoracle_od.process_arc, oracle.propagate_batch_stm).

Filter families, each forced explicitly and checked with `last_kernel()`:
  STRICT       per-thread filter (nyxb_od.cu), STRICT arithmetic
  FAST-thread  per-thread filter, FAST arithmetic                       set_kernel(KERNEL_THREAD)
  FAST-coop    warp-cooperative filter (nyxb_od_coop.cu), the FAST default for a field of degree >= 8
STM: nyxb_propagate_batch_stm, STRICT and FAST (one thread per trajectory).

Inputs: tests/od_matrix.py (13 filters over a 48-measurement arc and the edge-case arc, four force-model configurations, EKF / CKF,
msr_size 1 / 2, rejection on / off, SNC in RIC and in the integration frame with both disable branches, field shapes from 8x0 to
Luna 80x80; 32 STM trajectories with per-trajectory epochs, masses, SRP areas and Cr).

Exactly equal: status, final epochs, msr_flags, n_steps, and the NaN pattern of every per-measurement record.  Within bounds: final
state and est_state at every measurement, the final covariance entry by entry at correlation scale |dP_ij| / sqrt(P_ii P_jj),
est_covar_diag (relative), the CKF state deviation, residual ratios, prefit and postfit residuals; STM blocks rr, rv, vr, vv and the
Cr column per trajectory, relative to that trajectory's own block (STRICT STM propagation without SRP: bit-equal).  The bound of each quantity
is 10 x the spread of the oracle
against its FMA build and against its numpy filter with every matrix product summed in reverse order, computed on the same case
(od_matrix.filter_bounds), with a floor.  The two FAST filter kernels are compared with each other at 3 x the spread.

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), largest ratio GPU difference / oracle spread per family and quantity
(the bound is 10):

  family       dr   dv   est_dr est_dv Cr   covar est_covar state_dev ratio prefit km  postfit km  prefit km/s postfit km/s
  STRICT       1.3  1.2  1.7    1.9    1.1  1.6   2.1       1.1       1.6   1.7        1.4         1.2         0.97
  FAST-thread  1.1  1.4  1.7    1.7    2.0  2.0   1.6       1.9       1.4   1.3        1.5         1.1         1.3
  FAST-coop    1.4  1.4  1.7    1.7    2.0  2.9   1.9       1.7       1.4   1.3        1.5         1.1         1.3
  coop/thread  0.75 0.68 0.48   0.65   0.14 1.0   1.5       1.0       0.89  0.69       0.89        0.14        0.32   (bound 3)
  STM          dr   dv   rr   rv   vr   vv   Cr column
  FAST         1.6  1.5  1.1  0.69 1.1  0.81 1.3
  STRICT, SRP  0.11 0.064 0.051 0.064 0.11 0.081 1.6     (without SRP: bit-equal)
The typical spread is 1e-11 km on the Earth arcs and 1e-9 km on the Moon-centred arc; the whole file takes about 2.5 min on that
card, most of it in the oracle."""
import numpy as np
import pytest

import nyx_b200 as nb
from tests import od_matrix as om

pytestmark = pytest.mark.gpu

FAMILIES = ("STRICT", "FAST-thread", "FAST-coop")
COOP_VS_THREAD = 0.3


def run_filters(family, config, variant="ekf", arc_kind="regular", degree=21, order=None):
    mode = nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST
    prop = om.propagator(config, mode, degree, order)
    _, cfg, names, st_c, epochs, tracker, obs, st, cs, ep, cov = om.od_inputs(config, variant, arc_kind, prop)
    eng = prop.engine(om.frame(config), om.almanac(config))
    eng.set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    sol = eng.od_ekf_batch(cfg, len(names), st_c, epochs, tracker, obs, st, cs, ep, cov, record_estimates=True)
    assert eng.last_kernel() == (nb.KERNEL_COOP if family == "FAST-coop" else nb.KERNEL_THREAD), (family, eng.last_kernel())
    return sol


def assert_filter_parity(sol, ref, bounds, tag, spreads_per_bound=om.SPREAD_FACTOR):
    assert (ref["status"] == 0).all() and np.array_equal(sol.status, ref["status"]), (tag, sol.status)
    assert np.array_equal(sol.final_epoch_ns, ref["epoch"]), tag
    assert np.array_equal(sol.msr_flags, ref["msr_flags"]), (tag, np.argwhere(sol.msr_flags != ref["msr_flags"]))
    assert np.array_equal(sol.details["n_steps"], ref["n_steps"]), tag
    for f, g in (("est_state", sol.est_state), ("est_covar_diag", sol.est_covar_diag), ("resid_ratio", sol.resid_ratio),
                 ("prefit", sol.prefit), ("postfit", sol.postfit)):
        assert np.array_equal(np.isnan(g), np.isnan(ref[f])), (tag, f)
    d = np.sqrt(np.abs(np.einsum("nii->ni", ref["covar"])))
    dead = (d[:, :, None] * d[:, None, :]) == 0
    assert (sol.covar[dead] == ref["covar"][dead]).all(), tag       # Cd and mass rows stay exactly zero
    err = om.filter_errors(sol, ref)
    worst = max(err, key=lambda k: err[k] / bounds[k])
    print(f"ODMATRIX {tag} worst={worst} ratio_to_spread=" + " ".join(
        f"{k}={err[k] / (bounds[k] / spreads_per_bound):.2g}" for k in err))
    bad = {k: (err[k], bounds[k]) for k in err if not err[k] <= bounds[k]}
    assert not bad, (tag, bad)


def check(family, config, variant="ekf", arc_kind="regular", degree=21, order=None):
    case = (config, variant, arc_kind, degree, order)
    ref = om.oracle_filters(*case)
    sol = run_filters(family, config, variant, arc_kind, degree, order)
    assert_filter_parity(sol, ref, om.filter_bounds(*case), f"{family} {config} {variant} {arc_kind} {degree}x{order or degree}")
    return sol


# ---- filters: every family x every configuration (EKF, msr_size 2, 3-sigma rejection, SNC in RIC)
@pytest.mark.parametrize("config", om.CONFIGS)
@pytest.mark.parametrize("family", FAMILIES)
def test_filter_configurations(oracle, family, config):
    check(family, config)


# ---- filters: every family x the other filter settings, on the SRP configuration
@pytest.mark.parametrize("variant", [v for v in om.VARIANTS if v != "ekf"])
@pytest.mark.parametrize("family", FAMILIES)
def test_filter_variants(oracle, family, variant):
    sol = check(family, "srp", variant)
    if om.VARIANTS[variant][0] == om.CKF:
        assert np.abs(sol.state_deviation[:3]).max() > 0.0


@pytest.mark.parametrize("family", FAMILIES)
def test_filter_edge_case_arc(oracle, family):
    check(family, "srp", arc_kind="edge")


# ---- filters: field shapes where the cooperative kernel's column deal and power-table passes switch; truncated fields on every family
SHAPE_CASES = [("FAST-coop", *s) for s in om.SHAPES] + [
    ("FAST-thread", "field", 8, 1), ("FAST-thread", "field", 21, 4), ("FAST-thread", "field", 32, 32),
    ("STRICT", "field", 8, 1), ("STRICT", "field", 21, 4)]


@pytest.mark.parametrize("family,config,degree,order", SHAPE_CASES, ids=[f"{f}-{c}-{d}x{o}" for f, c, d, o in SHAPE_CASES])
def test_filter_field_shapes(oracle, family, config, degree, order):
    check(family, config, degree=degree, order=order)


def test_shape_grid_covers_every_column_count():
    """One, two and three columns per lane in the cooperative cases, and a truncated field (order < degree) on each family."""
    assert {om.coop_columns_per_lane(d, o) for f, _, d, o in SHAPE_CASES if f == "FAST-coop"} == {1, 2, 3}
    assert {f for f, _, d, o in SHAPE_CASES if o < d} == set(FAMILIES)


# ---- the two FAST filter kernels against each other
COOP_PAIRS = [("srp", 21, None), ("lunar", 21, None), ("field", 8, 1), ("field", 32, 32), ("field", 64, 64)]


@pytest.mark.parametrize("config,degree,order", COOP_PAIRS, ids=[f"{c}-{d}x{o or d}" for c, d, o in COOP_PAIRS])
def test_coop_against_per_thread_filter(oracle, config, degree, order):
    case = (config, "ekf", "regular", degree, order)
    coop = run_filters("FAST-coop", config, degree=degree, order=order)
    thread = run_filters("FAST-thread", config, degree=degree, order=order)
    as_ref = {"state": thread.final_state_soa, "covar": thread.covar, "state_dev": thread.state_deviation, "epoch": thread.final_epoch_ns,
              "resid_ratio": thread.resid_ratio, "prefit": thread.prefit, "postfit": thread.postfit, "msr_flags": thread.msr_flags,
              "est_state": thread.est_state, "est_covar_diag": thread.est_covar_diag, "n_steps": thread.details["n_steps"],
              "status": thread.status}
    tight = {k: v * COOP_VS_THREAD for k, v in om.filter_bounds(*case).items()}
    assert_filter_parity(coop, as_ref, tight, f"coop-vs-thread {config} {degree}x{order or degree}", om.SPREAD_FACTOR * COOP_VS_THREAD)


# ---- STM propagation, STRICT and FAST
MODES = {"STRICT": nb.MODE_STRICT, "FAST": nb.MODE_FAST}


def run_stm(mode, config, method=om.METHOD, degree=21, order=None, st=None, ep=None, end=om.STM_END, **kw):
    prop = om.propagator(config, MODES[mode], degree, order, method=method, step_s=om.stm_step(method))
    st0, cs, ep0 = om.stm_ensemble(config)
    eng = prop.engine(om.frame(config), om.almanac(config))
    got = eng.propagate_batch_stm(st0 if st is None else st, cs, ep0 if ep is None else ep, end, **kw)
    assert eng.last_kernel() == nb.KERNEL_THREAD
    return got


def assert_stm_parity(got, ref, bounds, tag):
    out, oep, stm, det, status = got
    assert (status == 0).all() and np.array_equal(status, ref[4]), (tag, status)
    assert np.array_equal(oep, ref[1]), tag
    assert np.array_equal(det["n_steps"], ref[3]["n_steps"]) and np.array_equal(det["n_rhs"], ref[3]["n_rhs"]), tag
    A = stm.T.reshape(-1, 9, 9).transpose(0, 2, 1)
    B = ref[2].T.reshape(-1, 9, 9).transpose(0, 2, 1)
    assert np.array_equal(A[:, 6:, :], B[:, 6:, :]) and np.array_equal(A[:, :6, 7:], B[:, :6, 7:]), tag
    err = om.stm_errors(got, ref)
    # STRICT is the oracle's arithmetic bit for bit, except that the shadow geometry goes through CUDA's acos / asin
    if tag.startswith("STRICT") and tag.split()[1] in ("field", "third_body"):
        assert np.array_equal(out, ref[0]) and np.array_equal(stm, ref[2]), tag
    print(f"ODMATRIX STM {tag} ratio_to_spread=" + " ".join(f"{k}={err[k] / (bounds[k] / om.SPREAD_FACTOR):.2g}" for k in err)
          + " abs=" + " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    bad = {k: (err[k], bounds[k]) for k in err if not err[k] <= bounds[k]}
    assert not bad, (tag, bad)


@pytest.mark.parametrize("config", om.STM_CONFIGS)
@pytest.mark.parametrize("mode", MODES)
def test_stm_configurations(oracle, mode, config):
    got = run_stm(mode, config)
    assert_stm_parity(got, om.oracle_stm(config), om.stm_bounds(config), f"{mode} {config}")
    if config in ("srp", "lunar"):
        assert np.abs(got[2][6 * 9: 6 * 9 + 6]).max() > 0.0      # the Cr column is live


@pytest.mark.parametrize("method", list(nb.IntegratorMethod), ids=lambda m: m.name)
@pytest.mark.parametrize("mode", MODES)
def test_stm_methods(oracle, mode, method):
    assert_stm_parity(run_stm(mode, "srp", method), om.oracle_stm("srp", method), om.stm_bounds("srp", method), f"{mode} srp {method.name}")


@pytest.mark.parametrize("mode", MODES)
def test_stm_backward(oracle, mode):
    st, ep = om.oracle_stm("srp")[:2]
    got = run_stm(mode, "srp", st=st, ep=ep, end=0)
    assert (got[1] == 0).all()
    case = ("srp", om.METHOD, 21, None, om.STM_END, True)
    assert_stm_parity(got, om.oracle_stm(*case), om.stm_bounds(*case), f"{mode} srp backward")


@pytest.mark.parametrize("mode", MODES)
def test_stm_split_run_equals_one_run(oracle, mode):
    """Two halves chained through stm_in and step_ns give the one-run answer bit for bit (all trajectories start at epoch 0 so the
    midpoint, 40 fixed steps, lies on every trajectory's step grid)."""
    st, cs, _ = om.stm_ensemble("srp")
    ep = np.zeros(st.shape[1], dtype=np.int64)
    step = np.full(st.shape[1], int(om.STEP_S * om.S), dtype=np.int64)
    mid, end = 40 * int(om.STEP_S * om.S), om.STM_END
    one = run_stm(mode, "srp", st=st, ep=ep, end=end)
    h1 = run_stm(mode, "srp", st=st, ep=ep, end=mid, step_ns=step)
    assert (h1[1] == mid).all() and (step == int(om.STEP_S * om.S)).all()
    h2 = run_stm(mode, "srp", st=h1[0], ep=h1[1], end=end, stm_in=h1[2], step_ns=step)
    for k in (0, 1, 2):
        assert np.array_equal(h2[k], one[k]), (mode, k)
    assert np.array_equal(h1[3]["n_steps"] + h2[3]["n_steps"], one[3]["n_steps"])


STM_SHAPES = [("field", 8, 0), ("field", 8, 1), ("field", 21, 4), ("field", 32, 32), ("field", 64, 64), ("field", 70, 70), ("lunar", 80, 80)]


@pytest.mark.parametrize("config,degree,order", STM_SHAPES, ids=[f"{c}-{d}x{o}" for c, d, o in STM_SHAPES])
@pytest.mark.parametrize("mode", MODES)
def test_stm_field_shapes(oracle, mode, config, degree, order):
    case = (config, om.METHOD, degree, order)
    assert_stm_parity(run_stm(mode, config, degree=degree, order=order), om.oracle_stm(*case), om.stm_bounds(*case),
                      f"{mode} {config} {degree}x{order}")
