"""CPU checks of the edge-of-span catalogue (tests/span_edges.py) that the GPU file (tests/test_gpu_span_edges.py) relies on:

  - the oracle agrees with the exact integer model on every call of every case: final epoch, the step array handed back (with its
    sign), details.step_ns, n_steps, n_rejected, attempts, the WARN_MAX_ATTEMPTS bit, the recorded epochs and their count, for the
    plain propagation and for the STM propagation, and the record epochs of the covariance prediction;
  - every case reaches the branch it is named for, shown with the oracle's own counters;
  - the oracle's distance from a 40-digit Kepler solution on every two-body case (the GPU bounds are derived from it);
  - a STRICT two-body run gives the same bits for every shift of its start epochs (the dynamics are autonomous)."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import span_edges as se

FIELDS = ("epoch", "step", "det_step", "attempts", "n_steps", "n_rejected", "warn")


def observed(ret, step, k, i):
    """the model's fields of trajectory i after call k, read from one chained run"""
    _, ep, det, status = ret[:4]
    return dict(epoch=int(ep[i]), step=int(step[i]), det_step=int(det["step_ns"][i]), attempts=int(det["attempts"][i]),
                n_steps=int(det["n_steps"][i]), n_rejected=int(det["n_rejected"][i]), warn=bool(status[i] & abi.WARN_MAX_ATTEMPTS))


def assert_matches_model(case, runs, with_records=True):
    for k, (call, (st, ep, det, status, step, rec)) in enumerate(zip(se.model(case), runs)):
        assert (status & 0xFF == 0).all(), (case.name, k, status)
        for i, m in enumerate(call):
            got = observed((st, ep, det, status), step, k, i)
            assert got == {f: m[f] for f in FIELDS}, (case.name, k, i, got, m)
            if with_records:
                cnt = int(rec[2][i])
                assert cnt == len(m["records"]) and rec[0][:cnt, i].tolist() == m["records"], (case.name, k, i)


@pytest.mark.parametrize("name", list(se.CASE))
def test_oracle_matches_integer_model(oracle, name):
    assert_matches_model(se.CASE[name], se.oracle_chain(name))


@pytest.mark.parametrize("name", list(se.CASE))
def test_oracle_stm_matches_integer_model(oracle, name):
    """The STM propagation of the oracle (the OD path's reference) keeps the same bookkeeping."""
    assert_matches_model(se.CASE[name], se.oracle_stm_chain(name), with_records=False)


def _branch_reached(case, runs):
    """the predicate of BRANCHES[case.branch] on the oracle's counters"""
    o = case.opts()
    step0 = case.first_step()
    spans = np.array(case.spans(), dtype=np.int64)
    st0, ep0, det0, status0, step_after0, rec0 = runs[0]
    n0, ds0 = det0["n_steps"], det0["step_ns"]
    diffs = [np.diff(rec0[0][: int(rec0[2][i]), i]) for i in range(case.size)]
    b = case.branch
    if b == "cut_first":
        return ((n0 == 1) & (np.abs(ds0) < abs(step0)) & (spans != 0)).any()
    if b == "stop_eq_epoch":
        hit = (spans > 0) & (spans % step0 == 0) & (ds0 == step0) & (n0 == spans // step0)
        return hit.any()
    if b == "cut_1ns":
        return any((np.abs(r[2]["step_ns"]) == 1).any() and (r[2]["n_steps"][np.abs(r[2]["step_ns"]) == 1] > 1).any() for r in runs)
    if b == "cut":
        return ((n0 > 1) & (np.abs(ds0) > 0) & (np.abs(ds0) < abs(step0))).any()
    if b == "back_boundary_then_fwd":
        hit = (spans < 0) & (spans % step0 == 0) & (ds0 == -step0) & (step_after0 == step0)
        return hit.any() and (runs[1][2]["n_steps"][hit] > 0).all() and (runs[1][1][hit] > runs[0][1][hit]).all()
    if b == "forced_min":
        adapt = n0 >= 2
        return (adapt & (det0["n_rejected"] == 0) & (np.abs(step_after0) == int(o.min_step))).any() and not (status0 & abi.WARN_MAX_ATTEMPTS).any()
    if b == "init_below_min":
        return any(len(d) > 1 and d[0] == int(o.init_step) and abs(d[1]) == int(o.min_step) for d in diffs)
    if b == "init_above_span":
        return ((n0 == 1) & (np.abs(spans) < int(o.init_step)) & (spans != 0) & (step_after0 == int(o.init_step))).any()
    if b == "span_below_min":
        return ((n0 == 1) & (np.abs(ds0) < int(o.min_step)) & (spans != 0)).any()
    if b == "step_carried":
        return (step_after0 != step0).any() and all((r[2]["n_steps"] > 0).any() for r in runs[1:])
    if b == "max_attempts":
        return ((status0 & abi.WARN_MAX_ATTEMPTS) != 0).any() and (det0["n_rejected"] == 0).all() and o.attempts == 1
    if b == "forced_min_rejected":
        return ((det0["n_rejected"] > 0) & (np.abs(step_after0) == int(o.min_step))).any()
    if b == "clamp_max":
        return (np.abs(step_after0) == int(o.max_step)).any() and any((d[:-1] == -int(o.max_step)).any() for d in diffs)
    if b == "lossy_step":
        return any(len(d) > 2 and (d[:-1] != abs(int(step_after0[i]))).any() for i, d in enumerate(diffs))
    if b == "saturating_max":
        return (step_after0 == se.INT64_MAX).any()
    if b == "negative_century":
        return (ep0 < -se.YEAR).all() and (case.epoch0() < -se.YEAR).all() and (n0 > 0).any()
    if b == "far_epoch":
        return (case.epoch0() > 50 * se.YEAR).all() and (n0 > 0).any()
    if b == "century_boundary":
        e0 = case.epoch0()
        below, above = e0 == case.t0 - 1, e0 == case.t0 + 1
        return below.any() and above.any() and (n0[below] > 0).all() and (n0[above] > 0).all()
    raise AssertionError(b)


@pytest.mark.parametrize("name", list(se.CASE))
def test_case_reaches_its_branch(oracle, name):
    case = se.CASE[name]
    runs = se.oracle_chain(name)
    det0 = runs[0][2]
    print(f"SPANEDGES {name} branch={case.branch} n={case.size} n_steps={int(det0['n_steps'].sum())} "
          f"n_rejected={int(det0['n_rejected'].sum())} max_attempts={int(det0['attempts'].max())} "
          f"warn={int(((runs[0][3] & abi.WARN_MAX_ATTEMPTS) != 0).sum())}")
    assert _branch_reached(case, runs), (name, se.BRANCHES[case.branch])
    # every ensemble mixes trajectories already at their end epoch with ones that run
    assert (np.array(case.spans()) == 0).any() or case.size == 1
    assert (runs[0][2]["n_steps"] > 0).any()


def test_catalogue_covers_every_branch_and_size():
    assert {c.branch for c in se.CASES} == set(se.BRANCHES)
    assert {c.size for c in se.CASES} == set(se.SIZES) - {1}
    assert {c.control for c in se.CASES} == {"fixed", "minmax", "unmet", "huge"}
    assert {c.attempts for c in se.CASES if c.control == "unmet"} >= {1, 255}


@pytest.mark.parametrize("name", se.KEPLER_CASES)
def test_oracle_distance_from_kepler(oracle, name):
    """Recorded per case; the GPU's two-body results are held to twice this distance (at least this distance plus the FAST
    fixed-step parity bound)."""
    d = se.kepler_distance(name, se.oracle_chain(name)[-1][0])
    print(f"SPANEDGES kepler {name}: oracle |dr| = {d:.3e} km, GPU bound {se.kepler_bound(name):.3e} km")
    assert d < 1e-5, (name, d)     # the largest: DP45 at 45 s over 4 min, 6.9e-6 km


def test_kepler_reference_closes_an_orbit():
    """The 40-digit reference itself: one period brings the state back, half a period and back again too."""
    st, _ = se.ensemble(33)
    r0, v0 = st[:3, 0], st[3:6, 0]
    a = 1.0 / (2.0 / np.linalg.norm(r0) - v0 @ v0 / se.TWOBODY_MU)
    period_ns = int(round(2 * np.pi * np.sqrt(a**3 / se.TWOBODY_MU) * 1e9))
    r, v = se.kepler(r0, v0, period_ns)
    assert np.abs(r - r0).max() < 1e-5 and np.abs(v - v0).max() < 1e-8     # 1 ns of rounding of the period: 7.7e-6 km
    rh, vh = se.kepler(r0, v0, period_ns // 2)
    rb, vb = se.kepler(rh, vh, -(period_ns // 2))
    assert np.abs(rb - r0).max() < 1e-9 and np.abs(vb - v0).max() < 1e-12


@pytest.mark.parametrize("name", [n for n in se.TWOBODY_CASES if n != "huge_saturating"])
def test_twobody_strict_bits_do_not_depend_on_start_epoch(oracle, name):
    """Two-body dynamics are autonomous, and the step bookkeeping is integer arithmetic on epochs: shifting every start and end
    epoch leaves every state bit, step and counter unchanged, around J2000, 20 years before it, 80 years after it and 1 ns on
    either side of the century boundaries, where dur_to_seconds changes branch.  (huge_saturating is left out: a step of INT64_MAX
    from a positive epoch overflows int64.)"""
    base = se.oracle_chain(name)
    case = se.CASE[name]
    for shift in se.EPOCH_SHIFTS:
        shift -= case.t0
        got = se.oracle_chain(name, shift)
        for k, (g, b) in enumerate(zip(got, base)):
            assert np.array_equal(g[0], b[0]), (name, shift, k)
            assert np.array_equal(g[1] - shift, b[1]) and np.array_equal(g[4], b[4]) and np.array_equal(g[3], b[3])
            for f in ("n_steps", "n_rejected", "attempts", "step_ns"):
                assert np.array_equal(g[2][f], b[2][f]), (name, shift, k, f)


@pytest.mark.parametrize("pname", [p[0] for p in se.PREDICT_CASES])
def test_predict_oracle_matches_integer_model(oracle, pname):
    """Chunk ends of `predict_until` at spans that are not multiples of the chunk, the integration step carried between chunks."""
    from tests import predict_oracle

    name, case, chunk, spans = next(p for p in se.PREDICT_CASES if p[0] == pname)
    for i, (sc, est, cs, end) in enumerate(se.predict_inputs(pname)):
        ref = predict_oracle.predict_until(*se.predict_oracle_args(pname), sc.to_vector(), cs, sc.epoch(), est.covar, end)
        rec, run = se.model_predict(case, chunk, sc.epoch(), end)
        assert ref["status"] == 0 and ref["rec_epoch"].tolist() == rec and ref["count"] == len(rec), (pname, i)
        assert ref["epoch"] == run.epoch and ref["n_steps"] == run.n_steps, (pname, i)
