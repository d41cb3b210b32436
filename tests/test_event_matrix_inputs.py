"""CPU side of the event-run matrix (tests/event_matrix.py): the ordinary cases leave FAST round-off no room to change a
crossing, every edge of the catalogue happens on the oracle, every status occurs, the time-sliced transposed kernel parks in the
middle of a count, and a one-step error in the counter changes a result the GPU test compares."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import event_matrix as em
from tests.span_edges import kepler
from tests.util import S


def _margin(case, i, exempt_start=False):
    y, rv = em.evaluated(case, i)
    dr, dv = case.bounds()
    ratio = np.abs(y) / em.perturbation(case.kind, rv, dr, dv)
    return ratio[1:].min() if exempt_start and len(ratio) > 1 else ratio.min() if len(ratio) else np.inf


@pytest.mark.parametrize("name", [c.name for c in em.ORDINARY] + ["start_on_value", "two_in_one_step", "statuses", "short_sink"])
def test_margins(oracle, name):
    """|scalar - value| >= 1e3 x (|dy/dr| FIXED_DR + |dy/dv| FIXED_DV) at the start and at every evaluated step end of every run
    (start_on_value: its run 0 starts on the value, exactly, in every build)"""
    case = em.CASES.get(name) or next(c for c in em.edges() if c.name == name)
    n = em.inputs(case)[0].shape[1]
    worst = min(_margin(case, i, exempt_start=(case.edge == "start_on_value" and i == 0)) for i in range(n))
    assert worst >= em.MARGIN, (name, worst)


@pytest.mark.parametrize("name", [c.name for c in em.ORDINARY])
def test_counter_model_reproduces_the_oracle(oracle, name):
    """The Python counter on the oracle's own step ends gives its stop step, crossings and status, run by run"""
    case = em.CASES[name]
    out, out_ep, det, status, rec, crossings = em.oracle(case)[:6]
    for i in range(len(status)):
        y, _ = em.evaluated(case, i)
        stop, count = em.count_model(y, case.trigger)
        if stop is None:
            assert status[i] & 0xFF == abi.ERR_EVENT_NOT_FOUND and crossings[i] == count, (name, i)
        else:
            assert status[i] == 0 and crossings[i] == case.trigger and det["n_steps"][i] == stop, (name, i)
            assert rec[2][i] == stop + 1 and out_ep[i] == rec[0][stop, i]


def test_every_status_and_scalar_stops_and_misses(oracle):
    codes = {abi.ERR_EVENT_NOT_FOUND: 0, 0: 0, abi.ERR_FUEL_EXHAUSTED: 0}
    by_kind = {k: [0, 0] for k in em.KINDS}
    for case in em.ORDINARY + em.edges():
        st = em.oracle(case)[3] & 0xFF
        for c in codes:
            codes[c] += int((st == c).sum())
        by_kind[case.kind][0] += int((st == 0).sum())
        by_kind[case.kind][1] += int((st == abi.ERR_EVENT_NOT_FOUND).sum())
    assert all(v > 0 for v in codes.values()), codes
    assert all(s > 0 and m > 0 for s, m in by_kind.values()), by_kind
    for case in em.ORDINARY:   # the last trigger is reached by most runs that cross at all
        if case.trigger >= 6:
            st, crossings = em.oracle(case)[3], em.oracle(case)[5]
            assert (st == 0).sum() >= 0.5 * (crossings > 0).sum(), case.name


def test_exact_step_end(oracle):
    """y at record k of run 0 is exactly 0.0 in the oracle's recording: the sign change at k is missed, the run goes on to the
    next one; counting zero products would have stopped it at k"""
    case = next(c for c in em.edges() if c.name == "exact_step_end")
    y, _ = em.evaluated(case, em.EXACT_RUN)
    k = em.EXACT_RECORD
    assert y[k] == 0.0 and y[k - 1] * y[k + 1] < 0.0
    ref = em.oracle(case)
    assert ref[3][em.EXACT_RUN] == 0 and ref[2]["n_steps"][em.EXACT_RUN] > k + 1
    assert em.count_model(y, 1, strict=False)[0] == k
    assert em.count_model(y, 1)[0] == ref[2]["n_steps"][em.EXACT_RUN]


def test_start_on_value(oracle):
    case = next(c for c in em.edges() if c.name == "start_on_value")
    y, _ = em.evaluated(case, 0)
    assert y[0] == 0.0 and y[1] != 0.0
    assert em.count_model(y, 1, strict=False)[0] == 1 and em.count_model(y, 1)[0] == em.oracle(case)[2]["n_steps"][0] > 1


def test_two_crossings_inside_one_step(oracle):
    """On the two-body copy of run 94, r passes under the value and back inside one step at every periapsis (the 40-digit Kepler
    flow at the periapsis epoch between two step ends), and the oracle counts nothing"""
    case = next(c for c in em.edges() if c.name == "two_in_one_step")
    j = case.cols.index(em.ECC_RUN)
    ref = em.oracle(case)
    assert ref[5][j] == 0 and ref[3][j] & 0xFF == abi.ERR_EVENT_NOT_FOUND
    st, cs, ep, end = em.inputs(case)
    t_ep, t_st, t_cnt = ref[4]
    y, _ = em.evaluated(case, j)
    assert (y > 0).all()
    dips = 0
    for s in np.flatnonzero((y[1:-1] < y[:-2]) & (y[1:-1] <= y[2:])) + 1:   # step ends next to a periapsis
        for a in (s - 1, s):
            lo, hi = int(t_ep[a, j]) - int(ep[j]), int(t_ep[a + 1, j]) - int(ep[j])
            mid = lo + (hi - lo) // 2
            # r at the end points of the step from the Kepler flow as well (the recording is the integrator's)
            rs = [em.scalar("RMAG", case.value, np.concatenate(kepler(st[:3, j], st[3:6, j], t)))
                  for t in np.linspace(lo, hi, 121).astype(np.int64)]
            if rs[0] > 0 and rs[-1] > 0 and min(rs) < 0:
                dips += 1
        assert mid > 0
    assert dips >= 3, dips


def test_cut_step(oracle):
    """The trigger-th crossing lies inside the final cut step: EVENT_NOT_FOUND, trigger - 1 crossings, the plain final state"""
    for case in em.cut_step_cases():
        ref = em.oracle(case)
        assert ref[3][0] == abi.ERR_EVENT_NOT_FOUND and ref[5][0] == case.trigger - 1, case.name
        t_ep, t_st, t_cnt = ref[4]
        k = int(t_cnt[0])
        z_before, z_end = t_st[2, k - 2, 0], ref[0][2, 0]
        assert z_before * z_end < 0 and (case.end - int(t_ep[k - 2, 0])) < 60 * S
        plain = em._run(case, *em.inputs(case)[:3], case.end, cap=0)
        assert np.array_equal(plain[0], ref[0]) and np.array_equal(plain[1], ref[1])


def test_short_sink_and_statuses(oracle):
    case = next(c for c in em.edges() if c.name == "short_sink")
    ref, full = em.oracle(case), em.oracle(em.CASES["field-RDOTV=0-t7"])
    ok = ref[3] == 0
    assert (ref[2]["n_steps"][ok] + 1 > case.cap).all() and (ref[2]["n_steps"][ok] + 1 == case.cap + 1).any()
    assert (ref[4][2][ok] == case.cap).all() and np.array_equal(ref[0], full[0]) and np.array_equal(ref[3], full[3])
    case = next(c for c in em.edges() if c.name == "statuses")
    st = em.oracle(case)[3] & 0xFF
    assert (st[[3, 40, 70, 95]] == abi.ERR_EVENT_NOT_FOUND).all() and (em.oracle(case)[5][[3, 40, 70, 95]] == 0).all()
    assert (st[[5, 66]] == abi.ERR_FUEL_EXHAUSTED).all()


def test_ragged_neighbours_stop_at_different_steps(oracle):
    for case in em.ORDINARY:
        if case.edge != "ragged":
            continue
        steps = em.oracle(case)[2]["n_steps"]
        for g in (4, 32):   # K2 at 8 lanes packs four runs per warp; K5 sets of 32
            groups = [steps[a:a + g] for a in range(0, len(steps), g)]
            assert sum(len(np.unique(x)) > 1 for x in groups) >= len(groups) // 2, (case.name, g)


def test_transposed_kernel_parks_mid_count(oracle):
    """set_tx_tuning(5, 1): every fixed-step attempt is accepted, so a set parks after every fifth step (with (1, 1) after every
    step); at least ten runs of each case at the last trigger hold 0 < crossings < trigger at a park"""
    for case in em.ORDINARY:
        if case.trigger < 6 or case.config == "twobody":
            continue
        rec = em.oracle(case)[4]
        mid = 0
        for i in range(rec[2].shape[0]):
            y, _ = em.evaluated(case, i, rec)
            counts = np.concatenate([[0], np.cumsum(y[1:] * y[:-1] < 0.0)])
            parks = counts[5::5]
            mid += bool(((parks > 0) & (parks < case.trigger)).any())
        assert mid >= 10, (case.name, mid)


def test_one_step_errors_change_a_result(oracle):
    """Shifting the value by a case's own margin (the closest approach of the scalar at a step end), or counting zero products,
    changes the stop step or the crossings of some run: the GPU comparison can see a one-step error"""
    moved = {k: False for k in em.KINDS}
    for case in em.ORDINARY:
        if moved[case.kind] or case.edge:
            continue
        for i in range(em.inputs(case)[0].shape[1]):
            y, _ = em.evaluated(case, i)
            j = int(np.argmin(np.abs(y[1:]))) + 1
            shifted = y - y[j] * (1 + 1e-9)
            if em.count_model(shifted, case.trigger) != em.count_model(y, case.trigger):
                moved[case.kind] = True
                break
    assert all(moved.values()), moved
    case = next(c for c in em.edges() if c.name == "exact_step_end")
    y, _ = em.evaluated(case, em.EXACT_RUN)
    assert em.count_model(y, 1, strict=False) != em.count_model(y, 1)
