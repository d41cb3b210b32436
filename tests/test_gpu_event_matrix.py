"""Event-terminated runs (`nyxb_propagate_batch_event`) and event location (`nyxb_event_locate`) of every kernel family against
the CPU oracle at a fixed step (inputs and edge catalogue: tests/event_matrix.py; CPU side: tests/test_event_matrix_inputs.py).

Families, each forced and checked with `last_kernel()`:
  K1-S / K1-F         per-thread kernel, STRICT / FAST (the only ones without a gravity field: the two-body cases)
  K2-G8 / G16 / G32   lane-cooperative FAST kernel, 8 / 16 / 32 lanes per trajectory
  K3-G8 / G16 / G32   lane-cooperative STRICT kernel
  K5-P8 / P10 / P16   transposed kernel, 8 / 10 / 16 walker positions per set
  K5-S5x1 / S1x1      transposed kernel time-sliced on one CTA (two set contexts for three sets of 32): 5 attempts or 1 attempt
                      per slice, so a set parks after every fifth step, or every step, with its crossing count and previous
                      scalar value (on three CTAs every set of these ensembles would have a context of its own and never park)

Runs, every family: status word, crossings, stop epochs, n_steps, n_rhs, details.step_ns, the step array handed back, the
recorded count and the recorded epochs equal to the oracle's; states and recorded states within fast_matrix.bounds (5e-9 km,
5e-12 km/s; RK4 at 10 s ten times that).  STRICT on "field" and two-body: every output bit-equal.  STRICT on "srp" and "all"
goes through CUDA's acos / asin / exp / pow, so it is held to the FAST assertions.  K5 time-sliced: bit-equal to K5-P8.

Location, on every family's own recording, resident and re-uploaded:
  (a) bit-equal to nyx_b200.event.locate_event on the same recording (the bracket: the last step taken), every scalar, forward
      and backward, at 1 ns, 1 us, 1 ms and 90 s (longer than the step) precision; values that put an end of the last step
      exactly on zero (Brent's fa == 0 / fb == 0 returns); skipped runs and single-record recordings give NYXB_TRAJ_NO_DATA;
  (b) against the oracle's recording located on the host: |dt| <= precision + 1 ns + 2 dy / |dy/dt|, with dy the scalar's
      sensitivity to (dr, dv), the difference of the two recordings interpolated at the event epoch (the records themselves are
      held to the fixed-step bounds above; the event lies in the end step of its interpolation window, where a worst-case
      difference could be amplified a thousandfold, so the actual one is carried), and the located state within (dr, dv) plus
      |v| |dt| (|a| |dt| for velocity);
  (c) two-body: against the root of the scalar on the 40-digit Kepler flow (mpmath.findroot), within precision + 1 ns plus
      twice the oracle's own distance from it, plus for FAST the root shift dy / |dy/dt| of (b) (r crosses 6 700 km at
      |dr/dt| ~ 0.1 km/s: 5e-9 km there is 50 ns).

Measured maxima on an H100 80GB HBM3 (SXM, 700 W power limit), |dr| km and |dv| km/s over final and recorded states:

  family      field          srp            all            backward       two-body       RK4 10 s       ragged         edges
  K1-S, K3-*  0 (bit-equal on every configuration, "srp" and "all" included)
  K1-F        2.0e-09 2e-12  2.6e-09 3e-12  3.1e-09 4e-12  2.9e-09 3e-12  1.7e-10 2e-13  2.8e-09 3e-12  1.9e-09 2e-12  1.7e-09 2e-12
  K2-G8/16/32 2.2e-09 3e-12  1.8e-09 2e-12  1.8e-09 2e-12  2.0e-09 2e-12  -              2.7e-09 3e-12  2.1e-09 2e-12  1.9e-09 2e-12
  K5-*        1.9e-09 2e-12  1.6e-09 2e-12  1.9e-09 2e-12  2.0e-09 2e-12  -              2.7e-09 3e-12  2.1e-09 2e-12  1.7e-09 2e-12
Location (b): the largest |dt| / bound is 0.53 (K2), with interpolated recording differences up to 7.2e-9 km and 7.9e-10 km/s;
(c): the largest distance from the Kepler root over its bound is 0.50 (K1-S) and 0.48 (K1-F).  The file takes about two minutes
on that card, most of it in the oracle's runs and the host searches.

Each of these one-line kernel mutations, applied alone, fails this file (found with the library built from the mutated source):
  K1 evaluating the stop condition on the final cut step too     test_event_runs[K1-S/K1-F-all, -back], test_event_edges[K1-*]
  K2 counting a crossing on a zero product (<= 0.0)              test_event_edges[K2-G8/G16/G32] (start_on_value)
  K3 not updating its previous scalar value after a step         test_event_runs[K3-*-*], test_event_edges[K3-*]
  K5 resuming a parked set with the previous value 0.0           test_event_runs[K5-S5x1/S1x1-*], test_event_edges[K5-S*]
  K5 resuming a parked set with the crossing count 0             test_event_runs[K5-S5x1/S1x1-*], test_event_edges[K5-S*]
  event_eval's VMAG reading the position (K1 built with it)      test_event_runs[K1-S-field, -srp, -all, -back, -twobody, -ragged]
One more candidate is not a fault this file can see: nyxb_event_locate_one taking t0 / t1 in recording order for descending
recordings (a bracket reversed in time) gives the same located events, bit for bit, on every case here (on the device at 1 ns
and 1 ms, on the host build of the same header at all four precisions): Brent's method does not depend on the orientation of
its bracket."""
import functools

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.event import Event
from tests import event_matrix as em
from tests.test_gpu_fast_matrix import force_family
from tests.util import S, leo_ensemble, max_dr_dv

pytestmark = pytest.mark.gpu

FAMILIES = ("K1-S", "K1-F", "K2-G8", "K2-G16", "K2-G32", "K3-G8", "K3-G16", "K3-G32", "K5-P8", "K5-P10", "K5-P16", "K5-S5x1",
            "K5-S1x1")
KERNEL = {"K1": nb.KERNEL_THREAD, "K2": nb.KERNEL_COOP, "K3": nb.KERNEL_COOP, "K5": nb.KERNEL_TRANSPOSED}
GROUPS = ("field", "srp", "all", "back", "twobody", "rk4", "ragged")
SUBSET = slice(0, None, 8)    # runs located on the host in (a) - (c): 12 of 96, LEO and eccentric


def strict(family):
    return family in ("K1-S",) or family.startswith("K3")


def engine(case, family):
    eng = em.propagator(case, nb.MODE_STRICT if strict(family) else nb.MODE_FAST).engine(nb.EARTH_J2000, em.almanac(case.config))
    kind, _, arg = family.partition("-")
    if kind == "K3":
        eng.set_kernel(nb.KERNEL_COOP)
        eng.set_lanes(int(arg[1:]))
    elif kind == "K1":
        eng.set_kernel(nb.KERNEL_THREAD)
    elif arg.startswith("S"):
        eng.set_kernel(nb.KERNEL_TRANSPOSED)
        eng.set_tx_tuning(*(int(x) for x in arg[1:].split("x")))
    else:
        force_family(eng, family)
    return eng


def run(case, family, eng=None):
    eng = eng or engine(case, family)
    st, cs, ep, end = em.inputs(case)
    step = np.full(st.shape[1], int(case.step_s * S), dtype=np.int64)
    got = eng.propagate_batch(st, cs, ep, end, step, traj_capacity=case.cap, event=case.event)
    assert eng.last_kernel() == KERNEL[family[:2]], (family, eng.last_kernel())
    return eng, got + (step,)


def check(tag, family, case, got, ref):
    """got, ref = (state, epoch, details, status, (epochs, states, count), crossings, step array)"""
    out, out_ep, det, status, (g_ep, g_st, g_cnt), cross, step = got
    r, r_ep, r_det, r_status, (o_ep, o_st, o_cnt), o_cross, o_step = ref
    assert np.array_equal(status, r_status), (tag, "status", np.flatnonzero(status != r_status)[:8])
    assert np.array_equal(cross, o_cross), (tag, "crossings", np.flatnonzero(cross != o_cross)[:8])
    assert np.array_equal(out_ep, r_ep), (tag, "epoch", np.flatnonzero(out_ep != r_ep)[:8])
    assert np.array_equal(step, o_step), (tag, "step array")
    for f in ("n_steps", "n_rhs", "step_ns"):
        assert np.array_equal(det[f], r_det[f]), (tag, f, np.flatnonzero(det[f] != r_det[f])[:8])
    assert np.array_equal(g_cnt, o_cnt) and np.array_equal(g_ep, o_ep), (tag, "recorded count / epochs")
    if strict(family) and case.config in ("field", "twobody"):
        assert np.array_equal(out, r) and np.array_equal(g_st, o_st) and np.array_equal(det, r_det), (tag, max_dr_dv(out, r))
        dr = dv = 0.0
    else:
        bdr, bdv = case.bounds()
        d = g_st - o_st
        dr = max(max_dr_dv(out, r)[0], float(np.sqrt((d[:3] ** 2).sum(0)).max()))
        dv = max(max_dr_dv(out, r)[1], float(np.sqrt((d[3:6] ** 2).sum(0)).max()))
        assert dr < bdr and dv < bdv, (tag, dr, dv)
        assert np.array_equal(out[6:], r[6:]), tag
    print(f"EVENTMATRIX {tag} dr={dr:.2e} dv={dv:.2e} stops={int((status == 0).sum())}/{len(status)}")


def _group(case):
    if case.edge == "ragged":
        return "ragged"
    if case.method == em.RK4:
        return "rk4"
    if case.config == "twobody":
        return "twobody"
    return "back" if case.backward else case.config


@functools.lru_cache(maxsize=None)
def _k5_reference(name):
    return run(em.CASES[name], "K5-P8")[1]


@pytest.mark.parametrize("group", GROUPS)
@pytest.mark.parametrize("family", FAMILIES)
def test_event_runs(oracle, family, group):
    if group == "twobody" and not family.startswith("K1"):
        pytest.skip("the cooperative and transposed kernels need a gravity field")
    engines = {}
    for case in (c for c in em.ORDINARY if _group(c) == group):
        key = (case.config, case.method)
        if key not in engines:
            engines[key] = engine(case, family)
        _, got = run(case, family, engines[key])
        check(f"{family} {case.name}", family, case, got, em.oracle(case))
        if family.startswith("K5-S"):
            ref = _k5_reference(case.name)
            for g, r in zip(got[:4] + got[5:], ref[:4] + ref[5:]):
                assert np.array_equal(g, r), (family, case.name)
            for g, r in zip(got[4], ref[4]):
                assert np.array_equal(g, r), (family, case.name)


@pytest.mark.parametrize("family", FAMILIES)
def test_event_edges(oracle, family):
    for case in em.edges() + em.cut_step_cases():
        if case.strict_only and not strict(family):
            continue
        if case.config == "twobody" and not family.startswith("K1"):
            continue
        _, got = run(case, family)
        check(f"{family} {case.name}", family, case, got, em.oracle(case))
        if case.edge == "cut_step":
            plain = em._run(case, *em.inputs(case)[:3], case.end, cap=0)
            assert got[3][0] == abi.ERR_EVENT_NOT_FOUND and got[5][0] == case.trigger - 1
            if strict(family):
                assert np.array_equal(got[0], plain[0])
        elif case.edge == "short_sink":
            ok = got[3] == 0
            assert (got[4][2][ok] == case.cap).all() and (got[2]["n_steps"][ok] + 1 > case.cap).all()
        elif case.edge == "two_in_one_step":
            assert got[5][case.cols.index(em.ECC_RUN)] == 0
        elif case.edge == "statuses":
            eng = engine(case, family)
            _, got = run(case, family, eng)
            ev = Event(*case.event[:2])
            codes = got[3] & 0xFF
            assert (codes[[5, 66]] == abi.ERR_FUEL_EXHAUSTED).all() and (codes[[3, 40, 70, 95]] == abi.ERR_EVENT_NOT_FOUND).all()
            # skipped runs and single-record recordings: NYXB_TRAJ_NO_DATA
            loc = eng.locate_events(ev.kind, ev.value, 1000, n=len(codes), run_status=got[3])
            assert (loc[2][codes != 0] == 1).all() and np.isnan(loc[1][:, codes != 0]).all()
            loc = eng.locate_events(ev.kind, ev.value, 1000, got[4])
            assert (loc[2][got[4][2] < 2] == 1).all() and (got[4][2][[3, 40, 70, 95]] == 1).all()


# ---- location
def _located_cases():
    out = []
    for kind in em.KINDS:
        out.append(em.CASES[f"field-{kind}={em.VALUES[kind][0]:g}-t7"])
        out.append(em.CASES[f"field-{kind}={em.VALUES[kind][0]:g}-t7-back"])
    return out


def interpolated_difference(rec_g, rec_o, i, t_ns):
    """(|dr|, |dv|) between the two recordings of run i interpolated at t_ns: what their difference becomes at the event (the
    Hermite interpolant is linear in the records; near the edge of its window it can amplify a difference, smooth ones little)"""
    def at(rec):
        k = int(rec[2][i])
        return em.traj(rec[0][:k, i], rec[1][:, :k, i]).at(int(t_ns)).orbit.to_cartesian_pos_vel()

    d = at(rec_g) - at(rec_o)
    return float(np.linalg.norm(d[:3])), float(np.linalg.norm(d[3:]))


def root_shift_ns(case, rv, dr, dv):
    """how far the event epoch moves (ns) when the interpolated state moves by (dr, dv): twice the first-order shift"""
    return 2e9 * em.perturbation(case.kind, rv, dr, dv) / np.abs(em.rate(case.kind, rv))


def _precision(k):
    """the k-th located case's precision: forward (even k) and backward (odd k) cases each go through all four"""
    return em.PRECISIONS[(k // 2 + k) % len(em.PRECISIONS)]


@functools.lru_cache(maxsize=None)
def _oracle_located(name, precision):
    case = next(c for c in em.ORDINARY if c.name == name)
    ref = em.oracle(case)
    return em.locate_all(ref[4], Event(*case.event[:2], epoch_precision_ns=precision), ref[3], range(ref[3].shape[0])[SUBSET])


def _assert_located_equal(tag, got, want, runs):
    for g, w in zip(got, want):
        assert np.array_equal(g[..., runs], w[..., runs], equal_nan=True), tag


@pytest.mark.parametrize("family", FAMILIES)
def test_event_location(oracle, family):
    runs = list(range(96))[SUBSET]
    worst = worst_dr = worst_dv = 0.0
    for k, case in enumerate(_located_cases()):
        prec = _precision(k)
        ev = Event(*case.event[:2], epoch_precision_ns=prec)
        eng, got = run(case, family)
        tag = f"{family} {case.name} precision {prec} ns"
        # (a) bit-equal to the host restatement on this family's recording, resident and re-uploaded
        want = em.locate_all(got[4], ev, got[3], runs)
        resident = eng.locate_events(ev.kind, ev.value, prec, n=96, run_status=got[3])
        uploaded = eng.locate_events(ev.kind, ev.value, prec, got[4], run_status=got[3])
        _assert_located_equal(tag, resident, want, runs)
        _assert_located_equal(tag, uploaded, want, runs)
        assert np.array_equal(resident[0], uploaded[0]) and np.array_equal(resident[1], uploaded[1], equal_nan=True)
        assert (want[2][runs][got[3][runs] == 0] == 0).all()
        # (b) against the oracle's recording
        ref_loc = _oracle_located(case.name, prec)
        assert np.array_equal(resident[2][runs], ref_loc[2][runs]), tag
        ok = np.array(runs)[ref_loc[2][runs] == 0]
        for i in ok:
            dr, dv = interpolated_difference(got[4], em.oracle(case)[4], i, resident[0][i])
            rv = ref_loc[1][:, i]
            dt = abs(int(resident[0][i]) - int(ref_loc[0][i]))
            bound = prec + 1.0 + float(root_shift_ns(case, rv[:, None], dr, dv)[0])
            assert dt <= bound, (tag, i, dt, bound)
            d = resident[1][:, i] - rv
            v_dt = 1.01 * np.linalg.norm(rv[3:]) * dt * 1e-9                # |v| and |a| along the step, with room for J2
            a_dt = 1.01 * nb.EARTH_J2000.mu / (rv[:3] ** 2).sum() * dt * 1e-9
            assert np.linalg.norm(d[:3]) <= dr * (1 + 1e-6) + v_dt + 1e-12, (tag, i)
            assert np.linalg.norm(d[3:]) <= dv * (1 + 1e-6) + a_dt + 1e-15, (tag, i)
            worst = max(worst, dt / bound)
            worst_dr, worst_dv = max(worst_dr, dr), max(worst_dv, dv)
        # Brent's early returns: a value on which an end of the last step sits exactly (component X, run 0)
        if case.kind == "X":
            cnt = int(got[4][2][0])
            for rec, end in ((cnt - 1, "last"), (cnt - 2, "previous")):
                value = float(got[4][1][0, rec, 0])
                ev2 = Event(abi.EVENT_X, value, epoch_precision_ns=prec)
                g2 = eng.locate_events(ev2.kind, ev2.value, prec, got[4], run_status=got[3])
                w2 = em.locate_all(got[4], ev2, got[3], [0])
                _assert_located_equal(f"{tag} X on the {end} record", g2, w2, [0])
                assert g2[2][0] == 0 and g2[0][0] == got[4][0][rec, 0], (tag, end)
    print(f"EVENTMATRIX {family} location max dt/bound={worst:.3f} interpolated record difference {worst_dr:.2e} km {worst_dv:.2e} km/s")


@functools.lru_cache(maxsize=None)
def _kepler_roots(name):
    """per located run of the oracle (1 ns precision): the Kepler root and the oracle's located epoch"""
    case = em.CASES[name]
    st, cs, ep, end = em.inputs(case)
    ref = em.oracle(case)
    loc = em.locate_all(ref[4], Event(*case.event[:2], epoch_precision_ns=1), ref[3], range(96)[SUBSET])
    out = {}
    for i in range(96)[SUBSET]:
        if loc[2][i] == 0:
            out[i] = (em.kepler_root(st[:3, i], st[3:6, i], int(ep[i]), case.kind, case.value, int(loc[0][i])), int(loc[0][i]))
    return out


@pytest.mark.parametrize("family", ("K1-S", "K1-F"))
def test_event_location_two_body_against_kepler(oracle, family):
    """(c): every scalar, both directions; STRICT within precision + 1 ns + twice the oracle's distance from the Kepler root,
    FAST that plus the root shift of (b)"""
    worst = 0.0
    for k, case in enumerate(c for c in em.ORDINARY if c.config == "twobody"):
        prec = _precision(k)
        eng, got = run(case, family)
        loc = eng.locate_events(case.event[0], case.value, prec, n=96, run_status=got[3])
        roots = _kepler_roots(case.name)
        assert len(roots) >= 6, case.name
        for i, (root, t_oracle) in roots.items():
            assert loc[2][i] == 0, (family, case.name, i)
            d_oracle = abs(t_oracle - root)
            d = abs(loc[0][i] - root)
            # FAST: its recording differs from the oracle's, which moves the root by root_shift_ns (0 for STRICT)
            dr, dv = interpolated_difference(got[4], em.oracle(case)[4], i, loc[0][i])
            bound = prec + 1.0 + 2.0 * d_oracle + float(root_shift_ns(case, loc[1][:, i:i + 1], dr, dv)[0])
            assert d <= bound, (family, case.name, i, prec, d, d_oracle)
            worst = max(worst, d / bound)
    print(f"EVENTMATRIX {family} two-body location max distance/bound={worst:.3f}")


def test_sink_too_small_is_never_searched(oracle):
    """nyxb_event_locate searches the last two records it is given, so a truncated recording would give a wrong event: the host
    API never searches one.  until_nth_event(capacity=too_small) raises; run_until_nth_event grows its sink and finds the same
    event as with room to spare."""
    mc, (st, cs, ep) = leo_ensemble(16, seed=3)
    dyn = em.dynamics("field")
    prop = nb.Propagator.new(dyn, em.RK89, nb.IntegratorOptions.with_fixed_step_s(60.0), mode=nb.MODE_FAST)
    ev = Event.node(epoch_precision_ns=1000)
    with pytest.raises(nb.PropagationError, match="too small"):
        prop.with_(mc.nominal_state, em.almanac("field")).until_nth_event(6 * 3600 * S, ev, trigger=3, capacity=20)
    small = mc.run_until_nth_event(prop, em.almanac("field"), 6 * 3600 * S, ev, 3, 16, traj_capacity=8)
    big = mc.run_until_nth_event(prop, em.almanac("field"), 6 * 3600 * S, ev, 3, 16, traj_capacity=1024)
    assert len(small.ok_runs()) == 16
    for a, b in zip(small.runs, big.runs):
        assert a.result[0].epoch() == b.result[0].epoch() and np.array_equal(a.result[0].to_vector(), b.result[0].to_vector())
        assert abs(ev.eval(a.result[0])) < 1e-4

