"""Event-terminated propagation (SURVEY.md §8 (f)-3): `until_nth_event` (propagators/event.rs:88-211) and
`MonteCarlo::run_until_nth_event` (mc/montecarlo.rs:93-183)."""
import math

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.event import Event, brent, locate_event
from nyx_b200.trajectory import Traj
from tests.util import S, leo_ensemble, leo_state


def _dyn(degree=8):
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
    return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))


def _oracle_event(oracle, prop, frame, st, cs, ep, end, cap, ev: Event, trigger):
    packed = prop.dynamics.pack(frame, None)
    return oracle.propagate_batch(packed.c, prop.opts.to_c(prop.method), st, cs, ep, end, traj_capacity=cap,
                                  event=(ev.kind, ev.value, trigger))


def test_brent_finds_roots_to_tolerance():
    assert abs(brent(lambda x: math.cos(x) - x, 0.0, 1.0, 1e-12) - 0.7390851332151607) < 1e-11
    assert abs(brent(lambda x: (x - 0.3) ** 3, -1.0, 2.0, 1e-9) - 0.3) < 1e-3  # flat root: still inside the bracket
    assert brent(lambda x: x, 0.0, 1.0, 1e-9) == 0.0
    with pytest.raises(ValueError):
        brent(lambda x: x * x + 1.0, -1.0, 1.0, 1e-9)


def test_event_eval_closed_set():
    rv = np.array([3.0, 4.0, 12.0, 1.0, -2.0, 0.5])
    assert Event.radius(10.0).eval_rv(rv) == 3.0
    assert Event.apsis().eval_rv(rv) == (3.0 - 8.0) + 6.0
    assert Event.node().eval_rv(rv) == 12.0 and Event.component("x", 1.0).eval_rv(rv) == 2.0
    assert abs(Event.speed(0.0).eval_rv(rv) - math.sqrt(5.25)) < 1e-15


def test_oracle_stop_condition_semantics(oracle):
    """event.rs:120-150 + instance.rs:243-252: crossings are counted between accepted non-final steps, the run stops at
    the end of the step holding the `trigger`-th one, and the recorded stream ends with that state."""
    frame = nb.EARTH_J2000
    mc, (st, cs, ep) = leo_ensemble(6, seed=7)
    prop = nb.Propagator.default(_dyn())
    end = 6 * 3600 * S
    ev = Event.apsis()
    for trigger in (1, 3):
        out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = _oracle_event(oracle, prop, frame, st, cs, ep, end, 512, ev, trigger)
        assert (status == 0).all() and (crossings == trigger).all() and (out_ep < end).all()
        for i in range(6):
            k = int(t_cnt[i])
            assert k == det["n_steps"][i] + 1 and t_ep[k - 1, i] == out_ep[i] and np.array_equal(t_st[:, k - 1, i], out[:6, i])
            vals = np.array([ev.eval_rv(t_st[:, j, i]) for j in range(k)])
            signs = np.sign(vals)
            assert (signs[1:] * signs[:-1] < 0).sum() == trigger and vals[-1] * vals[-2] < 0  # bracket = last two records
    # not reached inside the window -> NthEventError status, full-span propagation, found count reported
    out, out_ep, det, status, _, crossings = _oracle_event(oracle, prop, frame, st, cs, ep, 1800 * S, 512, Event.radius(9000.0), 1)
    assert (status == abi.ERR_EVENT_NOT_FOUND).all() and (crossings == 0).all() and (out_ep == 1800 * S).all()
    # no event == plain propagation
    plain = oracle.propagate_batch(prop.dynamics.pack(frame, None).c, prop.opts.to_c(prop.method), st, cs, ep, 1800 * S)
    assert np.array_equal(plain[0], out)


def test_locate_event_on_oracle_trajectory(oracle):
    """event.rs:186-211: Brent on the interpolated trajectory puts the event inside the last step, at the requested
    epoch precision, and the returned state satisfies the event to interpolation accuracy."""
    frame = nb.EARTH_J2000
    sc = leo_state(frame)
    st, cs, ep = nb.pack_spacecraft([sc])
    prop = nb.Propagator.default(_dyn())
    for ev, tol in ((Event.node(), 1e-5), (Event.apsis(), 1e-4), (Event.radius(float(np.linalg.norm(st[:3, 0])) + 2.0), 1e-5)):
        out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = _oracle_event(oracle, prop, frame, st, cs, ep, 6 * 3600 * S, 512, ev, 2)
        assert status[0] == 0
        k = int(t_cnt[0])
        tr = Traj(sc, t_ep[:k, 0].copy(), np.ascontiguousarray(t_st[:, :k, 0].T)).finalize()
        found = locate_event(tr, ev)
        assert tr.epochs_ns[-2] <= found.epoch() <= tr.epochs_ns[-1]
        assert abs(ev.eval(found)) < tol


@pytest.mark.parametrize("which", ["apo", "peri"])
def test_reference_stop_cond_third_apsis(oracle, which):
    """The reference's own `stop_cond_3rd_apo` / `stop_cond_3rd_peri` (tests/propagation/stopcond.rs:35-153): two-body, default
    propagator, search over five periods; the third apoapsis (periapsis) lies between two and three periods after the start
    and at true anomaly 180 deg within 1e-6 (0 deg within 1e-1).  Their `Event::apoapsis()` / `periapsis()` look at one apsis;
    the closed scalar set here has r.v, which changes sign at both, so the third apoapsis is the 5th crossing (the start moves
    outward: apo, peri, apo, peri, apo) and the third periapsis the 6th.  Consecutive apsides of the same kind are one period
    apart within 0.5 s (0.3 s), as the reference asserts on its event report."""
    from nyx_b200.param import StateParameter as P, evaluate
    frame = nb.EARTH_J2000
    orbit = nb.Orbit.cartesian(-2436.45, -2436.45, 6891.037, 5.088611, -5.088611, 0.01, 0, frame)
    sc = nb.Spacecraft.from_orbit(orbit)
    mu = frame.mu_km3_s2()
    rv0 = orbit.to_cartesian_pos_vel().reshape(6, 1)
    period_s = float(evaluate(P.Period, rv0, mu)[0])
    period = int(period_s * 1e9)
    st, cs, ep = nb.pack_spacecraft([sc])
    prop = nb.Propagator.default(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body()))
    ev = Event.apsis(epoch_precision_ns=1000)
    found = {}
    for trigger in (1, 2, 3, 4, 5, 6):
        out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = _oracle_event(oracle, prop, frame, st, cs, ep, 5 * period, 2048, ev, trigger)
        assert status[0] == 0 and crossings[0] == trigger
        k = int(t_cnt[0])
        found[trigger] = locate_event(Traj(sc, t_ep[:k, 0].copy(), np.ascontiguousarray(t_st[:, :k, 0].T)).finalize(), ev)
    third = found[5] if which == "apo" else found[6]
    assert 2 * period + 1 <= third.epoch() <= 3 * period + 1
    ta = float(evaluate(P.TrueAnomaly, third.orbit.to_cartesian_pos_vel().reshape(6, 1), mu)[0])
    if which == "apo":
        assert abs(180.0 - ta) < 1e-6
        same_kind = [found[1], found[3], found[5]]
        tol = 0.5
    else:
        assert ta < 1e-1 or 360.0 - ta < 1e-1
        same_kind = [found[2], found[4], found[6]]
        tol = 0.3
    for a, b in zip(same_kind, same_kind[1:]):
        assert abs((b.epoch() - a.epoch()) * 1e-9 - period_s) < tol


def _host_locate(sc, t_ep, t_st, t_cnt, ev, run_status=None):
    """locate_event per run -> (epoch[n], state[6][n], status[n]) with the device entry point's status convention"""
    n = t_ep.shape[1]
    ev_ep, ev_st, status = np.zeros(n, dtype=np.int64), np.full((6, n), np.nan), np.ones(n, dtype=np.int32)
    for i in range(n):
        k = int(t_cnt[i])
        if k < 2 or (run_status is not None and run_status[i] & 0xFF):
            continue
        tr = Traj(sc, t_ep[:k, i].copy(), np.ascontiguousarray(t_st[:, :k, i].T)).finalize()
        try:
            found = locate_event(tr, ev)
        except ValueError:
            status[i] = 2
            continue
        ev_ep[i], ev_st[:, i], status[i] = found.epoch(), found.orbit.to_cartesian_pos_vel(), 0
    return ev_ep, ev_st, status


def test_event_locate_core_matches_host_brent(oracle, tmp_path):
    """The function the event-location kernel runs per trajectory (nyxb_hermite.h), compiled for the host: same Brent
    iterates, same interpolation, hence the same event epoch (integer ns) and bit-identical state as `locate_event`."""
    from tests.util import hermite_shim
    frame = nb.EARTH_J2000
    n = 12
    mc, (st, cs, ep) = leo_ensemble(n, seed=29)
    sc = mc.nominal_state
    prop = nb.Propagator.default(_dyn())
    locate = hermite_shim(tmp_path).locate
    for ev in (Event.node(), Event.apsis(), Event.radius(6679.5), Event.component("x", 100.0), Event.speed(7.75),
               Event.node(epoch_precision_ns=50)):
        out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = _oracle_event(oracle, prop, frame, st, cs, ep, 5 * 3600 * S, 256, ev, 2)
        status = status.copy()
        t_cnt = t_cnt.copy()
        status[3] = abi.ERR_PROP_MATH      # a failed run is skipped
        t_cnt[5] = 1                       # a run without a bracket
        t_cnt[7] -= 1                      # its last remaining step does not contain the crossing
        want = _host_locate(sc, t_ep, t_st, t_cnt, ev, status)
        got = locate(t_ep, t_st, t_cnt, ev.kind, ev.value, ev.epoch_precision_ns, status)
        assert np.array_equal(got[2], want[2]) and got[2][3] == 1 and got[2][5] == 1
        ok = want[2] == 0
        assert ok.sum() >= n - 4 and np.array_equal(got[0], want[0]) and np.array_equal(got[1][:, ok], want[1][:, ok])
        assert np.isnan(got[1][:, ~ok]).all()
        if (status & 0xFF == 0)[7]:
            assert got[2][7] == 2


@pytest.mark.gpu
def test_gpu_event_locate_matches_host_brent(oracle):
    """nyxb_event_locate through the C ABI: bit-identical to the host restatement on the engine's own recording (resident and
    re-uploaded), failed runs skipped, argument checks."""
    frame = nb.EARTH_J2000
    n = 40
    mc, (st, cs, ep) = leo_ensemble(n, seed=31)
    sc = mc.nominal_state
    eng = nb.Propagator.default(_dyn(21), mode=nb.MODE_FAST).engine(frame, None)
    for ev in (Event.node(), Event.apsis(), Event.radius(6679.5)):
        out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = eng.propagate_batch(
            st, cs, ep, 5 * 3600 * S, traj_capacity=256, event=(ev.kind, ev.value, 2))
        want = _host_locate(sc, t_ep, t_st, t_cnt, ev, status)
        got = eng.locate_events(ev.kind, ev.value, ev.epoch_precision_ns, n=n, run_status=status)
        assert (want[2] == 0).sum() >= n // 2
        for g, w in zip(got, want):
            assert np.array_equal(g, w, equal_nan=True)
        status2 = status.copy()
        status2[1] = abi.ERR_PROP_MATH
        t_cnt2 = t_cnt.copy()
        t_cnt2[2] -= 1
        got2 = eng.locate_events(ev.kind, ev.value, ev.epoch_precision_ns, (t_ep, t_st, t_cnt2), run_status=status2)
        want2 = _host_locate(sc, t_ep, t_st, t_cnt2, ev, status2)
        for g, w in zip(got2, want2):
            assert np.array_equal(g, w, equal_nan=True)
        assert got2[2][1] == 1
    with pytest.raises(nb.PropagationError):
        eng.locate_events(99, 0.0, 1000, n=n)
    with pytest.raises(nb.PropagationError):
        eng.locate_events(ev.kind, 0.0, 1000, n=n + 1)
    with pytest.raises(ValueError):
        eng.locate_events(ev.kind, 0.0, 1000)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,lanes", [(nb.MODE_STRICT, 1), (nb.MODE_STRICT, 8), (nb.MODE_FAST, 1), (nb.MODE_FAST, 8), (nb.MODE_FAST, 32),
                                        (nb.MODE_FAST, "tx")])
@pytest.mark.parametrize("kind", ["apsis", "node", "radius"])
def test_gpu_event_stop_matches_oracle(oracle, mode, lanes, kind):
    """lanes = "tx": the transposed kernel."""
    frame = nb.EARTH_J2000
    n = 48
    mc, (st, cs, ep) = leo_ensemble(n, seed=17)
    ev = {"apsis": Event.apsis(), "node": Event.node(), "radius": Event.radius(6679.5)}[kind]
    prop = nb.Propagator.default(_dyn(48 if lanes == 32 else 21), mode=mode)
    eng = prop.engine(frame, None)
    if lanes == "tx":
        eng.set_kernel(nb.KERNEL_TRANSPOSED)
    else:
        eng.set_lanes(lanes)
    end = 5 * 3600 * S
    out, out_ep, det, status, (g_ep, g_st, g_cnt), g_cross = eng.propagate_batch(st, cs, ep, end, traj_capacity=256, event=(ev.kind, ev.value, 2))
    assert eng.last_kernel() == (nb.KERNEL_TRANSPOSED if lanes == "tx" else nb.KERNEL_THREAD if lanes == 1 else nb.KERNEL_COOP)
    ref, ref_ep, ref_det, ref_status, (o_ep, o_st, o_cnt), o_cross = _oracle_event(oracle, prop, frame, st, cs, ep, end, 256, ev, 2)
    assert np.array_equal(g_cnt, det["n_steps"] + 1)
    if mode == nb.MODE_STRICT:
        assert np.array_equal(status, ref_status) and np.array_equal(g_cross, o_cross)
        assert np.array_equal(out, ref) and np.array_equal(out_ep, ref_ep) and np.array_equal(g_cnt, o_cnt)
        assert np.array_equal(g_ep, o_ep) and np.array_equal(g_st, o_st)
    else:
        # the step sequences differ by the controller's rounding noise, so a crossing may land in a neighbouring step:
        # compare what the caller uses, the located event itself
        assert np.array_equal(status & 0xFF, ref_status & 0xFF) and np.array_equal(g_cross, o_cross)
        sc0 = mc.nominal_state
        for i in range(0, n, 5):
            if status[i] & 0xFF:
                continue
            tg = Traj(sc0, g_ep[: g_cnt[i], i].copy(), np.ascontiguousarray(g_st[:, : g_cnt[i], i].T)).finalize()
            to = Traj(sc0, o_ep[: o_cnt[i], i].copy(), np.ascontiguousarray(o_st[:, : o_cnt[i], i].T)).finalize()
            fg, fo = locate_event(tg, ev), locate_event(to, ev)
            assert abs(fg.epoch() - fo.epoch()) <= 2 * ev.epoch_precision_ns
    # trigger never reached: NthEventError status for every run, final state == plain propagation
    far = Event.radius(20000.0)
    o2, e2, d2, s2, c2 = eng.propagate_batch(st, cs, ep, 1200 * S, event=(far.kind, far.value, 1))
    p2 = eng.propagate_batch(st, cs, ep, 1200 * S)
    assert ((s2 & 0xFF) == abi.ERR_EVENT_NOT_FOUND).all() and (c2 == 0).all() and np.array_equal(o2, p2[0])


@pytest.mark.gpu
def test_until_nth_event_and_monte_carlo_api(oracle):
    """Public surface: `PropInstance::until_nth_event` and `MonteCarlo::run_until_nth_event`."""
    frame = nb.EARTH_J2000
    sc = leo_state(frame)
    prop = nb.Propagator.default(_dyn(21), mode=nb.MODE_STRICT)
    ev = Event.node()
    found, tr = prop.with_(sc).until_nth_event(6 * 3600 * S, ev, trigger=3)
    assert abs(ev.eval(found)) < 1e-5 and tr.epochs_ns[-2] <= found.epoch() <= tr.epochs_ns[-1]
    # same bracket as the oracle (STRICT is bit-identical), hence the same located state
    st, cs, ep = nb.pack_spacecraft([sc])
    o = _oracle_event(oracle, prop, frame, st, cs, ep, 6 * 3600 * S, 1024, ev, 3)
    k = int(o[4][2][0])
    to = Traj(sc, o[4][0][:k, 0].copy(), np.ascontiguousarray(o[4][1][:, :k, 0].T)).finalize()
    assert np.array_equal(to.epochs_ns, tr.epochs_ns) and np.array_equal(to.states, tr.states)
    assert locate_event(to, ev).epoch() == found.epoch()
    with pytest.raises(nb.PropagationError, match="NthEventError"):
        prop.with_(sc).until_nth_event(600 * S, Event.radius(30000.0), trigger=1)

    mc, _ = leo_ensemble(32, seed=3)
    res = mc.run_until_nth_event(nb.Propagator.default(_dyn(21)), None, 4 * 3600 * S, Event.apsis(), 2, 32, traj_capacity=64)
    assert len(res.runs) == 32 and len(res.ok_runs()) == 32
    for run in res.runs:
        state, traj = run.result
        assert abs(Event.apsis().eval(state)) < 1e-3 and traj.first().epoch() == 0 and state.epoch() <= traj.last().epoch()
