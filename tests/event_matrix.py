"""Inputs of the event-run matrix (tests/test_gpu_event_matrix.py) and of its CPU companion (tests/test_event_matrix_inputs.py):
event-terminated runs (`nyxb_propagate_batch_event`) at a fixed step, and the oracle results every kernel family is compared with.

At a fixed step the step sequence cannot diverge, so every discrete output of an event run (stop epoch, step count, crossings,
status, recorded count) is the same in STRICT and FAST as long as the event scalar is, at every step end, farther from the
desired value than FAST round-off can move it.  The ordinary cases are chosen so (tests/test_event_matrix_inputs.py checks the
margin), on the 96-trajectory ensemble of tests/fast_matrix.py: every scalar of the closed set, at zero where that makes sense and
at a value one of the two orbit families never reaches, with triggers 1, 2 and 7 (the 7th crossing, the 6th for x = 4 500 km:
reached by most runs, missed by the runs that start late or cross fewer times).

The edge catalogue states the outcome each entry claims, as the stop condition is coded in the reference (event.rs:115-145: a
crossing is a strict sign change of `scalar - value` between two accepted steps; instance.rs:243-259: it is evaluated after every
accepted step except the final cut one, and the run stops at the end of the step holding the `trigger`-th crossing):
  exact_step_end   X equal, bit for bit, to record k of run 0 of the oracle's STRICT recording: y_k = 0.0, so the crossing is
                   counted neither at step k nor at k + 1 and the run stops at a later one (STRICT only: FAST moves x_k)
  start_on_value   X equal to run 0's start x: y_0 = 0.0, the first step cannot count
  two_in_one_step  two-body, r = 10 m above run 94's periapsis: r dips under it for ~10 s between two step ends, every passage
                   (two crossings inside one step, none counted)
  cut_step         runs of one whose end epoch falls inside the step that holds the trigger-th crossing: the final cut step is
                   not evaluated, so EVENT_NOT_FOUND with trigger - 1 crossings and the state of the plain propagation
  short_sink       a sink one record shorter than the earliest stop: OK, count == capacity, the stop state returned
  statuses         runs already at the end epoch (0 crossings, EVENT_NOT_FOUND), runs with negative propellant mass
                   (FUEL_EXHAUSTED), and one run that is both (EVENT_NOT_FOUND: a zero span returns before the mass check)
  backward         every scalar from the 6 h states back to epoch 0: negative steps, descending recordings
  ragged           33, 70 and 160 runs: partial K2 lane groups and K5 sets whose members stop at different steps"""
import functools
from dataclasses import dataclass

import numpy as np

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.event import Event
from nyx_b200.trajectory import Traj
from tests import fast_matrix as fm
from tests.util import S

RK89, RK4 = nb.IntegratorMethod.RungeKutta89, nb.IntegratorMethod.RungeKutta4
END = fm.END
CAP = 400                       # records: 6 h at 60 s is at most 361
NO_STOP = 1 << 30               # a trigger no run reaches: the run records every step end
MARGIN = 1e3                    # ordinary cases: |scalar - value| >= MARGIN x the FAST perturbation at every evaluated step end
KINDS = ("RMAG", "RDOTV", "X", "Y", "Z", "VMAG")
KIND = {"RMAG": abi.EVENT_RMAG, "RDOTV": abi.EVENT_RDOTV, "X": abi.EVENT_X, "Y": abi.EVENT_Y, "Z": abi.EVENT_Z,
        "VMAG": abi.EVENT_VMAG}
# per scalar: a value every run crosses, and one that only the LEO (columns 0..63) or only the eccentric runs reach
VALUES = {"RMAG": (6700.0, 7000.0), "RDOTV": (0.0, 2000.0), "X": (0.0, 4500.0), "Y": (0.0, -6000.0), "Z": (0.0, 6000.0),
          "VMAG": (7.7, 7.9)}
TRIGGERS = (1, 2, 7)
LAST_TRIGGER = {("X", 4500.0): 6}           # the eccentric runs cross x = 4 500 km six times: 6 takes the place of 7
PRECISIONS = (1, 1000, 1_000_000, 90 * S)   # epoch precisions of the search: 1 ns, 1 us, 1 ms, longer than the step
ECC_RUN, PERIAPSIS_OFFSET = 94, 0.010      # two_in_one_step
EXACT_RUN, EXACT_RECORD = 0, 50             # exact_step_end
CUT_RUNS = (2, 30, 70, 90)                  # cut_step


@dataclass(frozen=True)
class Case:
    name: str
    config: str                  # a configuration of tests/fast_matrix.py, or "twobody"
    kind: str
    value: float
    trigger: int
    method: nb.IntegratorMethod = RK89
    step_s: float = 60.0
    backward: bool = False
    n: int = 96                  # n columns of the ensemble (every 37th), repeated with start epochs 7 s later past 96
    cols: tuple = ()             # or these columns
    at_end: tuple = ()           # runs that start at the end epoch
    no_fuel: tuple = ()          # runs with negative propellant mass
    cap: int = CAP
    end: int = END
    edge: str = ""
    strict_only: bool = False

    @property
    def event(self):
        return (KIND[self.kind], self.value, self.trigger)

    def bounds(self):
        return fm.bounds(self.method)


def _ordinary():
    out = []
    for config in ("field", "srp", "all"):
        for kind in KINDS:
            for value in VALUES[kind]:
                triggers = TRIGGERS[:2] + (LAST_TRIGGER.get((kind, value), TRIGGERS[2]),)
                for trigger in (triggers if config == "field" else triggers[1:]):
                    out.append(Case(f"{config}-{kind}={value:g}-t{trigger}", config, kind, value, trigger))
    out.append(Case("field-Z=0-t7-RK4", "field", "Z", 0.0, 7, method=RK4, step_s=10.0, cap=2200))
    for kind in KINDS:
        out.append(Case(f"field-{kind}={VALUES[kind][0]:g}-t7-back", "field", kind, VALUES[kind][0], 7, backward=True, end=0))
    for kind in KINDS:
        for backward in (False, True):
            out.append(Case(f"twobody-{kind}={VALUES[kind][0]:g}-t2{'-back' if backward else ''}", "twobody", kind,
                            VALUES[kind][0], 2, backward=backward, end=0 if backward else END))
    for n, kind, trigger in ((33, "RMAG", 7), (70, "Z", 2), (160, "VMAG", 7)):
        out.append(Case(f"ragged{n}-{kind}-t{trigger}", "field", kind, VALUES[kind][0], trigger, n=n, edge="ragged"))
    return out


ORDINARY = _ordinary()
CASES = {c.name: c for c in ORDINARY}


# ---- dynamics and inputs
@functools.lru_cache(maxsize=None)
def dynamics(config):
    if config == "twobody":
        return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.new([]))
    return fm.dynamics(config)


def propagator(case: Case, mode=nb.MODE_FAST):
    return nb.Propagator.new(dynamics(case.config), case.method, nb.IntegratorOptions.with_fixed_step_s(case.step_s), mode=mode)


def almanac(config):
    return None if config == "twobody" else fm.almanac()


def _run(case: Case, st, cs, ep, end, event=None, cap=None):
    from oracle import pyoracle

    prop = propagator(case)
    packed = prop.dynamics.pack(nb.EARTH_J2000, almanac(case.config))
    step = np.full(st.shape[1], int(case.step_s * S), dtype=np.int64)
    out = pyoracle.propagate_batch(packed.c, prop.opts.to_c(prop.method), st, cs, ep, end, step,
                                   traj_capacity=case.cap if cap is None else cap, event=event) + (step,)
    for a in (out[0], out[1], out[3], step):
        a.setflags(write=False)
    return out


@functools.lru_cache(maxsize=None)
def inputs(case: Case):
    """(state[9][n], consts[4][n], epoch0[n], end epoch) of a case"""
    st, cs, ep = fm.ensemble()
    if case.cols:
        idx = np.array(case.cols)
    else:
        idx = np.arange(96) if case.n == 96 else (np.arange(case.n) * 37) % 96   # ragged: LEO and eccentric runs interleaved
    st, cs = st[:, idx].copy(), cs[:, idx].copy()
    ep = ep[idx] + (np.arange(len(idx)) // 96) * 7 * S
    if case.backward:   # from the plain forward run's state at 6 h
        fwd = _run(Case("fwd", case.config, case.kind, 0.0, 1, case.method, case.step_s, n=case.n, cols=case.cols), st, cs, ep, END,
                   cap=0)
        st, ep = fwd[0].copy(), fwd[1].copy()
    for i in case.at_end:
        ep[i] = case.end
    for i in case.no_fuel:
        st[8, i] = -1.0
    for a in (st, cs, ep):
        a.setflags(write=False)
    return st, cs, ep, case.end


@functools.lru_cache(maxsize=None)
def oracle(case: Case):
    """(state, epoch, details, status, (epochs, states, count), crossings, step array handed back): the oracle's event run"""
    st, cs, ep, end = inputs(case)
    return _run(case, st, cs, ep, end, case.event)


@functools.lru_cache(maxsize=None)
def free(case: Case):
    """The same runs with a trigger no run reaches: every step end up to the end epoch, the crossings of the whole span"""
    st, cs, ep, end = inputs(case)
    return _run(case, st, cs, ep, end, (KIND[case.kind], case.value, NO_STOP), cap=max(case.cap, CAP))


# ---- the event scalar, its sensitivity and the counter, on recordings ([6][...] arrays)
def scalar(kind, value, rv):
    """`event_eval` vectorised, same operation order as the kernels and the oracle"""
    x, y, z, vx, vy, vz = rv[:6]
    s = {"RMAG": lambda: np.sqrt((x * x + y * y) + z * z), "RDOTV": lambda: (x * vx + y * vy) + z * vz, "X": lambda: x + 0.0,
         "Y": lambda: y + 0.0, "Z": lambda: z + 0.0, "VMAG": lambda: np.sqrt((vx * vx + vy * vy) + vz * vz)}[kind]()
    return s - value


def perturbation(kind, rv, dr, dv):
    """|dy/dr| dr + |dy/dv| dv: how far a state within (dr, dv) of another can move the scalar"""
    r = np.sqrt((rv[:3] ** 2).sum(0))
    v = np.sqrt((rv[3:6] ** 2).sum(0))
    if kind == "RDOTV":
        return v * dr + r * dv
    if kind == "VMAG":
        return np.full(np.shape(r), dv)
    return np.full(np.shape(r), dr)


def rate(kind, rv, mu=nb.EARTH_J2000.mu):
    """d(scalar)/dt on the two-body flow (the bounds only need its size)"""
    r, v = rv[:3], rv[3:6]
    rn = np.sqrt((r ** 2).sum(0))
    a = -mu * r / rn ** 3
    if kind == "RMAG":
        return (r * v).sum(0) / rn
    if kind == "RDOTV":
        return (v * v).sum(0) + (r * a).sum(0)
    if kind == "VMAG":
        return (v * a).sum(0) / np.sqrt((v ** 2).sum(0))
    return v["XYZ".index(kind)]


def count_model(y, trigger, strict=True):
    """The counter of event.rs:141-144 on the scalar at the start and at the evaluated step ends y[0..m]: (step at which the
    run stops or None, crossings).  strict=False counts a zero product as a crossing (the mutation the matrix must see)."""
    count = 0
    for j in range(1, len(y)):
        p = y[j - 1] * y[j]
        if p < 0.0 or (not strict and p <= 0.0):
            count += 1
        if count >= trigger:
            return j, count
    return None, count


def evaluated(case: Case, i, rec=None):
    """The scalar at the start and at every step end the counter sees for run i (the final cut step excluded)"""
    t_ep, t_st, t_cnt = (rec or free(case)[4])
    k = int(t_cnt[i])
    st, cs, ep, end = inputs(case)
    # the last record ends the final step, which is not evaluated: a cut one forward; backward every step that reaches the end
    # epoch is the final one, even a full step (instance.rs:151-153 tests `epoch + step <= stop` there)
    if k > 1 and (case.backward or (end - int(ep[i])) % int(case.step_s * S) != 0):
        k -= 1
    return scalar(case.kind, case.value, t_st[:, :k, i]), t_st[:, :k, i]


# ---- the edge catalogue
def _strict_record():
    plain = free(Case("plain", "field", "X", 0.0, 1))[4]
    return float(plain[1][0, EXACT_RECORD, EXACT_RUN])


def _periapsis(i):
    st = fm.ensemble()[0]
    mu = nb.EARTH_J2000.mu
    r0, v0 = st[:3, i], st[3:6, i]
    rn, vn = np.linalg.norm(r0), np.linalg.norm(v0)
    a = 1.0 / (2.0 / rn - vn * vn / mu)
    e = np.linalg.norm(np.cross(v0, np.cross(r0, v0)) / mu - r0 / rn)
    return a * (1.0 - e)


@functools.lru_cache(maxsize=None)
def edges():
    st = fm.ensemble()[0]
    out = [
        Case("exact_step_end", "field", "X", _strict_record(), 1, edge="exact_step_end", strict_only=True),
        Case("start_on_value", "field", "X", float(st[0, 0]), 1, edge="start_on_value"),
        Case("two_in_one_step", "twobody", "RMAG", _periapsis(ECC_RUN) + PERIAPSIS_OFFSET, 1, cols=tuple(range(64, 96)),
             edge="two_in_one_step"),
        Case("statuses", "all", "Z", 0.0, 2, at_end=(3, 40, 70, 95), no_fuel=(5, 66, 95), edge="statuses"),
    ]
    base = CASES["field-RDOTV=0-t7"]
    n_steps = oracle(base)[2]["n_steps"][oracle(base)[3] == 0]
    out.append(Case("short_sink", "field", "RDOTV", 0.0, 7, cap=int(n_steps.min()), edge="short_sink"))
    return out


def cut_step_cases():
    """cut_step: run i alone, ending halfway between the trigger-th crossing (located on the oracle's recording) and the end of
    the step that holds it"""
    base = CASES["field-Z=0-t2"]
    ref = oracle(base)
    t_ep, t_st, t_cnt = ref[4]
    out = []
    for i in CUT_RUNS:
        assert ref[3][i] == 0
        k = int(t_cnt[i])
        tc = locate(t_ep[:k, i], t_st[:, :k, i], Event(KIND["Z"], 0.0, epoch_precision_ns=1))[0]
        end = tc + (int(t_ep[k - 1, i]) - tc) // 2
        out.append(Case(f"cut_step{i}", "field", "Z", 0.0, 2, cols=(i,), end=end, edge="cut_step"))
    return out


EDGE_NAMES = ("exact_step_end", "start_on_value", "two_in_one_step", "statuses", "short_sink")


# ---- host location (nyx_b200.event.locate_event) inside the last recorded step
def traj(t_ep, t_st):
    """the finalized Traj of one recording (epochs[k], states[6][k])"""
    sc = nb.Spacecraft.from_orbit(nb.Orbit.cartesian(*t_st[:, 0], int(t_ep[0]), nb.EARTH_J2000))
    return Traj(sc, np.array(t_ep, dtype=np.int64), np.ascontiguousarray(np.asarray(t_st).T)).finalize()


def locate(t_ep, t_st, ev: Event):
    """locate_event on one recording (epochs[k], states[6][k]) in step order: the bracket is the last step taken, which for a
    descending (backward) recording is its two earliest epochs.  Returns (epoch, state[6]) or None when the last step does not
    bracket a root."""
    from nyx_b200.event import locate_event

    tr = traj(t_ep, t_st)
    a, b = sorted((int(t_ep[-2]), int(t_ep[-1])))
    try:
        found = locate_event(tr, ev, bracket=(a, b))
    except ValueError:
        return None
    return found.epoch(), found.orbit.to_cartesian_pos_vel()


def locate_all(rec, ev: Event, run_status=None, runs=None):
    """(epoch[n], state[6][n], status[n]) with the convention of nyxb_event_locate, over `runs` (default: all)"""
    t_ep, t_st, t_cnt = rec
    n = t_ep.shape[1]
    ev_ep, ev_st, status = np.zeros(n, dtype=np.int64), np.full((6, n), np.nan), np.ones(n, dtype=np.int32)
    for i in (range(n) if runs is None else runs):
        k = min(int(t_cnt[i]), t_ep.shape[0])
        if k < 2 or (run_status is not None and run_status[i] & 0xFF):
            continue
        got = locate(t_ep[:k, i], t_st[:, :k, i], ev)
        if got is None:
            status[i] = 2
            continue
        ev_ep[i], ev_st[:, i], status[i] = got[0], got[1], 0
    return ev_ep, ev_st, status


# ---- 40-digit two-body arbiter of the located epoch
def kepler_root(r0, v0, t0_ns, kind, value, guess_ns):
    """Epoch (float ns) at which the scalar of the Kepler flow through (r0, v0) at t0 equals value, near guess_ns
    (mpmath.findroot on tests/span_edges.kepler)"""
    import mpmath as mp

    from tests.span_edges import kepler

    def f(dt_ns):
        r, v = kepler(r0, v0, mp.mpf(dt_ns))
        return mp.mpf(float(scalar(kind, value, np.concatenate([r, v]))))

    with mp.workdps(40):   # the scalar is rounded to f64: the root is good to ~1e-4 ns, far below what is asserted
        root = mp.findroot(f, (mp.mpf(guess_ns - t0_ns), mp.mpf(guess_ns - t0_ns + 1000)), solver="secant", verify=False)
        return float(t0_ns) + float(root)
