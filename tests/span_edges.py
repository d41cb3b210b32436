"""Edge-of-span catalogue for the step bookkeeping of `PropInstance::propagate` (instance.rs:87-262, 358-493), shared by the CPU
check of the inputs (tests/test_span_edges_inputs.py) and the GPU parity file (tests/test_gpu_span_edges.py).

The loop around the shared controller helpers (csrc/nyxb_device.cuh, ctl_*) is written once per kernel family: the per-thread
kernel, the lane-cooperative FAST and STRICT kernels, the transposed kernel and the OD arc (STM, filter, prediction).  Each case
here drives one branch of that loop at the edge of a span:

  zero duration; the final step cut to land on the stop epoch, run as a fixed step, then the previous step and its sign restored;
  the `stop == epoch` early return after a regular step; back-propagation; the adapted step carried to the next call; acceptance
  forced at the minimum step or at the last attempt (WARN_MAX_ATTEMPTS); the clamps of the proposed step, up to the saturation of
  `dur_from_seconds`; start epochs around century boundaries, where `dur_to_seconds` changes branch.

A case is one engine configuration (dynamics, method, options) and one sequence of end epochs; its ensemble (1, 33, 70 or 160
trajectories) mixes the edge trajectories with ordinary ones and with trajectories already at their end epoch, so that an edge
trajectory shares a warp, a lane group or a transposed-kernel set with trajectories that run, at a different position per case.

`model()` is an exact arbiter that does not use the oracle: Python integers for the epochs and steps, and the same IEEE double
operations as `Duration::to_seconds` / `f64 * Unit::Second` for the seconds.  It applies to fixed steps and to adaptive runs whose
decisions do not depend on the value of the error estimate:
  "minmax"  min_step == max_step: every attempt has h <= min_step and is accepted; the next step is +-min_step either way;
  "unmet"   tolerance 1e-300: an attempt is accepted only at the minimum step or at the last attempt; a rejected attempt retries
            at min_step, since 0.9 h (1e-300 / err)^(1/(order-1)) is far below it;
  "huge"    tolerance 1e300: every attempt is accepted and 0.9 h (1e300 / err)^(1/order) exceeds any max_step: it is clamped."""
import functools
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np

import nyx_b200 as nb
from tests import fast_matrix as fm
from tests.util import S, leo_ensemble

NS_PER_CENTURY = 3_155_760_000 * S
YEAR = 31_557_600 * S                    # Julian year
DAY = 86_400 * S
INT64_MAX, INT64_MIN = 2**63 - 1, -(2**63)
RK89, DP78, DP45, RK4 = (nb.IntegratorMethod.RungeKutta89, nb.IntegratorMethod.DormandPrince78, nb.IntegratorMethod.DormandPrince45,
                         nb.IntegratorMethod.RungeKutta4)
SIZES = (1, 33, 70, 160)
UNMET, HUGE = 1e-300, 1e300
LOSSY_MAX = 1_000_000_007                # 1.000000007 s: dur_from_seconds(dur_to_seconds(x)) = x - 1 on this step and its neighbours


# ---- hifitime's Duration <-> seconds, as the oracle (nyx_oracle.c) and the kernels (nyxb_device.cuh) compute them
def dur_to_seconds(ns: int) -> float:
    cent, nanos = divmod(ns, NS_PER_CENTURY)          # floor division: centuries may be -1, nanos in [0, NS_PER_CENTURY)
    sec, sub = divmod(nanos, S)
    if cent == 0:
        return float(sec) + float(sub) * 1e-9
    return float(cent) * 3155760000.0 + float(sec) + float(sub) * 1e-9


def dur_from_seconds(s: float) -> int:
    ns = s * 1e9
    if ns != ns:
        return 0
    if ns >= 9.2e18:
        return INT64_MAX
    if ns <= -9.2e18:
        return INT64_MIN
    return int(ns)


# ---- the case catalogue
@dataclass(frozen=True)
class Case:
    name: str
    branch: str                  # the branch the case exists for (see BRANCHES)
    dyn: str                     # "twobody" (K1 and the OD path) or "jgm3" (JGM-3 21x21 + Moon / Sun: every family)
    method: nb.IntegratorMethod
    control: str                 # "fixed", "minmax", "unmet" or "huge"
    step: int                    # fixed step, or (min, max) of the adaptive ones below
    edge: Tuple[int, ...]        # spans of the edge trajectories to the first end epoch (negative: backward)
    targets: Tuple[int, ...] = (0,)   # end epochs of the successive calls, relative to t0
    t0: int = 0                  # epoch of the region (the first end epoch is t0 + targets[0])
    init: Optional[int] = None   # opts.init_step (default: step / max_step)
    step_in: Optional[int] = None     # the step array handed to the first call (default: init)
    min_step: Optional[int] = None
    max_step: Optional[int] = None
    attempts: int = 50
    size: int = 33
    ordinary: int = 600 * S      # span of the ordinary trajectories (sign follows the first edge span)

    def opts(self) -> nb.IntegratorOptions:
        if self.control == "fixed":
            o = nb.IntegratorOptions.with_fixed_step(self.step)
            if self.init is not None:
                o.init_step = self.init
            return o
        mn = self.min_step if self.min_step is not None else self.step
        mx = self.max_step if self.max_step is not None else self.step
        tol = {"minmax": 1e-12, "unmet": UNMET, "huge": HUGE}[self.control]
        return nb.IntegratorOptions(init_step=self.init if self.init is not None else mx, min_step=mn, max_step=mx, tolerance=tol,
                                    attempts=self.attempts, fixed_step=False, error_ctrl=nb.ErrorControl.RSSCartesianStep)

    def first_step(self) -> int:
        return self.step_in if self.step_in is not None else int(self.opts().init_step)

    def ends(self):
        return [self.t0 + t for t in self.targets]

    def spans(self):
        """span to the first end epoch of every trajectory: edge spans at positions that move with the case, a few trajectories
        already at the end epoch, ordinary spans elsewhere"""
        n = self.size
        if n == 1:
            return [self.edge[0]]
        sign = -1 if self.edge[0] < 0 else 1
        out = []
        shift = sum(map(ord, self.name)) % 5
        for i in range(n):
            k = (i + shift) % 5
            if k == 1 or k == 3:
                out.append(self.edge[((i + shift) // 5 * 2 + (k == 3)) % len(self.edge)])
            elif (i + shift) % 11 == 0:
                out.append(0)
            else:
                out.append(sign * (self.ordinary + (i % 7) * (self.ordinary // 7 + 7)))
        if 0 not in out:
            out[-1] = 0
        return out

    def epoch0(self):
        e = self.ends()[0]
        return np.array([e - s for s in self.spans()], dtype=np.int64)


M = 60 * S     # the fixed step of most cases
CASES = [
    # fixed steps
    Case("fixed_1ns", "cut_first", "twobody", RK89, "fixed", M, (1, -1, 2, -2), size=33),
    Case("fixed_1ns_jgm3", "cut_first", "jgm3", RK89, "fixed", M, (1, -1), size=70),
    Case("fixed_multiple", "stop_eq_epoch", "twobody", RK89, "fixed", M, (M, 2 * M, 7 * M, -M, -3 * M), size=70),
    Case("fixed_multiple_jgm3", "stop_eq_epoch", "jgm3", DP78, "fixed", M, (M, 3 * M, 5 * M, -2 * M), size=160),
    Case("fixed_cut_1ns", "cut_1ns", "twobody", RK89, "fixed", M, (3 * M + 1, 5 * M + 1, -(2 * M + 1)), size=160),
    Case("fixed_cut_1ns_jgm3", "cut_1ns", "jgm3", RK89, "fixed", M, (2 * M + 1, -(4 * M + 1), M - 1), size=33),
    Case("fixed_not_multiple", "cut", "jgm3", DP45, "fixed", 45_500_000_000, (455 * S // 2, 1000 * S + 3, -(700 * S + 7)), size=70),
    Case("fixed_step_1ns", "stop_eq_epoch", "twobody", RK4, "fixed", 1, (5, -4, 1), size=33, ordinary=9),
    Case("fixed_step_in_larger", "cut_first", "jgm3", RK89, "fixed", M, (30 * S, -(59 * S)), step_in=7 * M, size=33),
    Case("fixed_back_then_fwd", "back_boundary_then_fwd", "jgm3", RK89, "fixed", M, (-3 * M, -M, -5 * M),
         targets=(0, 150 * S, 390 * S, -M), size=70),
    Case("fixed_back_then_fwd_2b", "back_boundary_then_fwd", "twobody", RK89, "fixed", M, (-2 * M, -4 * M),
         targets=(0, 5 * M, 5 * M + 1, 0), size=33),
    # adaptive, min_step == max_step
    Case("minmax", "forced_min", "jgm3", DP78, "minmax", 30 * S, (30 * S, 90 * S, 75 * S, -(60 * S), -(45 * S)), size=160),
    Case("minmax_init_below_min", "init_below_min", "jgm3", RK89, "minmax", 30 * S, (100 * S, -(100 * S), 5 * S), init=5 * S,
         size=33),
    Case("minmax_init_above_span", "init_above_span", "twobody", DP78, "minmax", 30 * S, (7 * S, -(3 * S), 29 * S + 999_999_999),
         size=70),
    Case("minmax_below_min_span", "span_below_min", "jgm3", DP78, "minmax", 30 * S, (1, -1, 10 * S), size=70),
    Case("minmax_chain", "step_carried", "jgm3", DP78, "minmax", 30 * S, (95 * S, -(95 * S)),
         targets=(0, -(185 * S), 60 * S, 60 * S + 1), step_in=7 * S, size=33),
    # adaptive, a tolerance that cannot be met
    Case("unmet_attempts1", "max_attempts", "jgm3", RK89, "unmet", None, (5 * M + 3, -(2 * M + 1), 1), min_step=S,
         max_step=600 * S, init=45 * S, attempts=1, size=70),
    Case("unmet_attempts1_2b", "max_attempts", "twobody", DP45, "unmet", None, (4 * M, -(M + 7)), min_step=S, max_step=600 * S,
         init=45 * S, attempts=1, size=33),
    Case("unmet_forced_min", "forced_min_rejected", "jgm3", DP78, "unmet", None, (9 * S + 5, 20 * S, -(7 * S)), min_step=S,
         max_step=600 * S, init=4 * S, attempts=255, size=33, ordinary=25 * S),
    Case("unmet_warn_at_min", "forced_min_rejected", "jgm3", RK89, "unmet", None, (6 * S, -(3 * S)), min_step=S, max_step=60 * S,
         init=4 * S, attempts=2, size=160, ordinary=15 * S),
    # adaptive, an error far below the tolerance: the proposed step is clamped to max_step
    Case("huge_clamp", "clamp_max", "jgm3", DP78, "huge", None, (200 * S + 3, 90 * S, -(250 * S)), min_step=S // 1000,
         max_step=90 * S, init=10 * S, size=70),
    Case("huge_chain", "step_carried", "twobody", RK89, "huge", None, (300 * S, -(100 * S)), targets=(0, 270 * S, -(91 * S), 1),
         min_step=S // 1000, max_step=90 * S, init=10 * S, size=160),
    Case("huge_lossy", "lossy_step", "jgm3", RK89, "huge", None, (5 * S + 500_000_000, 3 * S), min_step=S // 1000,
         max_step=LOSSY_MAX, init=300_000_000, size=33, ordinary=20 * S),
    Case("huge_saturating", "saturating_max", "twobody", RK89, "huge", None, (DAY, 3 * M + 1), t0=-20 * YEAR, min_step=S // 1000,
         max_step=INT64_MAX, init=M, size=33, ordinary=2 * DAY),
    # start epochs far from J2000 and around century boundaries
    Case("epoch_m20y", "negative_century", "jgm3", RK89, "fixed", M, (3 * M + 1, -(2 * M), 1), t0=-20 * YEAR, size=70),
    Case("epoch_p80y", "far_epoch", "jgm3", RK89, "fixed", M, (3 * M + 1, -(2 * M), 1), t0=80 * YEAR, size=33),
    Case("epoch_century_0", "century_boundary", "jgm3", DP78, "minmax", 30 * S, (1, -1, 2, -2, 30 * S + 1, -(30 * S + 1)), size=70),
    Case("epoch_century_m1", "century_boundary", "twobody", RK89, "fixed", M, (1, -1, M + 1, -(M + 1)), t0=-NS_PER_CENTURY, size=33),
    Case("epoch_century_p1", "century_boundary", "jgm3", RK89, "fixed", M, (1, -1, M + 1, -(M + 1)), t0=NS_PER_CENTURY, size=33),
    Case("epoch_century_unmet", "century_boundary", "twobody", DP78, "unmet", None, (1, -1, 45 * S + 1, -(45 * S + 1)),
         t0=NS_PER_CENTURY, min_step=S, max_step=600 * S, init=45 * S, attempts=1, size=70),
]
CASE = {c.name: c for c in CASES}
assert len(CASE) == len(CASES)

# branches, and the oracle counter that proves a case reaches its branch (tests/test_span_edges_inputs.py)
BRANCHES = {
    "cut_first": "the first step is the final cut step (n_steps == 1, |det.step_ns| < |step_ns|)",
    "stop_eq_epoch": "a forward span that is a multiple of the step ends on `stop == epoch` after a regular step",
    "cut_1ns": "the final cut step is 1 ns",
    "cut": "a final step shorter than the step",
    "back_boundary_then_fwd": "a backward call ends on a step boundary, the next forward call starts from the step it handed back",
    "forced_min": "adaptive steps accepted at h <= min_step",
    "init_below_min": "init_step < min_step: the first adaptive step is shorter than min_step, the next one is min_step",
    "init_above_span": "init_step longer than the span: the run is one cut step, the step array is handed back unchanged",
    "span_below_min": "a span shorter than min_step: one cut step below the minimum step",
    "step_carried": "the adapted step of one call is the first step of the next",
    "max_attempts": "acceptance forced at the last attempt: WARN_MAX_ATTEMPTS set",
    "forced_min_rejected": "first attempts rejected, acceptance forced at min_step (n_rejected > 0)",
    "clamp_max": "the proposed step is clamped to max_step",
    "lossy_step": "dur_from_seconds(dur_to_seconds(step)) != step: det.step_ns differs from the step array by 1 ns",
    "saturating_max": "max_step saturates dur_from_seconds: the step array holds INT64_MAX",
    "negative_century": "start epochs 20 years before J2000",
    "far_epoch": "start epochs 80 years after J2000",
    "century_boundary": "start epochs 1 ns on either side of a century boundary",
}
assert all(c.branch in BRANCHES for c in CASES)

PREDICT_CHUNK = 150 * S
PREDICT_CASES = [
    # (name, case whose options and dynamics are used, chunk length, spans of the edge runs); each run ends at the first chunk end at
    # or after its end epoch
    ("predict_fixed", Case("p_fixed", "cut", "twobody", RK89, "fixed", M, (0,), size=1), PREDICT_CHUNK,
     (PREDICT_CHUNK * 3 + 1, 1, PREDICT_CHUNK * 2, 2 * PREDICT_CHUNK - 1, 0, -S)),
    ("predict_fixed_jgm3", Case("p_fixed_jgm3", "cut", "jgm3", DP78, "fixed", 45 * S, (0,), size=1), PREDICT_CHUNK,
     (PREDICT_CHUNK * 2 + 7, PREDICT_CHUNK, 3 * S)),
    ("predict_huge_lossy", Case("p_huge", "lossy_step", "twobody", RK89, "huge", None, (0,), min_step=S // 1000, max_step=LOSSY_MAX,
                                init=300_000_000, size=1), 5 * S + 500_000_000, (16 * S + 3, 5 * S, 1)),
    # the minimum step loses 1 ns in its round trip through seconds: an adaptive step at the minimum advances LOSSY_MAX - 1 ns, a
    # fixed one LOSSY_MAX, so a chunk that ran fixed after the previous chunk's cut step moves the states off the oracle's bits
    ("predict_unmet", Case("p_unmet", "forced_min_rejected", "jgm3", DP78, "unmet", None, (0,), min_step=LOSSY_MAX,
                           max_step=600 * S, init=4 * S, attempts=255, size=1), 5 * S + 500_000_000, (30 * S, 7 * S)),
]


# ---- the exact integer model of the bookkeeping
class NotDecided(Exception):
    """The outcome depends on the value of the error estimate: the model does not apply."""


@dataclass
class Run:
    epoch: int
    step: int
    fixed: bool
    det_step: int = 0
    attempts: int = 1
    n_steps: int = 0
    n_rejected: int = 0
    n_attempts: int = 0        # every attempt (accepted or rejected) of the call: n_rhs = stages x n_attempts
    warn: bool = False
    records: list = field(default_factory=list)


def _derive(r: Run, o, control, order):
    """instance.rs:358-493 for the decision-determined controls: returns the step taken (ns)"""
    r.attempts = 1
    if r.fixed:
        r.n_attempts += 1
        r.det_step = r.step
        return r.step
    h = dur_to_seconds(r.step)
    min_s, max_s = dur_to_seconds(int(o.min_step)), dur_to_seconds(int(o.max_step))
    while True:
        r.n_attempts += 1
        accept = control == "huge" or h <= min_s or r.attempts >= o.attempts
        if not accept:
            if control != "unmet":
                raise NotDecided(f"{control}: an attempt of {h} s above the minimum step")
            r.attempts += 1
            r.n_rejected += 1
            h = min_s            # 0.9 h (1e-300 / err)^(1/(order - 1)) < min_step
            continue
        if r.attempts >= o.attempts:
            r.warn = True
        r.det_step = dur_from_seconds(h)
        if control == "huge":          # (1e300 / err)^(1/order) is huge: |proposed| > max_step
            h = max_s * (-1.0 if np.signbit(h) else 1.0)
        # "unmet": err > tolerance, h is kept; "minmax": either way the clamp below gives +-min_step, provided h rounds to a
        # non-zero number of nanoseconds (a sub-nanosecond h with err < tolerance could flip the sign of the result)
        nxt = dur_from_seconds(h)
        if control == "minmax" and nxt == 0:
            raise NotDecided("minmax: a sub-nanosecond attempt")
        if abs(nxt) < int(o.min_step):
            nxt = -int(o.min_step) if nxt < 0 else int(o.min_step)
        if control == "minmax":
            assert abs(nxt) == int(o.min_step) == int(o.max_step)
        r.step = nxt
        return r.det_step


def _add(a, b):
    s = a + b
    if not INT64_MIN <= s <= INT64_MAX:
        raise OverflowError("epoch + step overflows int64: undefined in every implementation")
    return s


def _single_step(r, o, control, order):
    dt = _derive(r, o, control, order)
    r.epoch = _add(r.epoch, dt)
    r.n_steps += 1
    r.records.append(r.epoch)


def propagate(r: Run, duration: int, o, control: str, order: int, max_steps: int = 200_000):
    """instance.rs:87-262 on the integer state of one trajectory"""
    if duration == 0:
        return
    stop = r.epoch + duration
    back = duration < 0
    if back:
        r.step = -r.step
    for _ in range(max_steps):
        epoch = r.epoch
        nxt = _add(epoch, r.step)
        if (not back and nxt > stop) or (back and nxt <= stop):
            if stop == epoch:
                return
            prev, prev_fixed = r.step, r.fixed
            r.step, r.fixed = stop - epoch, True
            _single_step(r, o, control, order)
            r.step, r.fixed = prev, prev_fixed
            if back:
                r.step = -r.step
            return
        _single_step(r, o, control, order)
    raise RuntimeError("the model did not reach the stop epoch")


ORDER = {RK89: 9, DP78: 8, DP45: 5, RK4: 4, nb.IntegratorMethod.CashKarp45: 5, nb.IntegratorMethod.Verner56: 6}


def model(case: Case):
    """Per call of the case, per trajectory: dict(epoch, step, det_step, attempts, n_steps, n_rejected, n_attempts, warn, records)
    (records: the recorded epochs of that call, the start epoch first)."""
    o = case.opts()
    out = []
    runs = [Run(int(e), case.first_step(), bool(o.fixed_step)) for e in case.epoch0()]
    for end in case.ends():
        call = []
        for r in runs:
            r.det_step, r.attempts, r.n_steps, r.n_rejected, r.n_attempts, r.warn = int(o.init_step), 1, 0, 0, 0, False
            r.records = [r.epoch]
            propagate(r, end - r.epoch, o, case.control, ORDER[case.method])
            call.append(dict(epoch=r.epoch, step=r.step, det_step=r.det_step, attempts=r.attempts, n_steps=r.n_steps,
                             n_rejected=r.n_rejected, n_attempts=r.n_attempts, warn=r.warn, records=list(r.records)))
        out.append(call)
    return out


def model_predict(case: Case, chunk: int, epoch0: int, end: int):
    """`predict_until` (od/process/mod.rs:440-486) on the integer state: chunks of `chunk` until the first chunk end at or after
    `end`; the integration step carries over from chunk to chunk and the step counters accumulate.  -> (record epochs, run)"""
    o = case.opts()
    r = Run(int(epoch0), int(o.init_step), bool(o.fixed_step))
    rec = [r.epoch]
    while True:
        propagate(r, chunk, o, case.control, ORDER[case.method])
        rec.append(r.epoch)
        if r.epoch >= end:
            return rec, r


# ---- dynamics, ensembles and the oracle's runs
TWOBODY_MU = nb.EARTH_J2000.mu


@functools.lru_cache(maxsize=None)
def dynamics(kind):
    if kind == "twobody":
        return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.new([]))
    return fm.dynamics("third_body")


@functools.lru_cache(maxsize=None)
def almanac(kind, t0):
    """Moon / Sun ephemerides over the epochs of a region (None for two-body)"""
    if kind == "twobody":
        return None
    return nb.Almanac.synthetic(nb.EARTH_J2000, t0 - 3 * DAY, 6.0, pad_days=1.0)


def propagator(case: Case, mode):
    return nb.Propagator.new(dynamics(case.dyn), case.method, case.opts(), mode=mode)


@functools.lru_cache(maxsize=None)
def ensemble(size, seed=3):
    """(state[9][n], consts[4][n]): the dispersed 300 km LEO of tests/util.leo_ensemble"""
    _, (st, cs, _) = leo_ensemble(size, seed=seed)
    st.setflags(write=False)
    cs.setflags(write=False)
    return st, cs


def capacity(case: Case):
    """a recording sink with room for every record of the longest call"""
    return max(len(t["records"]) for call in model(case) for t in call)


def chain(run, case: Case, epoch0=None, cap=0):
    """[(state, epoch, details, status, step array after the call, recording or None)] for the successive calls of a case;
    `run(state, consts, epoch0, end, step, cap)` is one propagate_batch call"""
    st, cs = ensemble(case.size)
    ep = case.epoch0() if epoch0 is None else epoch0
    step = np.full(case.size, case.first_step(), dtype=np.int64)
    out = []
    cur, cep = st, ep
    shift = 0 if epoch0 is None else int(epoch0[0] - case.epoch0()[0])
    for end in case.ends():
        ret = run(cur, cs, cep, end + shift, step, cap)
        cur, cep = ret[0], ret[1]
        out.append((ret[0], ret[1], ret[2], ret[3], step.copy(), ret[4] if cap else None))
    return out


@functools.lru_cache(maxsize=None)
def oracle_chain(name, shift=0):
    """The oracle's chain of a case (recording sink of `capacity(case)` records); `shift` moves every epoch by that many ns."""
    from oracle import pyoracle

    case = CASE[name]
    prop = propagator(case, nb.MODE_STRICT)
    packed = prop.dynamics.pack(nb.EARTH_J2000, almanac(case.dyn, case.t0))
    oc = prop.opts.to_c(prop.method)

    def run(st, cs, ep, end, step, cap):
        return pyoracle.propagate_batch(packed.c, oc, st, cs, ep, end, step, traj_capacity=cap)

    return chain(run, case, case.epoch0() + shift, capacity(case))


@functools.lru_cache(maxsize=None)
def oracle_stm_chain(name):
    from oracle import pyoracle

    case = CASE[name]
    prop = propagator(case, nb.MODE_STRICT)
    packed = prop.dynamics.pack(nb.EARTH_J2000, almanac(case.dyn, case.t0))
    oc = prop.opts.to_c(prop.method)

    def run(st, cs, ep, end, step, cap):
        s, e, stm, det, status = pyoracle.propagate_batch_stm(packed.c, oc, st, cs, ep, end, step_ns=step)
        return s, e, det, status, stm

    return chain(run, case, cap=1)


# ---- 40-digit universal-variable Kepler solution (Curtis, Orbital Mechanics for Engineering Students, algorithm 3.3 / 3.4)
def kepler(r0, v0, dt_ns, mu=TWOBODY_MU, dps=40):
    """position (km) and velocity (km/s) after dt_ns on the two-body orbit through (r0, v0); dt_ns may be an mpmath number
    (a fraction of a nanosecond, for root searches)"""
    import mpmath as mp

    with mp.workdps(dps):
        mu = mp.mpf(mu)
        r0 = [mp.mpf(float(x)) for x in r0]
        v0 = [mp.mpf(float(x)) for x in v0]
        dt = (dt_ns if isinstance(dt_ns, mp.mpf) else mp.mpf(int(dt_ns))) / 10**9
        if dt == 0:
            return np.array([float(x) for x in r0]), np.array([float(x) for x in v0])
        rn = mp.sqrt(sum(x * x for x in r0))
        vr = sum(a * b for a, b in zip(r0, v0)) / rn
        alpha = 2 / rn - sum(x * x for x in v0) / mu
        smu = mp.sqrt(mu)

        def C(z):
            if z > 0:
                return (1 - mp.cos(mp.sqrt(z))) / z
            if z < 0:
                return (mp.cosh(mp.sqrt(-z)) - 1) / (-z)
            return mp.mpf(1) / 2

        def Sf(z):
            if z > 0:
                sz = mp.sqrt(z)
                return (sz - mp.sin(sz)) / sz**3
            if z < 0:
                sz = mp.sqrt(-z)
                return (mp.sinh(sz) - sz) / sz**3
            return mp.mpf(1) / 6

        x = smu * abs(alpha) * dt
        x = x if dt > 0 else -abs(x)
        for _ in range(200):
            z = alpha * x * x
            Cz, Sz = C(z), Sf(z)
            F = rn * vr / smu * x * x * Cz + (1 - alpha * rn) * x**3 * Sz + rn * x - smu * dt
            dF = rn * vr / smu * x * (1 - alpha * x * x * Sz) + (1 - alpha * rn) * x * x * Cz + rn
            dx = F / dF
            x -= dx
            if abs(dx) < mp.mpf(10) ** (-dps + 5):
                break
        z = alpha * x * x
        Cz, Sz = C(z), Sf(z)
        f = 1 - x * x / rn * Cz
        g = dt - x**3 * Sz / smu
        r = [f * a + g * b for a, b in zip(r0, v0)]
        rr = mp.sqrt(sum(c * c for c in r))
        fd = smu / (rr * rn) * (alpha * x**3 * Sz - x)
        gd = 1 - x * x / rr * Cz
        v = [fd * a + gd * b for a, b in zip(r0, v0)]
        return np.array([float(c) for c in r]), np.array([float(c) for c in v])


@functools.lru_cache(maxsize=None)
def kepler_final(name):
    """[6][n]: the Kepler state at the final epoch of the oracle's chain, from the start state of the case"""
    case = CASE[name]
    st, _ = ensemble(case.size)
    ep0 = case.epoch0()
    fin = oracle_chain(name)[-1][1]
    out = np.empty((6, case.size))
    for i in range(case.size):
        r, v = kepler(st[:3, i], st[3:6, i], int(fin[i]) - int(ep0[i]))
        out[:3, i], out[3:, i] = r, v
    return out


def kepler_distance(name, final_state):
    """max |dr| (km) of a final state [9][n] from the Kepler solution"""
    k = kepler_final(name)
    return float(np.sqrt(((final_state[:3] - k[:3]) ** 2).sum(0)).max())


def kepler_bound(name):
    """the GPU's distance bound from Kepler: twice the oracle's distance, and at least the oracle's distance plus the FAST
    fixed-step parity bound (a FAST result within that bound of the oracle is within this one of Kepler)"""
    d = kepler_distance(name, oracle_chain(name)[-1][0])
    return max(2.0 * d, d + fm.FIXED_DR)


TWOBODY_CASES = [c.name for c in CASES if c.dyn == "twobody"]
# huge_saturating takes one step of 60 s and then a cut step of up to two days: a bookkeeping case, not an accurate orbit
KEPLER_CASES = [n for n in TWOBODY_CASES if n != "huge_saturating"]
EPOCH_SHIFTS = (-20 * YEAR, 80 * YEAR, NS_PER_CENTURY - 1, NS_PER_CENTURY + 1, -NS_PER_CENTURY - 1, -NS_PER_CENTURY + 1, -1, 1)


# ---- covariance prediction (KalmanODProcess::predict_until) at chunk ends that miss the end epoch
PREDICT = {p[0]: p for p in PREDICT_CASES}


def predict_process(pname, mode=nb.MODE_STRICT):
    _, case, chunk, _ = PREDICT[pname]
    odp = nb.KalmanODProcess(propagator(case, mode), nb.KalmanVariant.ReferenceUpdate, None, {}, almanac(case.dyn, case.t0))
    odp.max_step = chunk
    return odp


@functools.lru_cache(maxsize=None)
def predict_inputs(pname):
    """[(spacecraft, estimate, consts[4], end epoch)]: start epochs staggered at the nanosecond"""
    _, case, _, spans = PREDICT[pname]
    st, _ = ensemble(33)
    out = []
    for i, span in enumerate(spans):
        e0 = case.t0 + i * 7 * S + 3 * i
        sc = nb.Spacecraft(orbit=nb.Orbit.cartesian(*st[:6, i], e0, nb.EARTH_J2000), mass=nb.Mass(100.0, 20.0, 0.0))
        est = nb.KfEstimate.from_diag(sc, [1.0, 1.0, 1.0, 1e-6, 1e-6, 1e-6, 0.0, 0.0, 0.0])
        cs = np.array([sc.mass.dry_mass_kg, sc.mass.extra_mass_kg, sc.srp.area_m2, sc.drag.area_m2])
        out.append((sc, est, cs, e0 + span))
    return out


def predict_oracle_args(pname):
    _, case, _, _ = PREDICT[pname]
    odp = predict_process(pname)
    return dynamics(case.dyn).pack(nb.EARTH_J2000, almanac(case.dyn, case.t0)).c, odp.prop.opts.to_c(odp.prop.method), odp.config_c()
