"""Impulsive differential correction: `Targeter` (md/opti/targeter.rs) with `try_achieve_fd` (md/opti/raphson_finite_diff.rs:41-747)
restricted to impulsive variables, over `nyxb_target_batch`: an ensemble of problems corrected together, one propagation launch of
every active problem's nominal and perturbed states per iteration.

Out of scope on this path, refused with `TargetingError`: finite-burn variables, `objective_frame` / `in_frame`, B-plane objectives and
any parameter that is not an orbital element of `nyxb_tgt_param`.
"""
from __future__ import annotations

import enum
from dataclasses import dataclass, field, replace
from typing import List, Optional, Sequence

import numpy as np

from . import abi
from .cosmic import Spacecraft, pack_spacecraft
from .od import LocalFrame
from .param import StateParameter, evaluate
from .propagator import Propagator, status_error


class TargetingError(RuntimeError):
    """`TargetingError` (md/opti/mod.rs); `variant` is the reference's variant name."""

    def __init__(self, variant: str, msg: str = ""):
        super().__init__(f"{variant}: {msg}" if msg else variant)
        self.variant = variant


class Vary(enum.IntEnum):
    """`Vary` (md/opti/target_variable.rs:28-85).  Only the six impulsive components run on this path."""

    PositionX = 0
    PositionY = 1
    PositionZ = 2
    VelocityX = 3
    VelocityY = 4
    VelocityZ = 5
    MnvrAlpha = 100
    MnvrAlphaDot = 101
    MnvrAlphaDDot = 102
    MnvrDelta = 103
    MnvrDeltaDot = 104
    MnvrDeltaDDot = 105
    StartEpoch = 106
    Duration = 107
    EndEpoch = 108
    ThrustX = 109
    ThrustY = 110
    ThrustZ = 111
    ThrustLevel = 112
    ThrustRateX = 113
    ThrustRateY = 114
    ThrustRateZ = 115
    ThrustAccelX = 116
    ThrustAccelY = 117
    ThrustAccelZ = 118

    def is_finite_burn(self) -> bool:
        return self.value >= 100


@dataclass
class Variable:
    """`Variable` with the reference's defaults for the impulsive components (target_variable.rs:219-244)."""

    component: Vary = Vary.VelocityX
    perturbation: float = 0.0001
    init_guess: float = 0.0
    max_step: float = 0.2
    max_value: float = 5.0
    min_value: float = -5.0

    @classmethod
    def from_vary(cls, vary: Vary) -> "Variable":
        if Vary(vary).is_finite_burn():
            raise TargetingError("UnsupportedVariable", f"{Vary(vary).name}: finite burns are not on this path")
        return cls(component=Vary(vary))

    def with_initial_guess(self, guess: float) -> "Variable":
        return replace(self, init_guess=float(guess))

    def with_pert(self, pert: float) -> "Variable":
        return replace(self, perturbation=float(pert))

    def with_min(self, v: float) -> "Variable":
        return replace(self, min_value=float(v))

    def with_max(self, v: float) -> "Variable":
        return replace(self, max_value=float(v))

    def valid(self) -> None:
        """`Variable::valid` (target_variable.rs:143-168)."""
        if self.max_step < 0.0:
            raise TargetingError("VariableError", f"{self.component.name}: max step is negative: {self.max_step}")
        if self.max_value < 0.0:
            raise TargetingError("VariableError", f"{self.component.name}: max value is negative: {self.max_value}")
        if self.min_value > self.max_value:
            raise TargetingError("VariableError", f"{self.component.name}: min value is greater than max value")


#: StateParameter -> enum nyxb_tgt_param
TGT_PARAMS = {p: i for i, p in enumerate([
    StateParameter.X, StateParameter.Y, StateParameter.Z, StateParameter.VX, StateParameter.VY, StateParameter.VZ, StateParameter.Rmag,
    StateParameter.Vmag, StateParameter.SemiMajorAxis, StateParameter.Eccentricity, StateParameter.Inclination, StateParameter.RAAN,
    StateParameter.AoP, StateParameter.TrueAnomaly, StateParameter.AoL, StateParameter.TrueLongitude, StateParameter.Period,
    StateParameter.Energy, StateParameter.Hmag, StateParameter.ApoapsisRadius, StateParameter.PeriapsisRadius, StateParameter.C3,
    StateParameter.Declination])}

#: variant names of the targeting statuses
TGT_STATUS = {abi.ERR_TGT_TOO_MANY_ITERATIONS: "TooManyIterations", abi.ERR_TGT_CORRECTION_INEFFECTIVE: "CorrectionIneffective",
              abi.ERR_TGT_SINGULAR_JACOBIAN: "SingularJacobian", abi.ERR_TGT_NON_FINITE: "NonFinite"}


@dataclass
class Objective:
    """`Objective` (md/objective.rs)."""

    parameter: StateParameter
    desired_value: float
    tolerance: float = 1e-3
    multiplicative_factor: float = 1.0
    additive_factor: float = 0.0

    @classmethod
    def new(cls, parameter: StateParameter, desired_value: float) -> "Objective":
        """Default tolerance of `default_event_precision` (md/param.rs:74-89): 0.1 s for the period, 1e-3 otherwise."""
        return cls(parameter, float(desired_value), 0.1 if parameter == StateParameter.Period else 1e-3)

    @classmethod
    def within_tolerance(cls, parameter: StateParameter, desired_value: float, tolerance: float) -> "Objective":
        return cls(parameter, float(desired_value), float(tolerance))

    def assess_value(self, achieved: float):
        err = self.multiplicative_factor * (self.desired_value - achieved) + self.additive_factor
        return abs(err) <= self.tolerance, err


@dataclass
class TargeterSolution:
    """`TargeterSolution` (md/opti/solution.rs:33-50)."""

    corrected_state: Spacecraft
    achieved_state: Spacecraft
    correction: np.ndarray
    variables: List[Variable]
    achieved_errors: np.ndarray
    achieved_objectives: List[Objective]
    iterations: int


@dataclass
class TargeterEnsembleSolution:
    """The outputs of `try_achieve_from_many`: corrected[9][n] / achieved[9][n] at the correction / achievement epochs,
    correction[n_vars][n], errors[n_objs][n], iterations[n], status[n] (0 converged; the last iteration's values on failure)."""

    targeter: "Targeter"
    states: List[Spacecraft]
    correction_epoch_ns: int
    achievement_epoch_ns: int
    corrected: np.ndarray
    achieved: np.ndarray
    correction: np.ndarray
    errors: np.ndarray
    iterations: np.ndarray
    status: np.ndarray

    def __len__(self) -> int:
        return len(self.states)

    def error(self, i: int) -> Optional[Exception]:
        """None when problem i converged, else the `TargetingError` or `PropagationError` try_achieve_from would raise."""
        code = int(self.status[i]) & 0xFF
        if code == 0:
            return None
        if code in TGT_STATUS:
            return TargetingError(TGT_STATUS[code], f"problem {i} after {int(self.iterations[i])} iterations")
        return status_error(code)

    def solution(self, i: int) -> TargeterSolution:
        err = self.error(i)
        if err is not None:
            raise err
        sc = self.states[i]
        return TargeterSolution(corrected_state=sc.with_vector(self.correction_epoch_ns, self.corrected[:, i]),
                                achieved_state=sc.with_vector(self.achievement_epoch_ns, self.achieved[:, i]),
                                correction=self.correction[:, i].copy(), variables=list(self.targeter.variables),
                                achieved_errors=self.errors[:, i].copy(), achieved_objectives=list(self.targeter.objectives),
                                iterations=int(self.iterations[i]))


@dataclass
class Targeter:
    """`Targeter` (md/opti/targeter.rs:34-56) for impulsive corrections."""

    prop: Propagator
    variables: List[Variable]
    objectives: List[Objective]
    iterations: int = 100
    correction_frame: Optional[LocalFrame] = None
    objective_frame: Optional[object] = None

    @classmethod
    def delta_v(cls, prop: Propagator, objectives: Sequence[Objective]) -> "Targeter":
        return cls(prop, [Variable.from_vary(v) for v in (Vary.VelocityX, Vary.VelocityY, Vary.VelocityZ)], list(objectives))

    @classmethod
    def delta_r(cls, prop: Propagator, objectives: Sequence[Objective]) -> "Targeter":
        return cls(prop, [Variable.from_vary(v) for v in (Vary.PositionX, Vary.PositionY, Vary.PositionZ)], list(objectives))

    @classmethod
    def vnc(cls, prop: Propagator, objectives: Sequence[Objective]) -> "Targeter":
        return cls(prop, [Variable.from_vary(v) for v in (Vary.VelocityX, Vary.VelocityY, Vary.VelocityZ)], list(objectives),
                   correction_frame=LocalFrame.VNC)

    @classmethod
    def new(cls, prop: Propagator, variables: Sequence[Variable], objectives: Sequence[Objective]) -> "Targeter":
        return cls(prop, list(variables), list(objectives))

    @classmethod
    def vnc_with_components(cls, prop: Propagator, variables: Sequence[Variable], objectives: Sequence[Objective]) -> "Targeter":
        return cls(prop, list(variables), list(objectives), correction_frame=LocalFrame.VNC)

    @classmethod
    def in_frame(cls, prop: Propagator, variables, objectives, objective_frame) -> "Targeter":
        return cls(prop, list(variables), list(objectives), objective_frame=objective_frame)

    def config_c(self) -> abi.TargetConfigC:
        """The nyxb_target_config of this targeter; raises TargetingError for what this path does not run."""
        if not self.objectives:
            raise TargetingError("UnderdeterminedProblem")
        if self.objective_frame is not None:
            raise TargetingError("UnsupportedObjectiveFrame", "objective frames are not on this path")
        if not 1 <= len(self.variables) <= 6 or len(self.objectives) > 6:
            raise TargetingError("UnsupportedProblem", "1 to 6 variables and objectives")
        frames = {None: abi.TGT_FRAME_NONE, LocalFrame.VNC: abi.TGT_FRAME_VNC, LocalFrame.RIC: abi.TGT_FRAME_RIC}
        if self.correction_frame not in frames:
            raise TargetingError("FrameError", f"correction frame {self.correction_frame!r} is not VNC or RIC")
        if self.iterations < 0:
            raise TargetingError("UnsupportedProblem", "iterations must not be negative")
        c = abi.TargetConfigC()
        c.n_vars, c.n_objs, c.correction_frame, c.iterations = len(self.variables), len(self.objectives), frames[self.correction_frame], int(self.iterations)
        for j, v in enumerate(self.variables):
            comp = Vary(v.component)
            if comp.is_finite_burn():
                raise TargetingError("UnsupportedVariable", f"{comp.name}: finite burns are not on this path")
            v.valid()
            if self.correction_frame is not None and comp < Vary.VelocityX:
                raise TargetingError("FrameError", f"Variable is in frame {self.correction_frame.name} but that frame cannot be used "
                                                   f"for a {comp.name} correction")
            if not (np.isfinite(v.perturbation) and v.perturbation != 0.0):
                raise TargetingError("VariableError", f"{comp.name}: the perturbation must be finite and nonzero")
            c.vars[j].component, c.vars[j].perturbation, c.vars[j].init_guess = int(comp), float(v.perturbation), float(v.init_guess)
            c.vars[j].max_step, c.vars[j].max_value, c.vars[j].min_value = float(v.max_step), float(v.max_value), float(v.min_value)
        for i, o in enumerate(self.objectives):
            if o.parameter not in TGT_PARAMS:
                raise TargetingError("UnsupportedObjective", f"{o.parameter} cannot be targeted on this path")
            c.objs[i].parameter, c.objs[i].desired, c.objs[i].tolerance = TGT_PARAMS[o.parameter], float(o.desired_value), float(o.tolerance)
            c.objs[i].multiplicative_factor, c.objs[i].additive_factor = float(o.multiplicative_factor), float(o.additive_factor)
        return c

    def try_achieve_from_many(self, states: Sequence[Spacecraft], correction_epoch_ns: int, achievement_epoch_ns: int,
                              almanac=None) -> TargeterEnsembleSolution:
        """Every state's problem in one `nyxb_target_batch` call.  The states share a frame; their epochs may differ."""
        states = list(states)
        cfg = self.config_c()
        if not states:
            raise ValueError("no states")
        st, cs, ep = pack_spacecraft(states)
        eng = self.prop.engine(states[0].orbit.frame, almanac)
        out = eng.target_batch(cfg, st, cs, ep, int(correction_epoch_ns), int(achievement_epoch_ns))
        return TargeterEnsembleSolution(self, states, int(correction_epoch_ns), int(achievement_epoch_ns), out["corrected"], out["achieved"],
                                        out["correction"], out["errors"], out["iterations"], out["status"])

    def try_achieve_from(self, initial_state: Spacecraft, correction_epoch_ns: int, achievement_epoch_ns: int,
                         almanac=None) -> TargeterSolution:
        """`Targeter::try_achieve_from` (targeter.rs:242-252)."""
        return self.try_achieve_from_many([initial_state], correction_epoch_ns, achievement_epoch_ns, almanac).solution(0)

    def _verify(self, states: List[Spacecraft], final_soa: np.ndarray, status: np.ndarray) -> List[Spacecraft]:
        mu = states[0].orbit.frame.mu_km3_s2()
        out = []
        for i, sc in enumerate(states):
            err = status_error(int(status[i]))
            if err is not None:
                raise err
            msg = ""
            for o in self.objectives:
                got = float(evaluate(o.parameter, final_soa[:6, i], mu))
                param_err = o.desired_value - got
                if abs(param_err) > o.tolerance:
                    msg += f"{o.parameter} = {got:.3f} BUT should be {o.desired_value:.3f} (± {o.tolerance:.1e}) (error = {param_err:.3f})"
            if msg:
                raise TargetingError("Verification", msg)
            out.append(sc)
        return out

    def apply_many(self, ensemble: TargeterEnsembleSolution, almanac=None) -> List[Spacecraft]:
        """`Targeter::apply` (targeter.rs:257-351) of every converged problem: the corrected states propagated to the achievement epoch
        in one batch call, each checked against the objectives (unscaled error within tolerance, else `Verification`)."""
        keep = [i for i in range(len(ensemble)) if ensemble.error(i) is None]
        sols = [ensemble.solution(i) for i in keep]
        return self._apply_solutions(sols, almanac)

    def apply(self, solution: TargeterSolution, almanac=None) -> Spacecraft:
        return self._apply_solutions([solution], almanac)[0]

    def _apply_solutions(self, sols: List[TargeterSolution], almanac) -> List[Spacecraft]:
        if not sols:
            return []
        starts = [s.corrected_state for s in sols]
        st, cs, ep = pack_spacecraft(starts)
        end = sols[0].achieved_state.epoch()
        out, out_ep, _, status = self.prop.engine(starts[0].orbit.frame, almanac).propagate_batch(st, cs, ep, end)
        finals = [sc.with_vector(int(out_ep[i]), out[:, i]) for i, sc in enumerate(starts)]
        return self._verify(finals, out, status)
