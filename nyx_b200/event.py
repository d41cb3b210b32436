"""Events for event-terminated propagation (SURVEY.md §8 row (f)-3).

Reference: `PropInstance::until_nth_event` (propagators/event.rs:88-211) takes an anise `analysis::Event` (an open-ended
`ScalarExpr` + `Condition`); anise is a crates.io dependency that is not in the tree, so the scalar set here is CLOSED
(the ones the device kernels evaluate, `enum nyxb_event_kind`) and the condition is `Equals(value)`: the monitored
function is `scalar - value`, a crossing is a strict sign change between two accepted steps (event.rs:141-144).

The device finds the bracketing step; the root inside it is located here on the Hermite-interpolated trajectory with
Brent's method (event.rs:186-196 calls anise's `brent_solver`; restated from the published algorithm, parity unpinned).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable

import numpy as np

from . import abi
from .trajectory import Traj


@dataclass(frozen=True)
class Event:
    kind: int
    value: float = 0.0
    epoch_precision_ns: int = 1_000_000  # 1 ms: stop the bracket search below this width

    # ---- constructors named after what they locate
    @classmethod
    def radius(cls, r_km: float, **kw) -> "Event":
        return cls(abi.EVENT_RMAG, float(r_km), **kw)

    @classmethod
    def apsis(cls, **kw) -> "Event":
        """r.v = 0: periapsis (rising) and apoapsis (falling) alike, as `Event::apoapsis/periapsis` bracket them."""
        return cls(abi.EVENT_RDOTV, 0.0, **kw)

    @classmethod
    def node(cls, **kw) -> "Event":
        """z = 0 in the integration frame: ascending/descending node."""
        return cls(abi.EVENT_Z, 0.0, **kw)

    @classmethod
    def component(cls, axis: str, value: float = 0.0, **kw) -> "Event":
        return cls({"x": abi.EVENT_X, "y": abi.EVENT_Y, "z": abi.EVENT_Z}[axis.lower()], float(value), **kw)

    @classmethod
    def speed(cls, v_km_s: float, **kw) -> "Event":
        return cls(abi.EVENT_VMAG, float(v_km_s), **kw)

    def eval_rv(self, rv) -> float:
        """Same operation order as the kernels' `event_eval` (nyxb_device.cuh)."""
        x, y, z, vx, vy, vz = (float(c) for c in rv[:6])
        k = self.kind
        if k == abi.EVENT_RMAG:
            s = math.sqrt((x * x + y * y) + z * z)
        elif k == abi.EVENT_RDOTV:
            s = (x * vx + y * vy) + z * vz
        elif k == abi.EVENT_X:
            s = x
        elif k == abi.EVENT_Y:
            s = y
        elif k == abi.EVENT_Z:
            s = z
        elif k == abi.EVENT_VMAG:
            s = math.sqrt((vx * vx + vy * vy) + vz * vz)
        else:
            raise ValueError(f"unknown event kind {k}")
        return s - self.value

    def eval(self, spacecraft) -> float:
        return self.eval_rv(spacecraft.to_vector())


def brent(f: Callable[[float], float], a: float, b: float, xtol: float, max_iter: int = 100) -> float:
    """Brent's root bracketing (Brent 1973, ch. 4): inverse quadratic / secant steps guarded by bisection."""
    fa, fb = f(a), f(b)
    if fa == 0.0:
        return a
    if fb == 0.0:
        return b
    if fa * fb > 0.0:
        raise ValueError("root not bracketed")
    c, fc = a, fa
    d = e = b - a
    for _ in range(max_iter):
        if fb * fc > 0.0:
            c, fc = a, fa
            d = e = b - a
        if abs(fc) < abs(fb):
            a, b, c = b, c, b
            fa, fb, fc = fb, fc, fb
        tol = 2.0 * np.finfo(float).eps * abs(b) + 0.5 * xtol
        m = 0.5 * (c - b)
        if abs(m) <= tol or fb == 0.0:
            return b
        if abs(e) >= tol and abs(fa) > abs(fb):
            s = fb / fa
            if a == c:
                p, q = 2.0 * m * s, 1.0 - s
            else:
                q, r = fa / fc, fb / fc
                p = s * (2.0 * m * q * (q - r) - (b - a) * (r - 1.0))
                q = (q - 1.0) * (r - 1.0) * (s - 1.0)
            if p > 0.0:
                q = -q
            p = abs(p)
            if 2.0 * p < min(3.0 * m * q - abs(tol * q), abs(e * q)):
                e, d = d, p / q
            else:
                d = e = m
        else:
            d = e = m
        a, fa = b, fb
        b = b + d if abs(d) > tol else b + math.copysign(tol, m)
        fb = f(b)
    return b


def locate_event(traj: Traj, event: Event, bracket=None):
    """event.rs:166-211: bracket = the last two recorded states (the device stopped at the end of the crossing step);
    Brent on `event(traj.at(epoch))`, then the interpolated state at the event epoch.  `bracket` = (t_a, t_b), t_a < t_b, the
    step to search instead: a backward run's last step is the earliest one of its (ascending) trajectory, which is where
    `nyxb_event_locate` searches."""
    if len(traj) < 2:
        raise ValueError("trajectory too short to hold an event bracket")
    t_a, t_b = (int(traj.epochs_ns[-2]), int(traj.epochs_ns[-1])) if bracket is None else (int(bracket[0]), int(bracket[1]))
    t0 = t_a

    def f(dt_s: float) -> float:
        return event.eval(traj.at(t0 + int(round(dt_s * 1e9))))

    root_s = brent(f, 0.0, (t_b - t_a) * 1e-9, event.epoch_precision_ns * 1e-9)
    return traj.at(t0 + int(round(root_s * 1e9)))
