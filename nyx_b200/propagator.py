"""`Propagator` / `PropInstance` / `IntegratorOptions` — host-side mirror of
``propagators/{propagator,instance,options}.rs`` driving the CUDA engine through the C ABI.

All numerical work (RK stages, error control, step-size controller, force models) runs in
``csrc/`` on the GPU; this module only packs/unpacks arrays and mirrors the reference's
call surface so that user code and the parity tests read like the reference's own:

    setup = Propagator.rk89(dynamics, IntegratorOptions.with_adaptive_step_s(0.1, 30.0, 1e-12, ErrorControl.RSSCartesianState))
    prop = setup.with_(spacecraft, almanac)
    final = prop.for_duration(1 * Unit.Day)
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass, replace
from typing import List, Optional, Sequence

import numpy as np

from . import abi
from .cosmic import Spacecraft, Unit, pack_spacecraft
from .dynamics import PackedDynamics, SpacecraftDynamics
from .frames import Almanac, Frame


class IntegratorMethod(enum.IntEnum):
    """`IntegratorMethod` (rk_methods/mod.rs:65-79)."""

    RungeKutta89 = abi.RK89
    DormandPrince78 = abi.DP78
    DormandPrince45 = abi.DP45
    RungeKutta4 = abi.RK4
    CashKarp45 = abi.CK45
    Verner56 = abi.V56

    @classmethod
    def from_str(cls, s: str) -> "IntegratorMethod":
        for m in cls:
            if m.name.lower() == s.lower():
                return m
        valid = ",".join(m.name for m in cls)
        raise PropagationError(f"unknow integration method `{s}`, must be one of {valid}")

    def order(self) -> int:
        return {0: 9, 1: 8, 2: 5, 3: 4, 4: 5, 5: 6}[int(self)]

    def stages(self) -> int:
        return {0: 16, 1: 13, 2: 7, 3: 4, 4: 6, 5: 8}[int(self)]


class ErrorControl(enum.IntEnum):
    """`ErrorControl` (error_ctrl.rs:30-71)."""

    RSSCartesianState = abi.RSS_CARTESIAN_STATE
    RSSCartesianStep = abi.RSS_CARTESIAN_STEP
    RSSState = abi.RSS_STATE
    RSSStep = abi.RSS_STEP
    LargestError = abi.LARGEST_ERROR
    LargestState = abi.LARGEST_STATE
    LargestStep = abi.LARGEST_STEP


class PropagationError(RuntimeError):
    """`PropagationError` (propagators/mod.rs:68-92)."""


_STATUS_MSG = {
    abi.ERR_PROP_MATH: "PropMathError: try another integration method, or decrease step size; part of state vector is NaN",
    abi.ERR_FUEL_EXHAUSTED: "DynamicsError::FuelExhausted: negative prop mass",
    abi.ERR_MASSLESS: "DynamicsError::MasslessSpacecraft",
    abi.ERR_EPHEMERIS: "DynamicsError::DynamicsAlmanacError: epoch outside ephemeris coverage",
    abi.ERR_EVENT_NOT_FOUND: "PropagationError::NthEventError: end of the search window reached before the n-th event",
}


def status_error(code: int) -> Optional[PropagationError]:
    code = int(code) & 0xFF
    return None if code == 0 else PropagationError(_STATUS_MSG.get(code, f"status {code}"))


@dataclass
class IntegratorOptions:
    """`IntegratorOptions` (options.rs:42-186); durations are integer nanoseconds."""

    init_step: int = 60 * Unit.Second
    min_step: int = 0.001 * Unit.Second
    max_step: int = 2700 * Unit.Second
    tolerance: float = 1e-12
    attempts: int = 50
    fixed_step: bool = False
    error_ctrl: ErrorControl = ErrorControl.RSSCartesianStep
    # options.rs:60: propagate in this frame instead of the state's own; the state is transformed before the loop and back after
    # it (instance.rs:117-142, 167-176, 211-220).  The frame's own mu / shape, when set, are the ones used (instance.rs:131-137).
    integration_frame: Optional[Frame] = None

    @classmethod
    def default(cls) -> "IntegratorOptions":
        return cls()

    @classmethod
    def with_adaptive_step(cls, min_step: int, max_step: int, tolerance: float, error_ctrl: ErrorControl):
        return cls(init_step=max_step, min_step=min_step, max_step=max_step, tolerance=tolerance, attempts=50,
                   fixed_step=False, error_ctrl=error_ctrl)  # options.rs:66-82

    @classmethod
    def with_adaptive_step_s(cls, min_step: float, max_step: float, tolerance: float, error_ctrl: ErrorControl):
        return cls.with_adaptive_step(min_step * Unit.Second, max_step * Unit.Second, tolerance, error_ctrl)

    @classmethod
    def with_fixed_step(cls, step: int):
        return cls(init_step=step, min_step=step, max_step=step, tolerance=0.0, fixed_step=True, attempts=0,
                   error_ctrl=ErrorControl.RSSCartesianStep)  # options.rs:100-111

    @classmethod
    def with_fixed_step_s(cls, step: float):
        return cls.with_fixed_step(step * Unit.Second)

    @classmethod
    def with_tolerance(cls, tolerance: float):
        return cls(tolerance=tolerance)

    @classmethod
    def with_max_step(cls, max_step: int):
        o = cls()
        o.set_max_step(max_step)
        return o

    def set_max_step(self, max_step: int) -> None:
        if self.init_step > max_step:
            self.init_step = max_step
        self.max_step = max_step

    def set_min_step(self, min_step: int) -> None:
        if self.init_step < min_step:
            self.init_step = min_step
        self.min_step = min_step

    def to_c(self, method: IntegratorMethod, state_center: int = 0) -> abi.IntegOpts:
        """`state_center`: 0 = the states are expressed in the frame the dynamics were packed for; k + 1 = they are relative to
        body k of that packing (see `nyxb_integ_opts.state_center`)."""
        return abi.IntegOpts(int(method), int(self.error_ctrl), int(self.init_step), int(self.min_step),
                             int(self.max_step), float(self.tolerance), int(self.attempts), int(bool(self.fixed_step)),
                             int(state_center), 0)


@dataclass
class IntegrationDetails:
    """`IntegrationDetails` (propagators/mod.rs:49-56) + step counters."""

    step: int
    error: float
    attempts: int
    n_steps: int = 0
    n_rejected: int = 0
    n_rhs: int = 0


class Engine:
    """Owns one `nyxb_engine` (device tables for a (dynamics, method, options, frame) tuple)."""

    def __init__(self, packed: PackedDynamics, opts_c: abi.IntegOpts, mode: int, device: int):
        self._lib = abi.load_library()
        self._packed = packed
        self._opts = opts_c
        self.mode = mode
        self.device = device
        self._h = self._lib.nyxb_engine_create(packed.byref(), C.byref(opts_c), mode, device)
        if not self._h:
            raise PropagationError(f"nyxb_engine_create failed: {abi.last_error()}")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.nyxb_engine_destroy(self._h)
            self._h = None

    __del__ = close

    @property
    def handle(self):
        return self._h

    def set_lanes(self, lanes: int):
        rc = self._lib.nyxb_engine_set_lanes(self._h, lanes)
        if rc != 0:
            raise PropagationError(f"set_lanes({lanes}): {abi.last_error()}")

    def lanes(self) -> int:
        return self._lib.nyxb_engine_get_lanes(self._h)

    def set_kernel(self, kernel: int):
        """Force a kernel family (abi.KERNEL_AUTO / _THREAD / _COOP / _TRANSPOSED, `nyxb_engine_set_kernel`)."""
        rc = self._lib.nyxb_engine_set_kernel(self._h, kernel)
        if rc != 0:
            raise PropagationError(f"set_kernel({kernel}): {abi.last_error()}")

    def last_kernel(self) -> int:
        return self._lib.nyxb_engine_last_kernel(self._h)

    def set_tx_positions(self, positions: int):
        """Transposed kernel: walker warps per set of 32 trajectories (0 = chosen by the field's degree)."""
        if self._lib.nyxb_engine_set_tx_positions(self._h, positions) != 0:
            raise PropagationError(f"set_tx_positions({positions}): {abi.last_error()}")

    def set_tx_tuning(self, slice_attempts: int = 64, max_ctas: int = 0):
        """Transposed kernel: step attempts per time slice and a bound on the persistent CTAs (0: every resident slot)."""
        if self._lib.nyxb_engine_set_tx_tuning(self._h, slice_attempts, max_ctas) != 0:
            raise PropagationError(f"set_tx_tuning({slice_attempts}, {max_ctas}): {abi.last_error()}")

    def launch_count(self) -> int:
        return self._lib.nyxb_engine_launch_count(self._h)

    def last_kernel_ms(self) -> float:
        return self._lib.nyxb_engine_last_kernel_ms(self._h)

    def propagate_batch(self, state_soa, consts_soa, epoch0_ns, end_epoch_ns, step_ns=None, traj_capacity: int = 0,
                        event=None):
        """Host-buffer call of `nyxb_propagate_batch[_traj]`. Returns (state, epoch, details, status) and, when
        `traj_capacity` > 0, a fifth element (epochs[cap][n], states[6][cap][n], count[n]): the start state and the
        state after every accepted step (instance.rs:297-326).  `event=(kind, value, trigger)` adds the stop condition of
        `until_nth_event` (`nyxb_propagate_batch_event`, event.rs:88-211) and appends crossings[n] to the result."""
        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        n = state_soa.shape[1]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n]")
        out_state = np.empty((9, n))
        out_epoch = np.empty(n, dtype=np.int64)
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        step_ptr = None
        if step_ns is not None:
            if step_ns.dtype != np.int64 or step_ns.shape != (n,) or not step_ns.flags["C_CONTIGUOUS"]:
                raise ValueError("step_ns must be a contiguous int64[n] array")
            step_ptr = step_ns.ctypes.data
        sink = None
        if traj_capacity:
            t_ep = np.zeros((traj_capacity, n), dtype=np.int64)
            t_st = np.zeros((6, traj_capacity, n), dtype=np.float64)
            t_cnt = np.zeros(n, dtype=np.int64)
            sink = abi.TrajSink(int(traj_capacity), t_ep.ctypes.data, t_st.ctypes.data, t_cnt.ctypes.data)
        ev = None
        if event is not None:
            crossings = np.zeros(n, dtype=np.int32)
            ev = abi.EventC(int(event[0]), int(event[2]), float(event[1]), crossings.ctypes.data)
        rc = self._lib.nyxb_propagate_batch_event(self._h, n, state_soa.ctypes.data, consts_soa.ctypes.data,
                                                  epoch0_ns.ctypes.data, int(end_epoch_ns), step_ptr, out_state.ctypes.data,
                                                  out_epoch.ctypes.data, details.ctypes.data, status.ctypes.data,
                                                  C.byref(sink) if sink is not None else None,
                                                  C.byref(ev) if ev is not None else None)
        if rc != 0:
            raise PropagationError(f"nyxb_propagate_batch rc={rc}: {abi.last_error()}")
        ret = (out_state, out_epoch, details, status)
        if traj_capacity:
            ret = ret + ((t_ep, t_st, t_cnt),)
        if ev is not None:
            ret = ret + (crossings,)
        return ret

    def target_batch(self, cfg_c: abi.TargetConfigC, state_soa, consts_soa, epoch0_ns, correction_epoch_ns: int, achievement_epoch_ns: int):
        """`nyxb_target_batch`: `Targeter::try_achieve_fd` for n problems sharing the two epochs.  Returns a dict of corrected[9][n],
        achieved[9][n], correction[n_vars][n], errors[n_objs][n], iterations[n], status[n]."""
        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        n = state_soa.shape[1]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n]")
        out = {"corrected": np.empty((9, n)), "achieved": np.empty((9, n)), "correction": np.empty((max(cfg_c.n_vars, 0), n)),
               "errors": np.empty((max(cfg_c.n_objs, 0), n)), "iterations": np.zeros(n, dtype=np.int32), "status": np.zeros(n, dtype=np.int32)}
        rc = self._lib.nyxb_target_batch(self._h, C.byref(cfg_c), n, state_soa.ctypes.data, consts_soa.ctypes.data, epoch0_ns.ctypes.data,
                                         int(correction_epoch_ns), int(achievement_epoch_ns), out["corrected"].ctypes.data,
                                         out["achieved"].ctypes.data, out["correction"].ctypes.data, out["errors"].ctypes.data,
                                         out["iterations"].ctypes.data, out["status"].ctypes.data)
        if rc != 0:
            raise PropagationError(f"nyxb_target_batch rc={rc}: {abi.last_error()}")
        return out

    def resample(self, query_epochs_ns, recording=None, n: Optional[int] = None):
        """`nyxb_traj_resample`: `Traj::at` (traj.rs:83-126) for every trajectory of a recording at every query epoch, one launch.
        `recording` = the (epochs[cap][n], states[6][cap][n], count[n]) tuple `propagate_batch(traj_capacity=...)` returned, or
        None to reuse the recording of this engine's last propagation still resident on the device (pass its `n`).
        Returns (states[6][m][n], status[m][n]); status 1 = no interpolation data at that epoch (values NaN)."""
        q = np.ascontiguousarray(query_epochs_ns, dtype=np.int64)
        if q.ndim != 1:
            raise ValueError("query epochs must be a 1-D int64 array")
        sink = None
        if recording is not None:
            t_ep, t_st, t_cnt = (np.ascontiguousarray(a) for a in recording)
            cap, n = t_ep.shape
            if t_ep.dtype != np.int64 or t_st.shape != (6, cap, n) or t_st.dtype != np.float64 or t_cnt.shape != (n,) or t_cnt.dtype != np.int64:
                raise ValueError("expected epochs int64[cap][n], states float64[6][cap][n], count int64[n]")
            sink = abi.TrajSink(int(cap), t_ep.ctypes.data, t_st.ctypes.data, t_cnt.ctypes.data)
        elif n is None:
            raise ValueError("pass the number of trajectories of the resident recording")
        m = len(q)
        out = np.empty((6, m, n))
        status = np.empty((m, n), dtype=np.int32)
        rc = self._lib.nyxb_traj_resample(self._h, n, C.byref(sink) if sink is not None else None, m, q.ctypes.data,
                                          out.ctypes.data, status.ctypes.data)
        if rc != 0:
            raise PropagationError(f"nyxb_traj_resample rc={rc}: {abi.last_error()}")
        return out, status

    def locate_events(self, kind: int, value: float, epoch_precision_ns: int, recording=None, n: Optional[int] = None, run_status=None):
        """`nyxb_event_locate`: the Brent search of `until_nth_event` (event.rs:186-211) inside the last recorded step of every
        trajectory, one launch.  `recording` / `n` as for `resample`; `run_status` = the propagation's status array (failed runs
        are skipped).  Returns (event_epoch_ns[n], event_state[6][n], status[n]): status 0 located, 1 no bracket / skipped,
        2 the last step does not bracket a root."""
        sink = None
        if recording is not None:
            t_ep, t_st, t_cnt = (np.ascontiguousarray(a) for a in recording)
            cap, n = t_ep.shape
            if t_ep.dtype != np.int64 or t_st.shape != (6, cap, n) or t_st.dtype != np.float64 or t_cnt.shape != (n,) or t_cnt.dtype != np.int64:
                raise ValueError("expected epochs int64[cap][n], states float64[6][cap][n], count int64[n]")
            sink = abi.TrajSink(int(cap), t_ep.ctypes.data, t_st.ctypes.data, t_cnt.ctypes.data)
        elif n is None:
            raise ValueError("pass the number of trajectories of the resident recording")
        rs_ptr = None
        if run_status is not None:
            run_status = np.ascontiguousarray(run_status, dtype=np.int32)
            if run_status.shape != (n,):
                raise ValueError("run_status must be int32[n]")
            rs_ptr = run_status.ctypes.data
        ev_epoch = np.zeros(n, dtype=np.int64)
        ev_state = np.empty((6, n))
        status = np.empty(n, dtype=np.int32)
        rc = self._lib.nyxb_event_locate(self._h, n, C.byref(sink) if sink is not None else None, int(kind), float(value),
                                         int(epoch_precision_ns), rs_ptr, ev_epoch.ctypes.data, ev_state.ctypes.data, status.ctypes.data)
        if rc != 0:
            raise PropagationError(f"nyxb_event_locate rc={rc}: {abi.last_error()}")
        return ev_epoch, ev_state, status

    def propagate_batch_stm(self, state_soa, consts_soa, epoch0_ns, end_epoch_ns, stm_in=None, step_ns=None):
        """`nyxb_propagate_batch_stm`: `Spacecraft::with_stm()` + propagate (spacecraft.rs:203-227, 312-363).
        Returns (state[9][n], epoch[n], stm[81][n] column-major per trajectory, details, status)."""
        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        n = state_soa.shape[1]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n]")
        if stm_in is not None:
            stm_in = np.ascontiguousarray(stm_in, dtype=np.float64)
            if stm_in.shape != (81, n):
                raise ValueError("expected stm_in[81][n]")
        out_state = np.empty((9, n))
        out_epoch = np.empty(n, dtype=np.int64)
        out_stm = np.empty((81, n))
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        rc = self._lib.nyxb_propagate_batch_stm(
            self._h, n, state_soa.ctypes.data, consts_soa.ctypes.data, epoch0_ns.ctypes.data, int(end_epoch_ns),
            step_ns.ctypes.data if step_ns is not None else None, stm_in.ctypes.data if stm_in is not None else None,
            out_state.ctypes.data, out_epoch.ctypes.data, out_stm.ctypes.data, details.ctypes.data, status.ctypes.data)
        if rc != 0:
            raise PropagationError(f"nyxb_propagate_batch_stm rc={rc}: {abi.last_error()}")
        return out_state, out_epoch, out_stm, details, status

    def od_ekf_batch(self, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns,
                     covar0_soa, record_estimates: bool = False, estimates_capacity: Optional[int] = None):
        """`nyxb_od_ekf_batch`: n sequential Kalman filters over one tracking schedule in ONE launch (od/process/mod.rs:128-497).
        With `estimates_capacity` K, `nyxb_od_ekf_record_batch` also keeps the first K entries of each filter's ODSolution.estimates
        (ODSolution.records); the filter's results are the same bits."""
        from .od import ODSolution

        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        covar0_soa = np.ascontiguousarray(covar0_soa, dtype=np.float64)
        msr_epoch_ns = np.ascontiguousarray(msr_epoch_ns, dtype=np.int64)
        msr_tracker = np.ascontiguousarray(msr_tracker, dtype=np.int32)
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        n = state_soa.shape[1]
        m = msr_epoch_ns.shape[0]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,) or covar0_soa.shape != (81, n):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n], covar0[81][n]")
        if obs.shape != (m, 2, n) or msr_tracker.shape != (m,):
            raise ValueError("expected obs[m][2][n], tracker[m]")
        arc = abi.TrackingArcC(m, msr_epoch_ns.ctypes.data, msr_tracker.ctypes.data, obs.ctypes.data)
        out_state = np.empty((9, n)); out_epoch = np.empty(n, dtype=np.int64); out_cov = np.empty((81, n)); out_dev = np.empty((9, n))
        ratio = np.full((m, 2, n), np.nan); prefit = np.full((m, 2, n), np.nan); postfit = np.full((m, 2, n), np.nan)
        flags = np.zeros((m, n), dtype=np.int32)
        est_state = np.full((m, 9, n), np.nan) if record_estimates else None
        est_cov = np.full((m, 9, n), np.nan) if record_estimates else None
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        out = abi.OdOutputsC(out_state.ctypes.data, out_epoch.ctypes.data, out_cov.ctypes.data, out_dev.ctypes.data,
                             ratio.ctypes.data, prefit.ctypes.data, postfit.ctypes.data, flags.ctypes.data,
                             est_state.ctypes.data if record_estimates else None, est_cov.ctypes.data if record_estimates else None,
                             details.ctypes.data, status.ctypes.data)
        records = None
        if estimates_capacity is None:
            rc = self._lib.nyxb_od_ekf_batch(self._h, C.byref(cfg_c), int(n_stations), stations_c, C.byref(arc), n,
                                             state_soa.ctypes.data, consts_soa.ctypes.data, epoch0_ns.ctypes.data,
                                             covar0_soa.ctypes.data, C.byref(out))
        else:
            records, rec_c = _od_records(int(estimates_capacity), n)
            rc = self._lib.nyxb_od_ekf_record_batch(self._h, C.byref(cfg_c), int(n_stations), stations_c, C.byref(arc), n,
                                                    state_soa.ctypes.data, consts_soa.ctypes.data, epoch0_ns.ctypes.data,
                                                    covar0_soa.ctypes.data, C.byref(out), C.byref(rec_c))
        if rc != 0:
            raise PropagationError(f"nyxb_od_ekf_batch rc={rc}: {abi.last_error()}")
        covar = np.ascontiguousarray(out_cov.T.reshape(n, 9, 9).transpose(0, 2, 1))  # (c*9+r) -> [i][r][c]
        return ODSolution(out_state, out_epoch, covar, out_dev, ratio, prefit, postfit, flags, est_state, est_cov, details, status,
                          records=records)

    def od_smooth_batch(self, cfg_c, n_stations, stations_c, msr_tracker, obs, records: dict, filter_status, outputs=None):
        """`nyxb_od_smooth_batch`: ODSolution::smooth (od/process/solution/smooth.rs:104-249) of n filters in ONE launch, from their
        estimate records (dict as ODSolution.records).  `outputs`: the names among state, deviation, covar, fs_ratio, postfit to
        compute (default all).  Returns a dict of them ([K][..][n], NaN where the reference has None) and status [n]."""
        msr_tracker = np.ascontiguousarray(msr_tracker, dtype=np.int32)
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        filter_status = np.ascontiguousarray(filter_status, dtype=np.int32)
        cap, n = records["epoch"].shape
        m = msr_tracker.shape[0]
        if obs.shape != (m, 2, n) or filter_status.shape != (n,):
            raise ValueError("expected obs[m][2][n], filter_status[n]")
        rec_c = abi.OdRecordsC(cap, *(np.ascontiguousarray(records[k]).ctypes.data for k in _REC_KEYS))
        shapes = {"state": 9, "deviation": 9, "covar": 81, "fs_ratio": 9, "postfit": 2}
        want = shapes if outputs is None else {k: shapes[k] for k in outputs}
        r = {k: np.empty((cap, rows, n)) for k, rows in want.items()}
        r["status"] = np.zeros(n, dtype=np.int32)
        out = abi.SmoothOutputsC(*(r[k].ctypes.data if k in r else None for k in ("state", "deviation", "covar", "fs_ratio", "postfit")),
                                 r["status"].ctypes.data)
        arc = abi.TrackingArcC(m, None, msr_tracker.ctypes.data, obs.ctypes.data)
        rc = self._lib.nyxb_od_smooth_batch(self._h, C.byref(cfg_c), int(n_stations), stations_c, C.byref(arc), n, C.byref(rec_c),
                                            filter_status.ctypes.data, C.byref(out))
        if rc != 0:
            raise PropagationError(f"nyxb_od_smooth_batch rc={rc}: {abi.last_error()}")
        return r

    def od_position_batch(self, cfg_c, n_devices, devices_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns,
                          covar0_soa, record_estimates: bool = False, estimates_capacity: Optional[int] = None):
        """`nyxb_od_position_batch`: n sequential Kalman filters over one schedule of position fixes (obs [m][3][n], slot = type - X)
        in ONE launch; per-measurement outputs [m][3][n].  `record_estimates`: the estimated state and covariance diagonal after each
        measurement, as od_ekf_batch.  With `estimates_capacity` K the first K estimates of each filter are recorded (tags
        NYXB_OD_POS_TAG); the filter's results are the same bits."""
        return self._od_slots_batch("nyxb_od_position_batch", abi.PositionArcC, 3, cfg_c, n_devices, devices_c, msr_epoch_ns, msr_tracker,
                                    obs, state_soa, consts_soa, epoch0_ns, covar0_soa, record_estimates, estimates_capacity)

    def od_aer_batch(self, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns,
                     covar0_soa, record_estimates: bool = False, estimates_capacity: Optional[int] = None):
        """`nyxb_od_aer_batch`: od_position_batch's contract for ground stations with angles (nyxb_aer_station): obs [m][4][n], slot =
        type (Range, Doppler, Azimuth, Elevation); per-measurement outputs [m][4][n], the ratio of window w in slot w."""
        return self._od_slots_batch("nyxb_od_aer_batch", abi.TrackingArcC, 4, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker,
                                    obs, state_soa, consts_soa, epoch0_ns, covar0_soa, record_estimates, estimates_capacity)

    def od_interlink_batch(self, cfg_c, n_devices, devices_c, tx_sink, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns,
                           covar0_soa, record_estimates: bool = False, estimates_capacity: Optional[int] = None):
        """`nyxb_od_interlink_batch`: od_ekf_batch's contract for interlink transmitters (nyxb_interlink_tx) whose recordings are
        `tx_sink` (interlink_sink's (sink, n_tx, arrays)): obs [m][2][n], slot = type; per-measurement outputs [m][2][n]."""
        sink_c, n_tx, _keep = tx_sink
        return self._od_slots_batch("nyxb_od_interlink_batch", abi.TrackingArcC, 2, cfg_c, n_devices, devices_c, msr_epoch_ns, msr_tracker,
                                    obs, state_soa, consts_soa, epoch0_ns, covar0_soa, record_estimates, estimates_capacity,
                                    extra=(n_tx, C.byref(sink_c)))

    def _od_slots_batch(self, fn, arc_cls, ns, cfg_c, n_devices, devices_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa,
                        epoch0_ns, covar0_soa, record_estimates, estimates_capacity, extra=()):
        from .od import ODSolution

        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        covar0_soa = np.ascontiguousarray(covar0_soa, dtype=np.float64)
        msr_epoch_ns = np.ascontiguousarray(msr_epoch_ns, dtype=np.int64)
        msr_tracker = np.ascontiguousarray(msr_tracker, dtype=np.int32)
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        n = state_soa.shape[1]
        m = msr_epoch_ns.shape[0]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,) or covar0_soa.shape != (81, n):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n], covar0[81][n]")
        if obs.shape != (m, ns, n) or msr_tracker.shape != (m,):
            raise ValueError(f"expected obs[m][{ns}][n], tracker[m]")
        arc = arc_cls(m, msr_epoch_ns.ctypes.data, msr_tracker.ctypes.data, obs.ctypes.data)
        out_state = np.empty((9, n)); out_epoch = np.empty(n, dtype=np.int64); out_cov = np.empty((81, n)); out_dev = np.empty((9, n))
        ratio = np.full((m, ns, n), np.nan); prefit = np.full((m, ns, n), np.nan); postfit = np.full((m, ns, n), np.nan)
        flags = np.zeros((m, n), dtype=np.int32)
        est_state = np.full((m, 9, n), np.nan) if record_estimates else None
        est_cov = np.full((m, 9, n), np.nan) if record_estimates else None
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        out = abi.OdOutputsC(out_state.ctypes.data, out_epoch.ctypes.data, out_cov.ctypes.data, out_dev.ctypes.data,
                             ratio.ctypes.data, prefit.ctypes.data, postfit.ctypes.data, flags.ctypes.data,
                             est_state.ctypes.data if record_estimates else None, est_cov.ctypes.data if record_estimates else None,
                             details.ctypes.data, status.ctypes.data)
        records, rec_p = None, None
        if estimates_capacity is not None:
            records, rec_c = _od_records(int(estimates_capacity), n)
            rec_p = C.byref(rec_c)
        rc = getattr(self._lib, fn)(self._h, C.byref(cfg_c), int(n_devices), devices_c, *extra, C.byref(arc), n, state_soa.ctypes.data,
                                    consts_soa.ctypes.data, epoch0_ns.ctypes.data, covar0_soa.ctypes.data, C.byref(out), rec_p)
        if rc != 0:
            raise PropagationError(f"{fn} rc={rc}: {abi.last_error()}")
        covar = np.ascontiguousarray(out_cov.T.reshape(n, 9, 9).transpose(0, 2, 1))
        return ODSolution(out_state, out_epoch, covar, out_dev, ratio, prefit, postfit, flags, est_state, est_cov, details, status,
                          records=records)

    def od_position_smooth_batch(self, cfg_c, n_devices, devices_c, msr_tracker, obs, records: dict, filter_status, outputs=None):
        """`nyxb_od_position_smooth_batch`: od_smooth_batch for the records of od_position_batch; postfit is [K][3][n]."""
        return self._od_slots_smooth("nyxb_od_position_smooth_batch", abi.PositionArcC, 3, cfg_c, n_devices, devices_c, msr_tracker, obs,
                                     records, filter_status, outputs)

    def od_aer_smooth_batch(self, cfg_c, n_stations, stations_c, msr_tracker, obs, records: dict, filter_status, outputs=None):
        """`nyxb_od_aer_smooth_batch`: od_smooth_batch for the records of od_aer_batch; obs [m][4][n], postfit [K][4][n]."""
        return self._od_slots_smooth("nyxb_od_aer_smooth_batch", abi.TrackingArcC, 4, cfg_c, n_stations, stations_c, msr_tracker, obs,
                                     records, filter_status, outputs)

    def od_interlink_smooth_batch(self, cfg_c, n_devices, devices_c, tx_sink, msr_tracker, obs, records: dict, filter_status, outputs=None):
        """`nyxb_od_interlink_smooth_batch`: od_smooth_batch for the records of od_interlink_batch, with the same transmitter recordings."""
        sink_c, n_tx, _keep = tx_sink
        return self._od_slots_smooth("nyxb_od_interlink_smooth_batch", abi.TrackingArcC, 2, cfg_c, n_devices, devices_c, msr_tracker, obs,
                                     records, filter_status, outputs, extra=(n_tx, C.byref(sink_c)))

    def _od_slots_smooth(self, fn, arc_cls, ns, cfg_c, n_devices, devices_c, msr_tracker, obs, records, filter_status, outputs, extra=()):
        msr_tracker = np.ascontiguousarray(msr_tracker, dtype=np.int32)
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        filter_status = np.ascontiguousarray(filter_status, dtype=np.int32)
        cap, n = records["epoch"].shape
        m = msr_tracker.shape[0]
        if obs.shape != (m, ns, n) or filter_status.shape != (n,):
            raise ValueError(f"expected obs[m][{ns}][n], filter_status[n]")
        rec_c = abi.OdRecordsC(cap, *(np.ascontiguousarray(records[k]).ctypes.data for k in _REC_KEYS))
        shapes = {"state": 9, "deviation": 9, "covar": 81, "fs_ratio": 9, "postfit": ns}
        want = shapes if outputs is None else {k: shapes[k] for k in outputs}
        r = {k: np.empty((cap, rows, n)) for k, rows in want.items()}
        r["status"] = np.zeros(n, dtype=np.int32)
        out = abi.SmoothOutputsC(*(r[k].ctypes.data if k in r else None for k in ("state", "deviation", "covar", "fs_ratio", "postfit")),
                                 r["status"].ctypes.data)
        arc = arc_cls(m, None, msr_tracker.ctypes.data, obs.ctypes.data)
        rc = getattr(self._lib, fn)(self._h, C.byref(cfg_c), int(n_devices), devices_c, *extra, C.byref(arc), n, C.byref(rec_c),
                                    filter_status.ctypes.data, C.byref(out))
        if rc != 0:
            raise PropagationError(f"{fn} rc={rc}: {abi.last_error()}")
        return r

    def _bls_args(self, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns):
        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        msr_epoch_ns = np.ascontiguousarray(msr_epoch_ns, dtype=np.int64)
        msr_tracker = np.ascontiguousarray(msr_tracker, dtype=np.int32)
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        n = state_soa.shape[1]
        m = msr_epoch_ns.shape[0]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n]")
        if obs.shape != (m, 2, n) or msr_tracker.shape != (m,):
            raise ValueError("expected obs[m][2][n], tracker[m]")
        arc = abi.TrackingArcC(m, msr_epoch_ns.ctypes.data, msr_tracker.ctypes.data, obs.ctypes.data)
        return n, arc, (msr_epoch_ns, msr_tracker, obs), state_soa, consts_soa, epoch0_ns

    def od_bls_batch(self, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns):
        """`nyxb_od_bls_batch`: n batch least-squares estimates (`BatchLeastSquares::estimate`, od/blse/mod.rs:146-446) over one
        tracking schedule in ONE launch.  Returns a dict of the output arrays; covariances as [n][9][9]."""
        n, arc, keep, state_soa, consts_soa, epoch0_ns = self._bls_args(msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns)
        r = dict(state=np.empty((9, n)), epoch=np.empty(n, dtype=np.int64), covar=np.empty((81, n)), iterations=np.zeros(n, dtype=np.int32),
                 final_rms=np.empty(n), final_corr_pos_km=np.empty(n), converged=np.zeros(n, dtype=np.int32),
                 details=np.zeros(n, dtype=abi.DETAILS_DTYPE), status=np.zeros(n, dtype=np.int32))
        out = abi.BlsOutputsC(*(r[k].ctypes.data for k in ("state", "epoch", "covar", "iterations", "final_rms", "final_corr_pos_km",
                                                           "converged", "details", "status")))
        rc = self._lib.nyxb_od_bls_batch(self._h, C.byref(cfg_c), int(n_stations), stations_c, C.byref(arc), n, state_soa.ctypes.data,
                                         consts_soa.ctypes.data, epoch0_ns.ctypes.data, C.byref(out))
        if rc != 0:
            raise PropagationError(f"nyxb_od_bls_batch rc={rc}: {abi.last_error()}")
        r["covar"] = np.ascontiguousarray(r["covar"].T.reshape(n, 9, 9).transpose(0, 2, 1))  # (c*9+r) -> [i][r][c]
        return r

    def od_bls_evaluate_batch(self, cfg_c, n_stations, stations_c, msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns):
        """`nyxb_od_bls_evaluate_batch` (`BatchLeastSquares::evaluate`, od/blse/mod.rs:450-541): (rms[n], status[n])."""
        n, arc, keep, state_soa, consts_soa, epoch0_ns = self._bls_args(msr_epoch_ns, msr_tracker, obs, state_soa, consts_soa, epoch0_ns)
        rms = np.empty(n)
        status = np.zeros(n, dtype=np.int32)
        rc = self._lib.nyxb_od_bls_evaluate_batch(self._h, C.byref(cfg_c), int(n_stations), stations_c, C.byref(arc), n,
                                                  state_soa.ctypes.data, consts_soa.ctypes.data, epoch0_ns.ctypes.data, rms.ctypes.data,
                                                  status.ctypes.data)
        if rc != 0:
            raise PropagationError(f"nyxb_od_bls_evaluate_batch rc={rc}: {abi.last_error()}")
        return rms, status

    def od_predict_batch(self, cfg_c, state_soa, consts_soa, epoch0_ns, end_epoch_ns, covar0_soa, state_dev0_soa=None,
                         capacity: int = 0, record_states: bool = True, record_covars: bool = True):
        """`nyxb_od_predict_batch`: n covariance predictions (`KalmanODProcess::predict_until`, od/process/mod.rs:440-486) in ONE
        launch.  Records 0 .. capacity-1 of each run are kept; `record_states` / `record_covars` = False skip an array."""
        from .od import PredictionSolution

        state_soa = np.ascontiguousarray(state_soa, dtype=np.float64)
        consts_soa = np.ascontiguousarray(consts_soa, dtype=np.float64)
        epoch0_ns = np.ascontiguousarray(epoch0_ns, dtype=np.int64)
        end_epoch_ns = np.ascontiguousarray(end_epoch_ns, dtype=np.int64)
        covar0_soa = np.ascontiguousarray(covar0_soa, dtype=np.float64)
        n = state_soa.shape[1]
        if state_soa.shape != (9, n) or consts_soa.shape != (4, n) or epoch0_ns.shape != (n,) or end_epoch_ns.shape != (n,) \
                or covar0_soa.shape != (81, n):
            raise ValueError("expected state[9][n], consts[4][n], epoch0[n], end_epoch[n], covar0[81][n]")
        if state_dev0_soa is not None:
            state_dev0_soa = np.ascontiguousarray(state_dev0_soa, dtype=np.float64)
            if state_dev0_soa.shape != (9, n):
                raise ValueError("expected state_dev0[9][n]")
        cap = int(capacity)
        out_state = np.empty((9, n)); out_epoch = np.empty(n, dtype=np.int64); out_cov = np.empty((81, n)); out_dev = np.empty((9, n))
        details = np.zeros(n, dtype=abi.DETAILS_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        count = np.zeros(n, dtype=np.int64)
        rec_state = np.empty((cap, 9, n)) if cap and record_states else None
        rec_covar = np.empty((cap, 81, n)) if cap and record_covars else None
        out = abi.PredictOutputsC(out_state.ctypes.data, out_epoch.ctypes.data, out_cov.ctypes.data, out_dev.ctypes.data,
                                  details.ctypes.data, status.ctypes.data, cap,
                                  rec_state.ctypes.data if rec_state is not None else None,
                                  rec_covar.ctypes.data if rec_covar is not None else None, count.ctypes.data)
        rc = self._lib.nyxb_od_predict_batch(self._h, C.byref(cfg_c), n, state_soa.ctypes.data, consts_soa.ctypes.data,
                                             epoch0_ns.ctypes.data, end_epoch_ns.ctypes.data, covar0_soa.ctypes.data,
                                             state_dev0_soa.ctypes.data if state_dev0_soa is not None else None, C.byref(out))
        if rc != 0:
            raise PropagationError(f"nyxb_od_predict_batch rc={rc}: {abi.last_error()}")
        covar = np.ascontiguousarray(out_cov.T.reshape(n, 9, 9).transpose(0, 2, 1))  # (c*9+r) -> [i][r][c]
        return PredictionSolution(out_state, out_epoch, covar, out_dev, details, status, count, rec_state, rec_covar, epoch0_ns.copy(),
                                  int(cfg_c.max_step_ns))

    def propagate_batch_dev(self, n, state_ptr, consts_ptr, epoch0_ptr, end_epoch_ns, step_ptr, out_state_ptr,
                            out_epoch_ptr, details_ptr, status_ptr, stream_ptr=None):
        """Device-pointer call (`nyxb_propagate_batch_dev`): asynchronous on `stream_ptr`."""
        rc = self._lib.nyxb_propagate_batch_dev(self._h, n, state_ptr, consts_ptr, epoch0_ptr, int(end_epoch_ns), step_ptr,
                                                out_state_ptr, out_epoch_ptr, details_ptr, status_ptr, stream_ptr)
        if rc != 0:
            raise PropagationError(f"nyxb_propagate_batch_dev rc={rc}: {abi.last_error()}")


_REC_KEYS = ("epoch", "tag", "nominal", "deviation", "covar", "stm", "count")


def _od_records(cap: int, n: int):
    """Host arrays of nyxb_od_records for `cap` records of n filters, and the struct pointing at them."""
    if cap < 0:
        raise ValueError("negative estimates capacity")
    rec = {"epoch": np.empty((cap, n), dtype=np.int64), "tag": np.empty((cap, n), dtype=np.int64), "nominal": np.empty((cap, 9, n)),
           "deviation": np.empty((cap, 9, n)), "covar": np.empty((cap, 81, n)), "stm": np.empty((cap, 81, n)),
           "count": np.zeros(n, dtype=np.int64)}
    return rec, abi.OdRecordsC(cap, *(rec[k].ctypes.data for k in _REC_KEYS))


@dataclass
class Propagator:
    """`Propagator<SpacecraftDynamics>` (propagator.rs:34-118)."""

    dynamics: SpacecraftDynamics
    method: IntegratorMethod = IntegratorMethod.RungeKutta89
    opts: IntegratorOptions = None  # type: ignore[assignment]
    mode: int = abi.MODE_STRICT  # NYXB_MODE_STRICT (bit parity) | NYXB_MODE_FAST
    device: int = 0

    def __post_init__(self):
        if self.opts is None:
            self.opts = IntegratorOptions.default()
        self._engines = {}

    # constructors -----------------------------------------------------------------------------
    @classmethod
    def new(cls, dynamics, method: IntegratorMethod, opts: IntegratorOptions, **kw) -> "Propagator":
        return cls(dynamics, method, opts, **kw)

    @classmethod
    def rk89(cls, dynamics, opts: IntegratorOptions, **kw) -> "Propagator":
        return cls(dynamics, IntegratorMethod.RungeKutta89, opts, **kw)

    @classmethod
    def dp78(cls, dynamics, opts: IntegratorOptions, **kw) -> "Propagator":
        return cls(dynamics, IntegratorMethod.DormandPrince78, opts, **kw)

    @classmethod
    def default(cls, dynamics, **kw) -> "Propagator":
        return cls.rk89(dynamics, IntegratorOptions.default(), **kw)

    @classmethod
    def default_dp78(cls, dynamics, **kw) -> "Propagator":
        return cls.dp78(dynamics, IntegratorOptions.default(), **kw)

    def set_tolerance(self, tol: float):
        self.opts.tolerance = tol
        self._engines.clear()

    def set_max_step(self, step: int):
        self.opts.set_max_step(step)
        self._engines.clear()

    def set_min_step(self, step: int):
        self.opts.set_min_step(step)
        self._engines.clear()

    # engine cache ------------------------------------------------------------------------------
    _MAX_ENGINES = 8   # each engine owns device tables and staging buffers: the cache is bounded (oldest evicted)

    def engine(self, frame: Frame, almanac: Optional[Almanac]) -> Engine:
        """Device engine for states expressed in `frame`.  The cache key covers everything the engine was built from — method,
        mode, device, every option field, the dynamics object and the almanac (held by a strong reference, so `id()` cannot be
        recycled while the entry lives) — so mutating `prop.opts.*`, `prop.method` or `prop.dynamics` rebuilds it."""
        o = self.opts
        key = (id(almanac), frame, int(self.method), self.mode, self.device, id(self.dynamics),
               (o.init_step, o.min_step, o.max_step, o.tolerance, o.attempts, o.fixed_step, int(o.error_ctrl),
                getattr(o, "integration_frame", None)))
        hit = self._engines.get(key)
        if hit is not None:
            return hit[0]
        packed, opts_c = self.lower(frame, almanac)
        eng = Engine(packed, opts_c, self.mode, self.device)
        if len(self._engines) >= self._MAX_ENGINES:
            old = next(iter(self._engines))
            self._engines.pop(old)[0].close()
        self._engines[key] = (eng, almanac, self.dynamics)
        return eng

    def engines(self, frame: Frame, almanac: Optional[Almanac], devices: Sequence[int]) -> List[Engine]:
        """One engine per CUDA device for `nyx_b200.dist.propagate_batch_multi` (a fresh, uncached engine per device)."""
        packed, opts_c = self.lower(frame, almanac)
        return [Engine(packed, opts_c, self.mode, int(d)) for d in devices]

    def lower(self, frame: Frame, almanac: Optional[Almanac]):
        """(nyxb_dynamics, nyxb_integ_opts) for states expressed in `frame`.  With `opts.integration_frame` set to another frame
        the dynamics are lowered for THAT frame (its own mu / shape when given, instance.rs:131-137) and `state_center` tells the
        engine which body of the almanac the caller's states are relative to: it translates them in and out (instance.rs:117-142,
        167-176, 211-220)."""
        integ, state_center = frame, 0
        f = self.opts.integration_frame
        if f is not None and f.ephemeris_id != frame.ephemeris_id:
            if almanac is None or not almanac.has_body(frame.ephemeris_id):
                raise PropagationError(f"integration_frame {f.name}: the almanac holds no ephemeris of {frame.name} relative to it")
            known = almanac.frame_info(f)
            integ = replace(known, mu=f.mu if f.mu is not None else known.mu, radius_km=f.radius_km if f.radius_km is not None else known.radius_km)
            state_center = almanac.body_index(frame.ephemeris_id) + 1
        return self.dynamics.pack(integ, almanac), self.opts.to_c(self.method, state_center)

    # instances ---------------------------------------------------------------------------------
    def with_(self, state: Spacecraft, almanac: Optional[Almanac] = None) -> "PropInstance":
        """`Propagator::with` (propagator.rs:88-108)."""
        return PropInstance(self, state, almanac)

    def many_until_epoch(self, spacecraft: Sequence[Spacecraft], epoch_ns: int, almanac: Optional[Almanac] = None,
                         trajectory: bool = False, traj_capacity: int = 1024):
        """nyx-py `Propagator.many_until_epoch(list, epoch, trajectory)` (py_md.rs:224-271): ONE batched launch; failed runs
        are dropped (py_md.rs:251-254, 262-265).  Returns the final states, or with `trajectory=True` a list of
        (state, Traj) like the reference's `PropagationResult{state, trajectory}`; the recording sink grows until no run
        overflows it.  Start epochs may differ per spacecraft."""
        spacecraft = list(spacecraft)
        if not spacecraft:
            return []
        frame = spacecraft[0].orbit.frame
        st, cs, ep = pack_spacecraft(spacecraft)
        eng = self.engine(frame, almanac)
        if not trajectory:
            out, out_ep, _, status = eng.propagate_batch(st, cs, ep, epoch_ns)
            return [sc.with_vector(int(out_ep[i]), out[:, i]) for i, sc in enumerate(spacecraft) if (status[i] & 0xFF) == 0]
        from .trajectory import Traj

        cap = max(2, int(traj_capacity))
        while True:
            out, out_ep, det, status, (t_ep, t_st, t_cnt) = eng.propagate_batch(st, cs, ep, epoch_ns, traj_capacity=cap)
            if int(det["n_steps"].max()) + 1 <= cap:
                break
            cap = int(det["n_steps"].max()) + 1
        res = []
        for i, sc in enumerate(spacecraft):
            if (status[i] & 0xFF) != 0:
                continue
            k = int(t_cnt[i])
            res.append((sc.with_vector(int(out_ep[i]), out[:, i]), Traj(sc, t_ep[:k, i].copy(), np.ascontiguousarray(t_st[:, :k, i].T)).finalize()))
        return res

    def many_for_duration(self, spacecraft: Sequence[Spacecraft], duration_ns: int, almanac: Optional[Almanac] = None,
                          trajectory: bool = False, traj_capacity: int = 1024):
        """nyx-py `Propagator.many_for_duration` (py_md.rs:273-320): every spacecraft from its own epoch for `duration`; one
        launch per distinct end epoch (one, when they share the start epoch)."""
        spacecraft = list(spacecraft)
        ends = [sc.epoch() + int(duration_ns) for sc in spacecraft]
        out = [None] * len(spacecraft)
        for end in sorted(set(ends)):
            idx = [i for i, e in enumerate(ends) if e == end]
            ok = self._many_indexed([spacecraft[i] for i in idx], end, almanac, trajectory, traj_capacity)
            for j, r in ok:
                out[idx[j]] = r
        return [r for r in out if r is not None]

    def _many_indexed(self, spacecraft, epoch_ns, almanac, trajectory, traj_capacity):
        """many_until_epoch keeping the input index of the surviving runs"""
        marked = [s for s in spacecraft]
        res = self.many_until_epoch(marked, epoch_ns, almanac, trajectory, traj_capacity)
        if len(res) == len(marked):
            return list(enumerate(res))
        # some runs failed: recover the indices through the per-run status of a plain launch
        st, cs, ep = pack_spacecraft(marked)
        status = self.engine(marked[0].orbit.frame, almanac).propagate_batch(st, cs, ep, epoch_ns)[3]
        keep = [i for i in range(len(marked)) if (status[i] & 0xFF) == 0]
        return list(zip(keep, res))


class PropInstance:
    """`PropInstance` (instance.rs:41-499): one spacecraft, keeps the adapted step between calls."""

    def __init__(self, prop: Propagator, state: Spacecraft, almanac: Optional[Almanac]):
        self.prop = prop
        self.state = state
        self.almanac = almanac
        self.details = IntegrationDetails(step=prop.opts.init_step, error=0.0, attempts=1)
        self._step_ns = np.array([prop.opts.init_step], dtype=np.int64)  # instance.rs:56 step_size

    def latest_details(self) -> IntegrationDetails:
        return self.details

    def for_duration(self, duration_ns: int) -> Spacecraft:
        """instance.rs:265-267"""
        return self.until_epoch(self.state.epoch() + int(duration_ns))

    def for_duration_with_traj(self, duration_ns: int, capacity: Optional[int] = None):
        """instance.rs:297-326: returns (end state, Traj of the start state + every accepted step)."""
        return self.until_epoch_with_traj(self.state.epoch() + int(duration_ns), capacity)

    def until_epoch_with_traj(self, end_ns: int, capacity: Optional[int] = None):
        """instance.rs:330-340.  `capacity` bounds the records kept (default: enough for min-step-free propagation at
        1/4 of the current step; the call is repeated with a larger buffer if it overflowed)."""
        from .trajectory import Traj

        start = self.state
        span = abs(int(end_ns) - start.epoch())
        cap = capacity or max(64, 4 * span // max(abs(int(self._step_ns[0])), 1) + 64)
        while True:
            step_before = self._step_ns.copy()
            final, tr, overflow = self._run(end_ns, cap, start)
            if not overflow:
                break
            self.state, self._step_ns = start, step_before  # retry with a larger sink
            if capacity:   # an explicit capacity is a hard bound: a truncated Traj is never returned
                raise PropagationError(f"trajectory capacity {capacity} too small: the run takes {self.details.n_steps + 1} records")
            cap *= 4
        return final, tr

    def _run(self, end_ns, cap, start):
        from .trajectory import Traj

        st, cs, ep = pack_spacecraft([self.state])
        eng = self.prop.engine(self.state.orbit.frame, self.almanac)
        out, out_ep, det, status, (t_ep, t_st, t_cnt) = eng.propagate_batch(st, cs, ep, int(end_ns), self._step_ns, traj_capacity=cap)
        err = status_error(status[0])
        if err is not None:
            raise err
        d = det[0]
        if d["n_steps"] > 0:
            self.details = IntegrationDetails(int(d["step_ns"]), float(d["error"]), int(d["attempts"]), int(d["n_steps"]),
                                              int(d["n_rejected"]), int(d["n_rhs"]))
        self.state = self.state.with_vector(int(out_ep[0]), out[:, 0])
        k = int(t_cnt[0])
        tr = Traj(start, t_ep[:k, 0].copy(), np.ascontiguousarray(t_st[:, :k, 0].T)).finalize()
        return self.state, tr, int(d["n_steps"]) + 1 > cap

    def until_nth_event(self, max_duration_ns: int, event, trigger: int = 1, capacity: Optional[int] = None):
        """event.rs:88-211: propagate until `event` crossed zero `trigger` times (or raise NthEventError after
        `max_duration_ns`); returns (state interpolated at the event epoch, Traj up to the end of the bracketing step).
        The stop condition runs inside the propagation kernel; the Brent search (event.rs:186-196) runs on the recording it
        left on the device (`nyxb_event_locate`; `nyx_b200.event.locate_event` is the host restatement the tests check it with)."""
        from .trajectory import Traj

        start = self.state
        end_ns = start.epoch() + int(max_duration_ns)
        cap = capacity or max(64, 4 * abs(int(max_duration_ns)) // max(abs(int(self._step_ns[0])), 1) + 64)
        while True:
            step_before = self._step_ns.copy()
            st, cs, ep = pack_spacecraft([start])
            eng = self.prop.engine(start.orbit.frame, self.almanac)
            out, out_ep, det, status, (t_ep, t_st, t_cnt), crossings = eng.propagate_batch(
                st, cs, ep, end_ns, self._step_ns, traj_capacity=cap, event=(event.kind, event.value, trigger))
            if int(det[0]["n_steps"]) + 1 <= cap:
                break
            self._step_ns = step_before
            if capacity:   # the event search needs the bracketing (last) step on the recording: never search a truncated one
                raise PropagationError(f"trajectory capacity {capacity} too small: the run takes {int(det[0]['n_steps']) + 1} records")
            cap *= 4
        d = det[0]
        if d["n_steps"] > 0:
            self.details = IntegrationDetails(int(d["step_ns"]), float(d["error"]), int(d["attempts"]), int(d["n_steps"]),
                                              int(d["n_rejected"]), int(d["n_rhs"]))
        self.state = start.with_vector(int(out_ep[0]), out[:, 0])
        code = int(status[0]) & 0xFF
        if code == abi.ERR_EVENT_NOT_FOUND:
            raise PropagationError(f"NthEventError: nth={trigger}, found={int(crossings[0])}")
        err = status_error(status[0])
        if err is not None:
            raise err
        k = int(t_cnt[0])
        tr = Traj(start, t_ep[:k, 0].copy(), np.ascontiguousarray(t_st[:, :k, 0].T)).finalize()
        ev_ep, ev_st, ev_status = eng.locate_events(event.kind, event.value, event.epoch_precision_ns, n=1)  # resident recording
        if ev_status[0] != 0:
            raise PropagationError(f"event search failed in the bracketing step (status {int(ev_status[0])})")
        return tr._sc(int(ev_ep[0]), ev_st[:, 0]), tr

    def until_epoch(self, end_ns: int) -> Spacecraft:
        """instance.rs:279-282"""
        st, cs, ep = pack_spacecraft([self.state])
        eng = self.prop.engine(self.state.orbit.frame, self.almanac)
        out, out_ep, det, status = eng.propagate_batch(st, cs, ep, int(end_ns), self._step_ns)
        err = status_error(status[0])
        if err is not None:
            raise err
        d = det[0]
        if d["n_steps"] > 0:
            self.details = IntegrationDetails(int(d["step_ns"]), float(d["error"]), int(d["attempts"]), int(d["n_steps"]),
                                              int(d["n_rejected"]), int(d["n_rhs"]))
        self.state = self.state.with_vector(int(out_ep[0]), out[:, 0])
        return self.state
