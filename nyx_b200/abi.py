"""ctypes mirror of ``include/nyxb.h`` (the C-ABI PODs) and loader of ``libnyxb.so``.

The structs are layout-identical to the header; a unit test checks ``ctypes.sizeof``
against the values the library reports.  No compute lives here.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

NYXB_ABI_VERSION = 4  # include/nyxb.h
NYXB_MAX_FIELDS = 3
KERNEL_AUTO, KERNEL_THREAD, KERNEL_COOP, KERNEL_TRANSPOSED = 0, 1, 2, 3  # enum nyxb_kernel
NYXB_MAX_BODIES = 8
NYXB_CENTRAL_BODY = -1

# enum nyxb_method — propagators/rk_methods/mod.rs:65-79
RK89, DP78, DP45, RK4, CK45, V56 = range(6)
# enum nyxb_error_ctrl — propagators/error_ctrl.rs:30-71
(RSS_CARTESIAN_STATE, RSS_CARTESIAN_STEP, RSS_STATE, RSS_STEP, LARGEST_ERROR, LARGEST_STATE, LARGEST_STEP) = range(7)
# enum nyxb_status
OK, ERR_PROP_MATH, ERR_FUEL_EXHAUSTED, ERR_MASSLESS, ERR_EPHEMERIS, ERR_EVENT_NOT_FOUND = range(6)
WARN_MAX_ATTEMPTS = 0x100
ERR_TGT_TOO_MANY_ITERATIONS, ERR_TGT_CORRECTION_INEFFECTIVE, ERR_TGT_SINGULAR_JACOBIAN, ERR_TGT_NON_FINITE = 13, 14, 15, 16
# enum nyxb_tgt_frame
TGT_FRAME_NONE, TGT_FRAME_VNC, TGT_FRAME_RIC = 0, 1, 2
# enum nyxb_mode
MODE_STRICT, MODE_FAST = 0, 1
# enum nyxb_event_kind
EVENT_NONE, EVENT_RMAG, EVENT_RDOTV, EVENT_X, EVENT_Y, EVENT_Z, EVENT_VMAG = range(7)
# enum nyxb_density
DENSITY_CONSTANT, DENSITY_EXPONENTIAL, DENSITY_STDATM = range(3)

c_double_p = C.POINTER(C.c_double)
c_int64_p = C.POINTER(C.c_int64)
c_int32_p = C.POINTER(C.c_int32)


class IntegOpts(C.Structure):
    _fields_ = [
        ("method", C.c_int32),
        ("error_ctrl", C.c_int32),
        ("init_step_ns", C.c_int64),
        ("min_step_ns", C.c_int64),
        ("max_step_ns", C.c_int64),
        ("tolerance", C.c_double),
        ("attempts", C.c_int32),
        ("fixed_step", C.c_int32),
        ("state_center", C.c_int32),   # integration_frame: 0 none, k + 1: the states are relative to dynamics.bodies[k]
        ("_pad", C.c_int32),
    ]


class Rotation(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("_pad", C.c_int32),
        ("ra0_deg", C.c_double),
        ("ra1_deg_cy", C.c_double),
        ("dec0_deg", C.c_double),
        ("dec1_deg_cy", C.c_double),
        ("w0_deg", C.c_double),
        ("w1_deg_day", C.c_double),
    ]


class GravityFieldC(C.Structure):
    _fields_ = [
        ("degree", C.c_int32),
        ("order", C.c_int32),
        ("mu_km3_s2", C.c_double),
        ("r_eq_km", C.c_double),
        ("c_nm", c_double_p),
        ("s_nm", c_double_p),
        ("rot", Rotation),
        ("body", C.c_int32),   # NYXB_CENTRAL_BODY or index into DynamicsC.bodies: the body the field belongs to
        ("_pad", C.c_int32),
    ]


class BodyC(C.Structure):
    _fields_ = [
        ("mu_km3_s2", C.c_double),
        ("radius_km", C.c_double),
        ("t0_ns", C.c_int64),
        ("interval_ns", C.c_int64),
        ("n_intervals", C.c_int32),
        ("n_coeffs", C.c_int32),
        ("coeffs", c_double_p),
    ]


class SrpC(C.Structure):
    _fields_ = [
        ("phi_w_m2", C.c_double),
        ("sun_body", C.c_int32),
        ("n_shadow", C.c_int32),
        ("shadow_body", C.c_int32 * 4),
        ("estimate", C.c_int32),
        ("_pad", C.c_int32),
    ]


class DragC(C.Structure):
    _fields_ = [
        ("density", C.c_int32),
        ("_pad", C.c_int32),
        ("rho0", C.c_double),
        ("r0", C.c_double),
        ("ref_alt_m", C.c_double),
        ("r_eq_km", C.c_double),
        ("rot", Rotation),
    ]


class DynamicsC(C.Structure):
    _fields_ = [
        ("mu_central_km3_s2", C.c_double),
        ("central_radius_km", C.c_double),
        ("n_bodies", C.c_int32),
        ("n_gravity", C.c_int32),
        ("bodies", C.POINTER(BodyC)),
        ("point_mass_mask", C.c_uint32),
        ("n_point_masses", C.c_int32),
        ("gravity", C.POINTER(GravityFieldC)),   # array of n_gravity fields, accel-model order
        ("srp", C.POINTER(SrpC)),
        ("drag", C.POINTER(DragC)),
        ("point_mass_order", C.c_int32 * 8),
    ]


class Details(C.Structure):
    _fields_ = [
        ("step_ns", C.c_int64),
        ("error", C.c_double),
        ("attempts", C.c_int32),
        ("_pad", C.c_int32),
        ("n_steps", C.c_int64),
        ("n_rejected", C.c_int64),
        ("n_rhs", C.c_int64),
    ]


class TrajSink(C.Structure):
    _fields_ = [
        ("capacity", C.c_int64),
        ("epoch_ns", C.c_void_p),
        ("state", C.c_void_p),
        ("count", C.c_void_p),
    ]


class EventC(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("trigger", C.c_int32),
        ("value", C.c_double),
        ("crossings", C.c_void_p),
    ]


# ---- orbit determination (SURVEY.md §8 (f)-2): mirrors of nyxb_ground_station / nyxb_od_config / nyxb_tracking_arc / nyxb_od_outputs /
# nyxb_od_records / nyxb_smooth_outputs / nyxb_predict_outputs / nyxb_bls_config / nyxb_bls_outputs
MSR_RANGE, MSR_DOPPLER = 0, 1
MSR_AZIMUTH, MSR_ELEVATION = 2, 3  # degrees; ground stations with angles (nyxb_aer_station)
MSR_X, MSR_Y, MSR_Z = 6, 7, 8      # position fixes (nyxb_position_device)
KF_REFERENCE_UPDATE, KF_DEVIATION_TRACKING = 0, 1
MSRF_PROCESSED, MSRF_REJECTED, MSRF_NOT_VISIBLE, MSRF_ABSENT = 1, 2, 4, 8
BLS_NORMAL_EQUATIONS, BLS_LEVENBERG_MARQUARDT = 0, 1
ERR_TOO_FEW_MEASUREMENTS, ERR_SINGULAR_INFORMATION, ERR_INVALID_MEASUREMENT = 6, 7, 8
ERR_SINGULAR_STM, ERR_RECORDS_TRUNCATED = 9, 10
ERR_TX_NO_DATA, ERR_NO_RANGE = 11, 12   # interlink: the transmitter's recording misses the epoch; a Doppler row without a range
OD_TAG_TIME_UPDATE = -1   # estimate-record tags: NYXB_OD_TAG(k, w, rejected, msr_size) = ((k*2 + w)*2 + rejected)*2 + msr_size - 1


def od_tag(k, window, rejected, msr_size):
    return ((int(k) * 2 + int(window)) * 2 + int(rejected)) * 2 + int(msr_size) - 1


def od_pos_tag(k, window, rejected, msr_size):
    """NYXB_OD_POS_TAG: the record tag of the position-fix filter (window 0..2, msr_size 1..3)."""
    return ((int(k) * 4 + int(window)) * 2 + int(rejected)) * 4 + int(msr_size) - 1


def od_pos_tag_fields(tag):
    return tag >> 5, (tag >> 3) & 3, (tag >> 2) & 1, (tag & 3) + 1


def od_tag_fields(tag):
    """(measurement index, window, rejected, msr_size) of measurement-update tags (arrays or ints)."""
    return tag >> 3, (tag >> 2) & 1, (tag >> 1) & 1, (tag & 1) + 1


class GroundStationC(C.Structure):
    _fields_ = [
        ("pos_fixed_km", C.c_double * 3),
        ("up_fixed", C.c_double * 3),
        ("elevation_mask_deg", C.c_double),
        ("rot", Rotation),
        ("body", C.c_int32),
        ("n_types", C.c_int32),
        ("types", C.c_int32 * 2),
        ("_pad", C.c_int32),
        ("noise_var", C.c_double * 2),
        ("bias", C.c_double * 2),
        ("body_radius_km", C.c_double),
    ]


class AerStationC(C.Structure):
    _fields_ = [
        ("pos_fixed_km", C.c_double * 3),
        ("up_fixed", C.c_double * 3),
        ("north_fixed", C.c_double * 3),
        ("east_fixed", C.c_double * 3),
        ("elevation_mask_deg", C.c_double),
        ("rot", Rotation),
        ("body", C.c_int32),
        ("n_types", C.c_int32),
        ("types", C.c_int32 * 4),
        ("noise_var", C.c_double * 4),
        ("bias", C.c_double * 4),
        ("body_radius_km", C.c_double),
    ]


class InterlinkTxC(C.Structure):
    _fields_ = [
        ("tx", C.c_int32),
        ("n_types", C.c_int32),
        ("types", C.c_int32 * 2),
        ("noise_var", C.c_double * 2),
        ("bias", C.c_double * 2),
        ("body_radius_km", C.c_double),
    ]


class PositionDeviceC(C.Structure):
    _fields_ = [
        ("n_types", C.c_int32),
        ("types", C.c_int32 * 3),
        ("noise_var", C.c_double * 3),
        ("bias", C.c_double * 3),
    ]


class PositionArcC(C.Structure):
    _fields_ = [
        ("n_msr", C.c_int64),
        ("epoch_ns", C.c_void_p),
        ("tracker", C.c_void_p),
        ("obs", C.c_void_p),
    ]


class OdConfigC(C.Structure):
    _fields_ = [
        ("variant", C.c_int32),
        ("msr_size", C.c_int32),
        ("reject_num_sigmas", C.c_double),
        ("max_step_ns", C.c_int64),
        ("epoch_precision_ns", C.c_int64),
        ("snc_enabled", C.c_int32),
        ("snc_frame", C.c_int32),
        ("snc_diag", C.c_double * 3),
        ("snc_disable_time_ns", C.c_int64),
    ]


class TrackingArcC(C.Structure):
    _fields_ = [
        ("n_msr", C.c_int64),
        ("epoch_ns", C.c_void_p),
        ("tracker", C.c_void_p),
        ("obs", C.c_void_p),
    ]


class OdOutputsC(C.Structure):
    _fields_ = [
        ("state_soa", C.c_void_p),
        ("epoch_ns", C.c_void_p),
        ("covar_soa", C.c_void_p),
        ("state_dev_soa", C.c_void_p),
        ("resid_ratio", C.c_void_p),
        ("prefit", C.c_void_p),
        ("postfit", C.c_void_p),
        ("msr_flags", C.c_void_p),
        ("est_state", C.c_void_p),
        ("est_covar_diag", C.c_void_p),
        ("details", C.c_void_p),
        ("status", C.c_void_p),
    ]


class PredictOutputsC(C.Structure):
    _fields_ = [
        ("state_soa", C.c_void_p),
        ("epoch_ns", C.c_void_p),
        ("covar_soa", C.c_void_p),
        ("state_dev_soa", C.c_void_p),
        ("details", C.c_void_p),
        ("status", C.c_void_p),
        ("capacity", C.c_int64),
        ("rec_state", C.c_void_p),
        ("rec_covar", C.c_void_p),
        ("rec_count", C.c_void_p),
    ]


class OdRecordsC(C.Structure):
    _fields_ = [
        ("capacity", C.c_int64),
        ("epoch_ns", C.c_void_p),
        ("tag", C.c_void_p),
        ("nominal", C.c_void_p),
        ("deviation", C.c_void_p),
        ("covar", C.c_void_p),
        ("stm", C.c_void_p),
        ("count", C.c_void_p),
    ]


class SmoothOutputsC(C.Structure):
    _fields_ = [
        ("state", C.c_void_p),
        ("deviation", C.c_void_p),
        ("covar", C.c_void_p),
        ("fs_ratio", C.c_void_p),
        ("postfit", C.c_void_p),
        ("status", C.c_void_p),
    ]


class BlsConfigC(C.Structure):
    _fields_ = [
        ("solver", C.c_int32),
        ("max_iterations", C.c_int32),
        ("tolerance_pos_km", C.c_double),
        ("max_step_ns", C.c_int64),
        ("epoch_precision_ns", C.c_int64),
        ("lm_lambda_init", C.c_double),
        ("lm_lambda_decrease", C.c_double),
        ("lm_lambda_increase", C.c_double),
        ("lm_lambda_min", C.c_double),
        ("lm_lambda_max", C.c_double),
        ("lm_use_diag_scaling", C.c_int32),
        ("_pad", C.c_int32),
    ]


class BlsOutputsC(C.Structure):
    _fields_ = [
        ("state_soa", C.c_void_p),
        ("epoch_ns", C.c_void_p),
        ("covar_soa", C.c_void_p),
        ("iterations", C.c_void_p),
        ("final_rms", C.c_void_p),
        ("final_corr_pos_km", C.c_void_p),
        ("converged", C.c_void_p),
        ("details", C.c_void_p),
        ("status", C.c_void_p),
    ]


class TgtVariableC(C.Structure):
    _fields_ = [
        ("component", C.c_int32),
        ("_pad", C.c_int32),
        ("perturbation", C.c_double),
        ("init_guess", C.c_double),
        ("max_step", C.c_double),
        ("max_value", C.c_double),
        ("min_value", C.c_double),
    ]


class TgtObjectiveC(C.Structure):
    _fields_ = [
        ("parameter", C.c_int32),
        ("_pad", C.c_int32),
        ("desired", C.c_double),
        ("tolerance", C.c_double),
        ("multiplicative_factor", C.c_double),
        ("additive_factor", C.c_double),
    ]


class TargetConfigC(C.Structure):
    _fields_ = [
        ("n_vars", C.c_int32),
        ("n_objs", C.c_int32),
        ("correction_frame", C.c_int32),
        ("iterations", C.c_int32),
        ("vars", TgtVariableC * 6),
        ("objs", TgtObjectiveC * 6),
    ]


DETAILS_DTYPE = np.dtype(
    [
        ("step_ns", "<i8"),
        ("error", "<f8"),
        ("attempts", "<i4"),
        ("_pad", "<i4"),
        ("n_steps", "<i8"),
        ("n_rejected", "<i8"),
        ("n_rhs", "<i8"),
    ]
)
assert DETAILS_DTYPE.itemsize == C.sizeof(Details) == 48


def as_double_p(a: np.ndarray):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_double_p)


def as_int64_p(a: np.ndarray):
    assert a.dtype == np.int64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_int64_p)


def as_int32_p(a: np.ndarray):
    assert a.dtype == np.int32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_int32_p)


# --------------------------------------------------------------------------- library loading
_PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = _PKG_DIR / "csrc" / "libnyxb.so"
_lib = None


class NyxbLibraryMissing(RuntimeError):
    """Raised when the CUDA extension is absent: the product has NO CPU fallback."""


def _declare(lib):
    vp = C.c_void_p
    lib.nyxb_engine_create.restype = vp
    lib.nyxb_engine_create.argtypes = [C.POINTER(DynamicsC), C.POINTER(IntegOpts), C.c_int32, C.c_int32]
    lib.nyxb_engine_destroy.restype = None
    lib.nyxb_engine_destroy.argtypes = [vp]
    batch_args = [vp, C.c_size_t, vp, vp, vp, C.c_int64, vp, vp, vp, vp, vp]
    lib.nyxb_propagate_batch.restype = C.c_int32
    lib.nyxb_propagate_batch.argtypes = batch_args
    lib.nyxb_propagate_batch_multi.restype = C.c_int32
    lib.nyxb_propagate_batch_multi.argtypes = [C.POINTER(vp), C.c_int32] + batch_args[1:]
    lib.nyxb_propagate_batch_dev.restype = C.c_int32
    lib.nyxb_propagate_batch_dev.argtypes = batch_args + [vp]
    lib.nyxb_propagate_batch_traj.restype = C.c_int32
    lib.nyxb_propagate_batch_traj.argtypes = batch_args + [C.POINTER(TrajSink)]
    lib.nyxb_propagate_batch_traj_dev.restype = C.c_int32
    lib.nyxb_propagate_batch_traj_dev.argtypes = batch_args + [C.POINTER(TrajSink), vp]
    lib.nyxb_traj_resample.restype = C.c_int32
    lib.nyxb_traj_resample.argtypes = [vp, C.c_size_t, C.POINTER(TrajSink), C.c_size_t, vp, vp, vp]
    lib.nyxb_traj_resample_dev.restype = C.c_int32
    lib.nyxb_traj_resample_dev.argtypes = [vp, C.c_size_t, C.POINTER(TrajSink), C.c_size_t, vp, vp, vp, vp]
    lib.nyxb_event_locate.restype = C.c_int32
    lib.nyxb_event_locate.argtypes = [vp, C.c_size_t, C.POINTER(TrajSink), C.c_int32, C.c_double, C.c_int64, vp, vp, vp, vp]
    lib.nyxb_event_locate_dev.restype = C.c_int32
    lib.nyxb_event_locate_dev.argtypes = [vp, C.c_size_t, C.POINTER(TrajSink), C.c_int32, C.c_double, C.c_int64, vp, vp, vp, vp, vp]
    lib.nyxb_propagate_batch_event.restype = C.c_int32
    lib.nyxb_propagate_batch_event.argtypes = batch_args + [C.POINTER(TrajSink), C.POINTER(EventC)]
    lib.nyxb_propagate_batch_stm.restype = C.c_int32
    lib.nyxb_propagate_batch_stm.argtypes = [vp, C.c_size_t, vp, vp, vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp]
    lib.nyxb_od_ekf_batch.restype = C.c_int32
    lib.nyxb_od_ekf_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(GroundStationC), C.POINTER(TrackingArcC),
                                      C.c_size_t, vp, vp, vp, vp, C.POINTER(OdOutputsC)]
    lib.nyxb_od_ekf_record_batch.restype = C.c_int32
    lib.nyxb_od_ekf_record_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(GroundStationC), C.POINTER(TrackingArcC),
                                             C.c_size_t, vp, vp, vp, vp, C.POINTER(OdOutputsC), C.POINTER(OdRecordsC)]
    lib.nyxb_od_smooth_batch.restype = C.c_int32
    lib.nyxb_od_smooth_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(GroundStationC), C.POINTER(TrackingArcC),
                                         C.c_size_t, C.POINTER(OdRecordsC), vp, C.POINTER(SmoothOutputsC)]
    lib.nyxb_od_aer_batch.restype = C.c_int32
    lib.nyxb_od_aer_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(AerStationC), C.POINTER(TrackingArcC), C.c_size_t,
                                      vp, vp, vp, vp, C.POINTER(OdOutputsC), C.POINTER(OdRecordsC)]
    lib.nyxb_od_aer_smooth_batch.restype = C.c_int32
    lib.nyxb_od_aer_smooth_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(AerStationC), C.POINTER(TrackingArcC),
                                             C.c_size_t, C.POINTER(OdRecordsC), vp, C.POINTER(SmoothOutputsC)]
    lib.nyxb_od_interlink_batch.restype = C.c_int32
    lib.nyxb_od_interlink_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(InterlinkTxC), C.c_size_t, C.POINTER(TrajSink),
                                            C.POINTER(TrackingArcC), C.c_size_t, vp, vp, vp, vp, C.POINTER(OdOutputsC), C.POINTER(OdRecordsC)]
    lib.nyxb_od_interlink_smooth_batch.restype = C.c_int32
    lib.nyxb_od_interlink_smooth_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(InterlinkTxC), C.c_size_t,
                                                   C.POINTER(TrajSink), C.POINTER(TrackingArcC), C.c_size_t, C.POINTER(OdRecordsC), vp,
                                                   C.POINTER(SmoothOutputsC)]
    lib.nyxb_od_position_batch.restype = C.c_int32
    lib.nyxb_od_position_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(PositionDeviceC), C.POINTER(PositionArcC),
                                           C.c_size_t, vp, vp, vp, vp, C.POINTER(OdOutputsC), C.POINTER(OdRecordsC)]
    lib.nyxb_od_position_smooth_batch.restype = C.c_int32
    lib.nyxb_od_position_smooth_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_int32, C.POINTER(PositionDeviceC), C.POINTER(PositionArcC),
                                                  C.c_size_t, C.POINTER(OdRecordsC), vp, C.POINTER(SmoothOutputsC)]
    lib.nyxb_od_predict_batch.restype = C.c_int32
    lib.nyxb_od_predict_batch.argtypes = [vp, C.POINTER(OdConfigC), C.c_size_t, vp, vp, vp, vp, vp, vp, C.POINTER(PredictOutputsC)]
    lib.nyxb_od_bls_batch.restype = C.c_int32
    lib.nyxb_od_bls_batch.argtypes = [vp, C.POINTER(BlsConfigC), C.c_int32, C.POINTER(GroundStationC), C.POINTER(TrackingArcC),
                                      C.c_size_t, vp, vp, vp, C.POINTER(BlsOutputsC)]
    lib.nyxb_od_bls_evaluate_batch.restype = C.c_int32
    lib.nyxb_od_bls_evaluate_batch.argtypes = [vp, C.POINTER(BlsConfigC), C.c_int32, C.POINTER(GroundStationC), C.POINTER(TrackingArcC),
                                               C.c_size_t, vp, vp, vp, vp, vp]
    lib.nyxb_mvn_sample.restype = C.c_int32
    lib.nyxb_mvn_sample.argtypes = [C.c_int32, C.c_uint64, C.c_uint64, C.c_size_t, vp, vp, vp, vp, vp]
    lib.nyxb_mvn_sample_dev.restype = C.c_int32
    lib.nyxb_mvn_sample_dev.argtypes = [C.c_int32, C.c_uint64, C.c_uint64, C.c_size_t, vp, vp, vp, vp, vp, vp]
    lib.nyxb_reference_normals.restype = C.c_int32
    lib.nyxb_reference_normals.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_size_t, vp]
    lib.nyxb_pcg64mcg_u64.restype = C.c_int32
    lib.nyxb_pcg64mcg_u64.argtypes = [C.c_uint64, C.c_uint64, C.c_size_t, vp]
    lib.nyxb_ziggurat_tables.restype = C.c_int32
    lib.nyxb_ziggurat_tables.argtypes = [vp, vp]
    lib.nyxb_engine_set_lanes.restype = C.c_int32
    lib.nyxb_engine_set_lanes.argtypes = [vp, C.c_int32]
    lib.nyxb_engine_get_lanes.restype = C.c_int32
    lib.nyxb_engine_get_lanes.argtypes = [vp]
    lib.nyxb_engine_launch_count.restype = C.c_int64
    lib.nyxb_engine_launch_count.argtypes = [vp]
    lib.nyxb_engine_last_kernel_ms.restype = C.c_double
    lib.nyxb_engine_last_kernel_ms.argtypes = [vp]
    lib.nyxb_measure_fp64_tflops.restype = C.c_double
    lib.nyxb_measure_fp64_tflops.argtypes = [C.c_int32, C.c_int32]
    lib.nyxb_coop_table_dump.restype = C.c_int32
    lib.nyxb_coop_table_dump.argtypes = [C.POINTER(GravityFieldC), C.c_int32, c_int32_p, c_int32_p, vp, vp, vp, vp]
    lib.nyxb_tx_table_dump.restype = C.c_int32
    lib.nyxb_tx_table_dump.argtypes = [C.POINTER(GravityFieldC), C.c_int32, c_int32_p, c_int32_p, vp, vp, vp, vp]
    lib.nyxb_engine_set_kernel.restype = C.c_int32
    lib.nyxb_engine_set_kernel.argtypes = [vp, C.c_int32]
    lib.nyxb_engine_last_kernel.restype = C.c_int32
    lib.nyxb_engine_last_kernel.argtypes = [vp]
    lib.nyxb_engine_set_tx_positions.restype = C.c_int32
    lib.nyxb_engine_set_tx_positions.argtypes = [vp, C.c_int32]
    lib.nyxb_engine_set_tx_tuning.restype = C.c_int32
    lib.nyxb_engine_set_tx_tuning.argtypes = [vp, C.c_int32, C.c_int32]
    lib.nyxb_target_batch.restype = C.c_int32
    lib.nyxb_target_batch.argtypes = [vp, C.POINTER(TargetConfigC), C.c_size_t, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp]
    lib.nyxb_abi_version.restype = C.c_int32
    lib.nyxb_abi_version.argtypes = []
    lib.nyxb_last_error.restype = C.c_char_p
    lib.nyxb_last_error.argtypes = []
    return lib


EXPORTED_SYMBOLS = [
    "nyxb_engine_create",
    "nyxb_engine_destroy",
    "nyxb_propagate_batch",
    "nyxb_propagate_batch_multi",
    "nyxb_propagate_batch_dev",
    "nyxb_propagate_batch_traj",
    "nyxb_propagate_batch_traj_dev",
    "nyxb_traj_resample",
    "nyxb_traj_resample_dev",
    "nyxb_event_locate",
    "nyxb_event_locate_dev",
    "nyxb_propagate_batch_event",
    "nyxb_propagate_batch_stm",
    "nyxb_od_ekf_batch",
    "nyxb_od_ekf_record_batch",
    "nyxb_od_smooth_batch",
    "nyxb_od_position_batch",
    "nyxb_od_position_smooth_batch",
    "nyxb_od_aer_batch",
    "nyxb_od_aer_smooth_batch",
    "nyxb_od_predict_batch",
    "nyxb_od_bls_batch",
    "nyxb_od_bls_evaluate_batch",
    "nyxb_mvn_sample",
    "nyxb_mvn_sample_dev",
    "nyxb_reference_normals",
    "nyxb_pcg64mcg_u64",
    "nyxb_ziggurat_tables",
    "nyxb_engine_set_lanes",
    "nyxb_engine_get_lanes",
    "nyxb_engine_launch_count",
    "nyxb_engine_last_kernel_ms",
    "nyxb_measure_fp64_tflops",
    "nyxb_coop_table_dump",
    "nyxb_tx_table_dump",
    "nyxb_engine_set_kernel",
    "nyxb_engine_last_kernel",
    "nyxb_engine_set_tx_tuning",
    "nyxb_engine_set_tx_positions",
    "nyxb_abi_version",
    "nyxb_last_error",
    "nyxb_od_interlink_batch",
    "nyxb_od_interlink_smooth_batch",
    "nyxb_target_batch",
]


def load_library():
    """Load ``libnyxb.so`` (built in-tree by ``__graft_entry__.build()``); fail loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("NYXB_LIBRARY", LIB_PATH))
    if not path.exists():
        raise NyxbLibraryMissing(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nyx_b200 has no CPU fallback by design)"
        )
    _lib = _declare(C.CDLL(str(path)))
    if _lib.nyxb_abi_version() != NYXB_ABI_VERSION:
        raise NyxbLibraryMissing(f"{path} exports ABI {_lib.nyxb_abi_version()}, this package needs {NYXB_ABI_VERSION}: rebuild (make -C nyx_b200/csrc)")
    return _lib


def last_error() -> str:
    lib = load_library()
    msg = lib.nyxb_last_error()
    return msg.decode() if msg else ""
