"""Every argument check of the STM and orbit-determination entry points of the C ABI, table-driven: each case breaks one argument of
an otherwise valid call and pins the return code and a fragment of nyxb_last_error().  Every call is rejected before any device
allocation or launch; an engine is needed only because the checks read its setup."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi

pytestmark = pytest.mark.gpu
S = 10**9
BAD, UNSUP = -1, -4     # NYXB_RC_BAD_ARG, NYXB_RC_UNSUPPORTED


def _p(x):
    return None if x is None else x.ctypes.data


def _ref(x):
    return None if x is None else C.byref(x)


class Args:
    """A valid call of every entry point: one filter, two measurements, one ground station (range and Doppler, msr_size 2) or one
    position device (X, Y, Z, msr_size 3), two estimate records (a time update, then measurement 0)."""

    def __init__(self, eng):
        n, m = 1, 2
        self.eng, self.n = eng, n
        self.state = np.zeros((9, n))
        self.state[0], self.state[4] = 7000.0, 7.5
        self.consts = np.array([[100.0], [0.0], [0.0], [0.0]])
        self.epoch0 = np.zeros(n, np.int64)
        self.end = np.full(n, 60 * S, np.int64)
        self.covar0 = np.eye(9).reshape(81, 1).copy()
        self.out_state, self.out_epoch = np.zeros((9, n)), np.zeros(n, np.int64)
        self.out_stm, self.out_covar, self.status = np.zeros((81, n)), np.zeros((81, n)), np.zeros(n, np.int32)
        self.out = abi.OdOutputsC(_p(self.out_state), _p(self.out_epoch), _p(self.out_covar), None, None, None, None, None, None, None,
                                  None, _p(self.status))
        self.cfg = abi.OdConfigC(variant=abi.KF_REFERENCE_UPDATE, msr_size=2, reject_num_sigmas=-1.0, max_step_ns=60 * S,
                                 epoch_precision_ns=1000)
        gs = abi.GroundStationC()
        gs.body, gs.n_types = -1, 2          # NYXB_CENTRAL_BODY
        gs.types[0], gs.types[1] = abi.MSR_RANGE, abi.MSR_DOPPLER
        gs.noise_var[0], gs.noise_var[1] = 1e-3, 1e-6
        self.stations, self.n_stations = (abi.GroundStationC * 1)(gs), 1
        self.msr_epoch, self.tracker = np.array([60 * S, 120 * S], np.int64), np.zeros(m, np.int32)
        self.obs, self.pobs = np.zeros((m, 2, n)), np.zeros((m, 3, n))
        self.arc = abi.TrackingArcC(m, _p(self.msr_epoch), _p(self.tracker), _p(self.obs))
        pd = abi.PositionDeviceC()
        pd.n_types = 3
        for q, t in enumerate((abi.MSR_X, abi.MSR_Y, abi.MSR_Z)):
            pd.types[q], pd.noise_var[q] = t, 1e-6
        self.devices, self.n_devices = (abi.PositionDeviceC * 1)(pd), 1
        self.parc = abi.PositionArcC(m, _p(self.msr_epoch), _p(self.tracker), _p(self.pobs))
        self.pcfg = abi.OdConfigC(variant=abi.KF_REFERENCE_UPDATE, msr_size=3, reject_num_sigmas=-1.0, max_step_ns=60 * S,
                                  epoch_precision_ns=1000)
        cap = 2
        self.r = {k: np.zeros((cap, w, n)) for k, w in (("nominal", 9), ("deviation", 9), ("covar", 81), ("stm", 81))}
        self.r["epoch"] = np.zeros((cap, n), np.int64)
        self.tag = np.array([[abi.OD_TAG_TIME_UPDATE], [abi.od_tag(0, 0, 0, 2)]], np.int64)
        self.ptag = np.array([[abi.OD_TAG_TIME_UPDATE], [abi.od_pos_tag(0, 0, 0, 3)]], np.int64)
        self.count = np.full(n, 2, np.int64)
        self.rec = self._records(self.tag)
        self.prec = self._records(self.ptag)
        self.fstatus = np.zeros(n, np.int32)
        self.sout = abi.SmoothOutputsC(None, None, None, None, None, _p(self.status))
        self.pout = abi.PredictOutputsC(_p(self.out_state), _p(self.out_epoch), _p(self.out_covar), None, None, _p(self.status), 0, None,
                                        None, None)
        self.bcfg = abi.BlsConfigC(solver=abi.BLS_NORMAL_EQUATIONS, max_iterations=10, tolerance_pos_km=1e-4, max_step_ns=30 * S,
                                   epoch_precision_ns=1000, lm_lambda_init=10.0, lm_lambda_decrease=10.0, lm_lambda_increase=10.0,
                                   lm_lambda_min=1e-12, lm_lambda_max=1e12, lm_use_diag_scaling=1)
        self.bout = abi.BlsOutputsC(None, None, None, None, None, None, None, None, _p(self.status))
        self.rms = np.zeros(n)

    def _records(self, tag):
        r = self.r
        return abi.OdRecordsC(r["epoch"].shape[0], _p(r["epoch"]), _p(tag), _p(r["nominal"]), _p(r["deviation"]), _p(r["covar"]),
                              _p(r["stm"]), _p(self.count))


def stm(lib, a):
    return lib.nyxb_propagate_batch_stm(a.eng, a.n, _p(a.state), _p(a.consts), _p(a.epoch0), 60 * S, None, None, _p(a.out_state),
                                        _p(a.out_epoch), _p(a.out_stm), None, _p(a.status))


def ekf(lib, a):
    return lib.nyxb_od_ekf_batch(a.eng, _ref(a.cfg), a.n_stations, a.stations, _ref(a.arc), a.n, _p(a.state), _p(a.consts), _p(a.epoch0),
                                 _p(a.covar0), _ref(a.out))


def ekf_rec(lib, a):
    return lib.nyxb_od_ekf_record_batch(a.eng, _ref(a.cfg), a.n_stations, a.stations, _ref(a.arc), a.n, _p(a.state), _p(a.consts),
                                        _p(a.epoch0), _p(a.covar0), _ref(a.out), _ref(a.rec))


def smooth(lib, a):
    return lib.nyxb_od_smooth_batch(a.eng, _ref(a.cfg), a.n_stations, a.stations, _ref(a.arc), a.n, _ref(a.rec), _p(a.fstatus),
                                    _ref(a.sout))


def pos(lib, a):
    return lib.nyxb_od_position_batch(a.eng, _ref(a.pcfg), a.n_devices, a.devices, _ref(a.parc), a.n, _p(a.state), _p(a.consts),
                                      _p(a.epoch0), _p(a.covar0), _ref(a.out), _ref(a.prec))


def pos_smooth(lib, a):
    return lib.nyxb_od_position_smooth_batch(a.eng, _ref(a.pcfg), a.n_devices, a.devices, _ref(a.parc), a.n, _ref(a.prec), _p(a.fstatus),
                                             _ref(a.sout))


def predict(lib, a):
    return lib.nyxb_od_predict_batch(a.eng, _ref(a.cfg), a.n, _p(a.state), _p(a.consts), _p(a.epoch0), _p(a.end), _p(a.covar0), None,
                                     _ref(a.pout))


def bls(lib, a):
    return lib.nyxb_od_bls_batch(a.eng, _ref(a.bcfg), a.n_stations, a.stations, _ref(a.arc), a.n, _p(a.state), _p(a.consts), _p(a.epoch0),
                                 _ref(a.bout))


def bls_eval(lib, a):
    return lib.nyxb_od_bls_evaluate_batch(a.eng, _ref(a.bcfg), a.n_stations, a.stations, _ref(a.arc), a.n, _p(a.state), _p(a.consts),
                                          _p(a.epoch0), _p(a.rms), _p(a.status))


def _set(path, value):
    """a mutation that sets a.<path> (dotted, an index in brackets for the first device) to value"""
    def f(a):
        *head, last = path.split(".")
        obj = a
        for h in head:
            obj = getattr(obj, h[:-3])[0] if h.endswith("[0]") else getattr(obj, h)
        setattr(obj, last, value)
    return f


def _drag(a):
    a.eng = a.drag


def _both(*fs):
    def f(a):
        for g in fs:
            g(a)
    return f


def _tag(arr, value):
    def f(a):
        getattr(a, arr)[1, 0] = value
    return f


NULLS = [_set("eng", None), _set("state", None), _set("consts", None), _set("epoch0", None)]
FILTER_NULLS = NULLS + [_set("covar0", None), _set("out", None), _set("out.state_soa", None), _set("out.epoch_ns", None),
                        _set("out.covar_soa", None), _set("out.status", None)]
BAD_REC = [("rec.capacity", -1), ("rec.count", None), ("rec.epoch_ns", None), ("rec.tag", None), ("rec.nominal", None),
           ("rec.deviation", None), ("rec.covar", None), ("rec.stm", None)]
BAD_PREC = [("p" + k, v) for k, v in BAD_REC]
STATION = [("stations[0].n_types", 0, BAD, b"bad ground station"), ("stations[0].n_types", 3, BAD, b"bad ground station"),
           ("stations[0].body", 0, BAD, b"bad ground station"), ("stations[0].body", -2, BAD, b"bad ground station")]
DEVICE = [("devices[0].n_types", 0, BAD, b"n_types must be 1 to 3"), ("devices[0].n_types", 4, BAD, b"n_types must be 1 to 3")]


def _cases():
    c = []

    def add(fn, name, mut, rc, msg):
        c.append(pytest.param(fn, mut, rc, msg, id=f"{fn.__name__}-{name}"))

    # nyxb_propagate_batch_stm
    for k, f in enumerate(NULLS + [_set("out_state", None), _set("out_epoch", None), _set("out_stm", None), _set("status", None)]):
        add(stm, f"null{k}", f, BAD, b"null argument")
    add(stm, "drag", _drag, UNSUP, b"PartialsUndefined")
    # the ground-station filter, without and with records
    for fn in (ekf, ekf_rec):
        for k, f in enumerate(FILTER_NULLS + [_set("cfg", None), _set("arc", None), _set("stations", None), _set("n_stations", -1)]):
            add(fn, f"null{k}", f, BAD, b"null argument")
        add(fn, "drag", _drag, UNSUP, b"PartialsUndefined")
        add(fn, "drag-before-msr_size", _both(_drag, _set("cfg.msr_size", 3)), UNSUP, b"PartialsUndefined")
        for v in (0, 3):
            add(fn, f"msr_size{v}", _set("cfg.msr_size", v), BAD, b"msr_size must be 1 or 2")
        add(fn, "variant", _set("cfg.variant", 2), BAD, b"bad filter variant")
        add(fn, "max_step", _set("cfg.max_step_ns", 0), BAD, b"StepSize")
        add(fn, "one-msr", _set("arc.n_msr", 1), BAD, b"TooFewMeasurements")
        add(fn, "few-before-arrays", _both(_set("arc.n_msr", 1), _set("arc.obs", None)), BAD, b"TooFewMeasurements")
        for f in ("epoch_ns", "tracker", "obs"):
            add(fn, f"arc-{f}", _set(f"arc.{f}", None), BAD, b"null tracking arc arrays")
        for k, (path, v, rc, msg) in enumerate(STATION):
            add(fn, f"station{k}", _set(path, v), rc, msg)
        add(fn, "msr-type", _set("stations[0].types", (C.c_int32 * 2)(abi.MSR_RANGE, abi.MSR_X)), UNSUP, b"unsupported measurement type")
        add(fn, "types-per-msr_size", _set("stations[0].n_types", 1), UNSUP, b"multiple of msr_size")
    add(ekf_rec, "null-rec", _set("rec", None), BAD, b"null argument")
    for k, (path, v) in enumerate(BAD_REC):
        add(ekf_rec, f"rec{k}", _set(path, v), BAD, b"bad estimate records")
    add(ekf_rec, "rec-before-drag", _both(_drag, _set("rec.count", None)), BAD, b"bad estimate records")
    # the ground-station smoother
    for k, f in enumerate([_set("eng", None), _set("cfg", None), _set("arc", None), _set("rec", None), _set("fstatus", None),
                           _set("sout", None), _set("sout.status", None), _set("stations", None), _set("n_stations", -1)]):
        add(smooth, f"null{k}", f, BAD, b"null argument")
    add(smooth, "msr_size", _set("cfg.msr_size", 3), BAD, b"msr_size must be 1 or 2")
    for k, (path, v) in enumerate(BAD_REC):
        add(smooth, f"rec{k}", _set(path, v), BAD, b"bad estimate records")
    add(smooth, "n_msr", _set("arc.n_msr", -1), BAD, b"null tracking arc arrays")
    for f in ("tracker", "obs"):
        add(smooth, f"arc-{f}", _set(f"arc.{f}", None), BAD, b"null tracking arc arrays")
    for k, (path, v, rc, msg) in enumerate(STATION):
        add(smooth, f"station{k}", _set(path, v), rc, msg)
    add(smooth, "rec-msr_size", _tag("tag", abi.od_tag(0, 0, 0, 1)), BAD, b"another msr_size")
    add(smooth, "rec-msr", _tag("tag", abi.od_tag(2, 0, 0, 2)), BAD, b"do not match this tracking arc")
    add(smooth, "rec-window", _tag("tag", abi.od_tag(0, 1, 0, 2)), BAD, b"do not match this tracking arc")
    add(smooth, "rec-window-m1", _both(_set("cfg.msr_size", 1), _set("stations[0].n_types", 1), _tag("tag", abi.od_tag(0, 1, 0, 1))), BAD,
        b"do not match this tracking arc")
    add(smooth, "rec-tracker", lambda a: a.tracker.__setitem__(0, 1), BAD, b"do not match this tracking arc")
    # the position-fix filter
    for k, f in enumerate(FILTER_NULLS + [_set("pcfg", None), _set("parc", None), _set("devices", None), _set("n_devices", -1)]):
        add(pos, f"null{k}", f, BAD, b"null argument")
    for k, (path, v) in enumerate(BAD_PREC):
        add(pos, f"rec{k}", _set(path, v), BAD, b"bad estimate records")
    for v in (0, 4):
        add(pos, f"msr_size{v}", _set("pcfg.msr_size", v), BAD, b"msr_size must be 1, 2 or 3")
    add(pos, "variant", _set("pcfg.variant", -1), BAD, b"bad filter variant")
    add(pos, "max_step", _set("pcfg.max_step_ns", -5), BAD, b"StepSize")
    add(pos, "one-msr", _set("parc.n_msr", 1), BAD, b"TooFewMeasurements")
    for f in ("epoch_ns", "tracker", "obs"):
        add(pos, f"arc-{f}", _set(f"parc.{f}", None), BAD, b"null tracking arc arrays")
    for k, (path, v, rc, msg) in enumerate(DEVICE):
        add(pos, f"device{k}", _set(path, v), rc, msg)
    add(pos, "type", _set("devices[0].types", (C.c_int32 * 3)(abi.MSR_X, abi.MSR_RANGE, abi.MSR_Z)), BAD, b"must be X, Y or Z")
    add(pos, "duplicate", _set("devices[0].types", (C.c_int32 * 3)(abi.MSR_X, abi.MSR_Y, abi.MSR_X)), BAD, b"duplicate")
    add(pos, "drag", _drag, UNSUP, b"PartialsUndefined")
    add(pos, "device-before-drag", _both(_drag, _set("devices[0].n_types", 0)), BAD, b"n_types must be 1 to 3")
    add(pos, "msr_size-before-drag", _both(_drag, _set("pcfg.msr_size", 0)), BAD, b"msr_size")
    # the position-fix smoother
    for k, f in enumerate([_set("eng", None), _set("pcfg", None), _set("parc", None), _set("prec", None), _set("fstatus", None),
                           _set("sout", None), _set("sout.status", None), _set("devices", None), _set("n_devices", -1)]):
        add(pos_smooth, f"null{k}", f, BAD, b"null argument")
    add(pos_smooth, "msr_size", _set("pcfg.msr_size", 4), BAD, b"msr_size must be 1, 2 or 3")
    for k, (path, v) in enumerate(BAD_PREC):
        add(pos_smooth, f"rec{k}", _set(path, v), BAD, b"bad estimate records")
    add(pos_smooth, "n_msr", _set("parc.n_msr", -1), BAD, b"null tracking arc arrays")
    for f in ("tracker", "obs"):
        add(pos_smooth, f"arc-{f}", _set(f"parc.{f}", None), BAD, b"null tracking arc arrays")
    for k, (path, v, rc, msg) in enumerate(DEVICE):
        add(pos_smooth, f"device{k}", _set(path, v), rc, msg)
    add(pos_smooth, "duplicate", _set("devices[0].types", (C.c_int32 * 3)(abi.MSR_Z, abi.MSR_Y, abi.MSR_Z)), BAD, b"duplicate")
    add(pos_smooth, "rec-msr_size", _tag("ptag", abi.od_pos_tag(0, 0, 0, 1)), BAD, b"another msr_size")
    add(pos_smooth, "rec-msr", _tag("ptag", abi.od_pos_tag(2, 0, 0, 3)), BAD, b"do not match this tracking arc")
    add(pos_smooth, "rec-window", _tag("ptag", abi.od_pos_tag(0, 1, 0, 3)), BAD, b"do not match this tracking arc")
    add(pos_smooth, "rec-window-m1", _both(_set("pcfg.msr_size", 1), _set("devices[0].n_types", 2), _tag("ptag", abi.od_pos_tag(0, 2, 0, 1))),
        BAD, b"do not match this tracking arc")
    add(pos_smooth, "rec-tracker", lambda a: a.tracker.__setitem__(0, -1), BAD, b"do not match this tracking arc")
    # covariance prediction
    for k, f in enumerate(NULLS + [_set("cfg", None), _set("end", None), _set("covar0", None), _set("pout", None),
                                   _set("pout.state_soa", None), _set("pout.epoch_ns", None), _set("pout.covar_soa", None),
                                   _set("pout.status", None)]):
        add(predict, f"null{k}", f, BAD, b"null argument")
    add(predict, "variant", _set("cfg.variant", 2), BAD, b"bad filter variant")
    add(predict, "variant-before-null", _both(_set("eng", None), _set("cfg.variant", 2)), BAD, b"bad filter variant")
    add(predict, "max_step", _set("cfg.max_step_ns", 0), BAD, b"StepSize")
    add(predict, "capacity", _set("pout.capacity", -1), BAD, b"negative record capacity")
    add(predict, "drag", _drag, UNSUP, b"PartialsUndefined")
    # batch least squares
    for fn in (bls, bls_eval):
        for k, f in enumerate(NULLS + [_set("bcfg", None), _set("arc", None), _set("stations", None), _set("n_stations", -1)]):
            add(fn, f"null{k}", f, BAD, b"null argument")
        add(fn, "max_step", _set("bcfg.max_step_ns", 0), BAD, b"max_step")
        add(fn, "n_msr", _set("arc.n_msr", -1), BAD, b"null tracking arc arrays")
        for f in ("epoch_ns", "tracker", "obs"):
            add(fn, f"arc-{f}", _set(f"arc.{f}", None), BAD, b"null tracking arc arrays")
        add(fn, "drag", _drag, UNSUP, b"PartialsUndefined")
        add(fn, "drag-before-station", _both(_drag, _set("stations[0].n_types", 0)), UNSUP, b"PartialsUndefined")
        for k, (path, v, rc, msg) in enumerate(STATION):
            add(fn, f"station{k}", _set(path, v), rc, msg)
        add(fn, "msr-type", _set("stations[0].types", (C.c_int32 * 2)(abi.MSR_DOPPLER, abi.MSR_Y)), UNSUP, b"unsupported measurement type")
        add(fn, "noise", _set("stations[0].noise_var", (C.c_double * 2)(1e-3, 0.0)), BAD, b"SingularNoiseRk")
        add(fn, "noise-nan", _set("stations[0].noise_var", (C.c_double * 2)(float("nan"), 1e-6)), BAD, b"SingularNoiseRk")
    add(bls, "null-out", _set("bout", None), BAD, b"null argument")
    add(bls, "null-status", _set("bout.status", None), BAD, b"null argument")
    add(bls_eval, "null-status", _set("status", None), BAD, b"null argument")
    add(bls, "solver", _set("bcfg.solver", 2), BAD, b"bad BLS solver")          # evaluate() reads no solver setting
    add(bls, "max_iterations", _set("bcfg.max_iterations", -1), BAD, b"max_iterations")
    add(bls, "solver-before-arc", _both(_set("bcfg.solver", 2), _set("arc.n_msr", -1)), BAD, b"bad BLS solver")
    add(bls, "lambda", _both(_set("bcfg.solver", abi.BLS_LEVENBERG_MARQUARDT), _set("bcfg.lm_lambda_min", 0.0)), BAD, b"lambda")
    add(bls, "lambda-nan", _both(_set("bcfg.solver", abi.BLS_LEVENBERG_MARQUARDT), _set("bcfg.lm_lambda_max", float("nan"))), BAD, b"lambda")
    return c


@pytest.fixture(scope="module")
def engines():
    frame = nb.EARTH_J2000
    two_body = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    drag = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.two_body(), nb.Drag(nb.AtmDensity.Constant(1e-12), nb.IAU_EARTH_FRAME))
    ok = nb.Propagator.default(two_body, mode=nb.MODE_STRICT).engine(frame, None)
    bad = nb.Propagator.default(drag, mode=nb.MODE_STRICT).engine(frame, None)
    yield ok, bad


@pytest.mark.parametrize("fn, mutate, rc, msg", _cases())
def test_rejected(engines, fn, mutate, rc, msg):
    lib = abi.load_library()
    ok, bad = engines
    a = Args(ok._h)
    a.drag = bad._h
    status = a.status
    mutate(a)
    launches = lib.nyxb_engine_launch_count(ok._h) + lib.nyxb_engine_launch_count(bad._h)
    assert fn(lib, a) == rc
    assert msg in lib.nyxb_last_error(), lib.nyxb_last_error()
    assert lib.nyxb_engine_launch_count(ok._h) + lib.nyxb_engine_launch_count(bad._h) == launches
    assert not status.any()
