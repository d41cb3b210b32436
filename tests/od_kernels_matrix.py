"""Inputs of the parity matrix of the three ensemble entry points that share the filter's kernels (tests/test_gpu_od_kernels_matrix.py)
and of its CPU companion (tests/test_od_kernels_matrix_inputs.py):

  predict   nyxb_od_predict_batch (KalmanODProcess::predict_until)            nyxb_k_od[_coop]<OdPredictJob>
  bls       nyxb_od_bls_batch / nyxb_od_bls_evaluate_batch (BatchLeastSquares) nyxb_k_od[_coop]<OdBlsJob>
  position  nyxb_od_position_batch + nyxb_od_position_smooth_batch            nyxb_k_od[_coop]<OdFilterJob<DevPosDevice, REC>>,
                                                                              nyxb_k_smooth<PosTrk>

Everything is built from tests/od_matrix.py: its four force-model configurations at fixed 45.5 s DP78, its truth orbits, its 13
initial estimates (dispersed states, per-filter Cr, masses and SRP areas, a covariance with position-velocity and velocity-Cr
correlations), its stations and its field shapes.

  predict   each run starts from one of the 13 estimates with its own start epoch (0, 30 s, 0, 7 s + 3 ns, in turn) and its own end:
            an exact multiple of the 60 s chunk, an end 17 s short of one (the last chunk overshoots), an end before the start (one
            chunk), and an end 1 ns short of a multiple from the staggered start.  "ekf": no process noise; "ckf": a nonzero deviation
            mapped through the STM and SNC in RIC.
  bls       tests/test_gpu_blse.py's _om_case for the 13 filters: noise-free range + Doppler from the three stations in turn, guesses
            at a tenth of the filters' dispersion around the truth in sunlight (24 min into the Earth arcs, 1 min into the lunar one), three iterations that never
            converge.  Normal equations everywhere;
            Levenberg-Marquardt on "srp".  evaluate() on the same guesses.
  position  X / Y / Z fixes (1 m) of the configuration's truth in its integration frame (Moon-centred for "lunar"), 60 s apart.  The
            schedule alternates an X, Y, Z device with one that carries Z and X only; one fix comes from an unknown device; filter 1
            misses the Y of fix 2 (a zero H row with R kept at msr_size 3) and filter 3 misses fix 5 altogether.  "m3": EKF at
            msr_size 3 with SNC in RIC; the two-type device is left out of the device list, so its fixes are unknown trackers (at
            msr_size 3 its empty third slot is SingularNoiseRk).  "m1": CKF at msr_size 1 with both devices.  Every estimate is
            recorded and smoothed.

Spans: "long" (configurations: 48 chunks / 4 measurements / 48 fixes) and "short" (field shapes and ensembles: 3 chunks / 3
measurements / 8 fixes), so that the degree-96 oracle runs stay bounded.

Ensembles spanning several blocks: RAGGED = 37 runs, copies of the 13 set 50 m apart: two 32-thread blocks of the per-thread kernels
(the second holding 5) and ten 4-warp CTAs of the warp kernels (the last holding one warp)."""
import functools
import re
from pathlib import Path

import numpy as np

import nyx_b200 as nb
from nyx_b200 import abi
from tests import od_matrix as om

S = om.S
CHUNK = 60 * S                       # KalmanODProcess.max_step: one predict chunk
FAMILIES = ("STRICT", "FAST-thread", "FAST-coop")
KINDS = ("predict", "bls", "position")
RAGGED = 37
EDGE_RUNS = (0, 3, 4, 31, 32, 36)
CSRC = Path(__file__).resolve().parent.parent / "nyx_b200" / "csrc"

# Field shapes of the warp kernels: tests/od_matrix.SHAPES (1, 2 and 3 columns per lane, order 0 and truncated orders, Luna 80x80) and
# the top of the range, where 96x96 is the only shape with four columns per lane.  The per-thread families run 96x96 and a truncation.
COOP_SHAPES = list(om.SHAPES) + [("lunar", 96, 96), ("lunar", 96, 95), ("lunar", 95, 95), ("lunar", 81, 81)]
THREAD_SHAPES = [("lunar", 96, 96), ("field", 21, 4)]
SHAPE_CASES = [("FAST-coop", *s) for s in COOP_SHAPES] + [(f, *s) for f in ("STRICT", "FAST-thread") for s in THREAD_SHAPES]

# floors of the bounds, for quantities the oracle's self-probes leave (nearly) unmoved: tests/od_matrix.FLOORS, and
#   P_*      covariance, per 3x3 block (rr, rv, vr, vv) and the Cr row and column, relative to the largest entry of that block
#   stm      recorded STMs, relative to the largest entry;  rms / eval_rms  relative;  corr_km  the last BLS correction, absolute
FLOORS = dict(om.FLOORS, P_rr=1e-13, P_rv=1e-13, P_vr=1e-13, P_vv=1e-13, P_cr=1e-13, stm=1e-13, rms=1e-13, eval_rms=1e-13, corr_km=1e-12)
BLOCKS = (("P_rr", slice(0, 3), slice(0, 3)), ("P_rv", slice(0, 3), slice(3, 6)), ("P_vr", slice(3, 6), slice(0, 3)),
          ("P_vv", slice(3, 6), slice(3, 6)))
# the smoother works on the GPU's own records (no propagation): the bounds of tests/test_gpu_position.py, tightened where the
# measured differences allow (state 1e-7 -> 1e-11 km, postfit 1e-9 -> 1e-11 km; the covariance stays at 1e-6, measured 3e-7)
SMOOTH_BOUNDS = {"sm_dr": 1e-11, "sm_P": 1e-6, "sm_postfit_km": 1e-11}


def per_thread_block():
    """Threads per block of the per-thread filter kernels (nyxb_od.cu)."""
    sizes = set(re.findall(r"const int block = (\d+);", (CSRC / "nyxb_od.cu").read_text()))
    assert len(sizes) == 1, sizes
    return int(sizes.pop())


def warps_per_cta():
    """Filters (warps) per CTA of the warp-cooperative kernels (nyxb_od_coop.cu)."""
    return int(re.search(r"#define ODC_WPB (\d+)", (CSRC / "nyxb_od_coop.cu").read_text()).group(1))


def smooth_block():
    return int(re.search(r"const int block = (\d+);", (CSRC / "nyxb_smooth.cu").read_text()).group(1))


def case_id(kind, config, degree, order, setting, span, n):
    return f"{kind}-{setting}-{config}-{degree}x{order}-{span}-n{n}"


# ---- inputs ------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def estimates(config, n=om.N_F):
    """(state[9][n], consts[4][n], covar0[81][n] column-major): om.filters(config) cycled, copies set 50 m apart."""
    st, cs, _, cov = om.filters(config)
    idx = np.arange(n) % om.N_F
    st, cs, cov = st[:, idx].copy(), cs[:, idx].copy(), cov[:, idx].copy()
    st[0] += 0.05 * (np.arange(n) // om.N_F)
    for a in (st, cs, cov):
        a.setflags(write=False)
    return st, cs, cov


def _strict_prop(config, degree, order, drop=None):
    return om.propagator(config, nb.MODE_STRICT, degree, order, drop)


@functools.lru_cache(maxsize=None)
def predict_inputs(config, setting, span, n, degree=21, order=None, drop=None):
    prop = _strict_prop(config, degree, order, drop)
    st, cs, cov = estimates(config, n)
    chunks = 48 if span == "long" else 3
    ep = np.array([(0, 30 * S, 0, 7 * S + 3)[i % 4] for i in range(n)], dtype=np.int64)
    end = ep + np.array([(chunks * CHUNK, chunks * CHUNK - 17 * S, -S, chunks * CHUNK - 1)[i % 4] for i in range(n)], dtype=np.int64)
    if setting == "ekf":
        odp = nb.KalmanODProcess(prop, om.EKF, None, {}, om.almanac(config))
        dev0 = np.zeros((9, n))
    else:
        odp = nb.KalmanODProcess(prop, om.CKF, None, {}, om.almanac(config))
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12, 2e-12, 3e-12], 7200 * S, om.RIC))
        rng = np.random.default_rng(81)
        dev0 = np.vstack([rng.normal(0.0, 0.1, (3, n)), rng.normal(0.0, 1e-4, (3, n)), rng.normal(0.0, 0.02, (1, n)), np.zeros((2, n))])
    cap = int(1 + ((np.maximum(end - ep, 1) + CHUNK - 1) // CHUNK).max())
    return dict(prop=prop, cfg=odp.config_c(), st=st, cs=cs, ep=ep, end=end, cov=cov, dev0=dev0, cap=cap)


# the truth's measurement the guesses start at: in sunlight, so that SRP and its Cr partial act on the estimate (the Earth orbit
# spends its first 22 min in the Earth's shadow, the lunar one its minutes 20 to 30 or so in the Moon's)
BLS_START = {"lunar": 0}


def _bls_schedule(n_msr):
    names = list(om.devices(-90.0))
    return [names[k % 3] for k in range(n_msr)]


@functools.lru_cache(maxsize=None)
def bls_inputs(config, setting, span, n, degree=21, order=None, drop=None):
    prop = _strict_prop(config, degree, order, drop)
    n_msr = 4 if span == "long" else 3
    epochs, tr, y0 = om.truth(config, "regular")
    k0 = BLS_START.get(config, 24)
    t0, x0 = epochs[k0], tr[k0]
    epochs, tr = epochs[k0 + 1: k0 + 1 + n_msr], tr[k0 + 1: k0 + 1 + n_msr]
    dev = om.devices(-90.0)
    names = list(dev)
    schedule = _bls_schedule(n_msr)
    obs = nb.simulate_tracking(epochs, np.repeat(tr[:, :, None], n, axis=2), dev, schedule, om.frame(config), om.almanac(config),
                               np.random.default_rng(5)).obs
    st, cs, _ = estimates(config, n)
    st = st.copy()
    st[:6] = x0[:6, None] + 0.1 * (st[:6] - y0[:6, None])        # 30 m / 3 cm/s: inside the STM product's reach
    solver = nb.BLSSolver.LevenbergMarquardt if setting == "lm" else nb.BLSSolver.NormalEquations
    b = nb.BatchLeastSquares(prop, dev, om.almanac(config), solver=solver, max_iterations=3, tolerance_pos_km=1e-12)
    st_c = (abi.GroundStationC * len(names))(*[dev[k].to_c(om.frame(config), om.almanac(config)) for k in names])
    tracker = np.array([names.index(t) for t in schedule], dtype=np.int32)
    return dict(prop=prop, b=b, cfg=b.config_c(), n_st=len(names), st_c=st_c, epochs=epochs, tracker=tracker, obs=obs, st=st, cs=cs,
                ep=np.full(n, t0, dtype=np.int64))


UNKNOWN_FIX, PARTIAL_FIX, ABSENT_FIX = 6, (2, 1, 1), (5, 3)     # fix; (fix, component, filter); (fix, filter)


def position_schedule(n_fix):
    return ["nobody" if k == UNKNOWN_FIX else ("gnss2" if k % 4 == 3 else "gnss") for k in range(n_fix)]


def position_devices(setting):
    g = nb.PositionDevice("gnss")
    for t in (nb.MeasurementType.X, nb.MeasurementType.Y, nb.MeasurementType.Z):
        g.with_noise(t, nb.StochasticNoise(1e-3))
    g2 = nb.PositionDevice("gnss2")
    for t in (nb.MeasurementType.Z, nb.MeasurementType.X):
        g2.with_noise(t, nb.StochasticNoise(2e-3))
    return {"gnss": g} if setting == "m3" else {"gnss": g, "gnss2": g2}


@functools.lru_cache(maxsize=None)
def position_inputs(config, setting, span, n, degree=21, order=None, drop=None):
    prop = _strict_prop(config, degree, order, drop)
    n_fix = om.N_MSR if span == "long" else 8
    epochs, tr, _ = om.truth(config, "regular")
    epochs, tr = epochs[:n_fix], tr[:n_fix]
    schedule = position_schedule(n_fix)
    sim = position_devices("m1")
    sim["nobody"] = sim["gnss"]
    obs = nb.simulate_position_fixes(epochs, np.repeat(tr[:, :, None], n, axis=2), sim, schedule, np.random.default_rng(83)).obs
    k, q, f = PARTIAL_FIX
    obs[k, q, np.arange(n) % om.N_F == f] = np.nan
    obs[ABSENT_FIX[0], :, np.arange(n) % om.N_F == ABSENT_FIX[1]] = np.nan
    obs.setflags(write=False)
    dev = position_devices(setting)
    if setting == "m3":
        odp = nb.KalmanODProcess(prop, om.EKF, None, dev, om.almanac(config), msr_size=3)
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12, 1e-12, 1e-12], 7200 * S, om.RIC))
    else:
        odp = nb.KalmanODProcess(prop, om.CKF, None, dev, om.almanac(config), msr_size=1)
    names, dev_c = odp.position_devices_c()
    tracker = np.array([names.index(t) if t in names else -1 for t in schedule], dtype=np.int32)
    st, cs, cov = estimates(config, n)
    return dict(prop=prop, odp=odp, cfg=odp.config_c(), M=odp.msr_size, names=names, dev_c=dev_c, epochs=epochs, tracker=tracker, obs=obs,
                st=st, cs=cs, ep=np.zeros(n, dtype=np.int64), cov=cov, cap=6 * n_fix + 2)


INPUTS = {"predict": predict_inputs, "bls": bls_inputs, "position": position_inputs}


# ---- the restatements --------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def restated(kind, config, setting, span, n, degree=21, order=None, runs=None, drop=None, probe=None):
    """Restatement of each run in `runs` (default all): tests/predict_oracle.py, tests/blse_oracle.py (estimate and evaluate) or
    tests/position_oracle.py with its estimate records.  probe: a self-probe of tests/od_matrix.py ("fma", "reassoc")."""
    from oracle import pyoracle  # noqa: F401  (builds the oracle)

    from tests import blse_oracle as bo
    from tests import position_oracle as po
    from tests import predict_oracle as pr
    from tests.blse_util import oracle_cfg

    x = INPUTS[kind](config, setting, span, n, degree, order, drop)
    prop = x["prop"]
    packed = prop.dynamics.pack(om.frame(config), om.almanac(config))
    oc = prop.opts.to_c(prop.method)
    out = []
    with om._probe(probe):
        for i in (range(n) if runs is None else runs):
            y9, c4, ep0 = x["st"][:, i].copy(), x["cs"][:, i].copy(), int(x["ep"][i])
            if kind == "predict":
                r = pr.predict_until(packed.c, oc, x["cfg"], y9, c4, ep0, x["cov"][:, i].reshape(9, 9).T.copy(), int(x["end"][i]),
                                     x["dev0"][:, i].copy())
            elif kind == "bls":
                args = (packed.c, oc, oracle_cfg(x["b"]), x["st_c"], x["epochs"], x["tracker"], np.ascontiguousarray(x["obs"][:, :, i]))
                r = bo.estimate(*args, y9, c4, ep0)
                r["eval_rms"], r["eval_status"] = bo.evaluate(*args, y9, c4, ep0)
            else:
                sink = []
                r = po.process_arc(packed.c, oc, x["cfg"], x["dev_c"], x["epochs"], x["tracker"], np.ascontiguousarray(x["obs"][:, :, i]),
                                   y9, c4, ep0, x["cov"][:, i].reshape(9, 9).T.copy(), sink=sink)
                r["records"] = sink
            out.append(r)
    return out


# ---- the GPU side --------------------------------------------------------------------------------------------------------
def run(kind, family, config, setting, span, n, degree=21, order=None, only=None):
    """One launch of the entry point on `family` for all n runs (only=i: run i alone), then the smoother for the position filter.
    Returns (dict of outputs, the kernel family that ran the entry point)."""
    x = INPUTS[kind](config, setting, span, n, degree, order)
    mode = nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST
    prop = om.propagator(config, mode, degree, order)
    eng = prop.engine(om.frame(config), om.almanac(config))
    eng.set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    sl = slice(None) if only is None else slice(only, only + 1)
    st, cs, ep = x["st"][:, sl], x["cs"][:, sl], x["ep"][sl]
    if kind == "predict":
        sol = eng.od_predict_batch(x["cfg"], st, cs, ep, x["end"][sl], x["cov"][:, sl], x["dev0"][:, sl], capacity=x["cap"])
        got = dict(status=sol.status, epoch=sol.final_epoch_ns, n_steps=sol.details["n_steps"], state=sol.final_state_soa, covar=sol.covar,
                   dev=sol.state_deviation, count=sol.rec_count, rec_state=sol.rec_state, rec_covar=sol.rec_covar, sol=sol,
                   kernel=eng.last_kernel())
    elif kind == "bls":
        args = (x["cfg"], x["n_st"], x["st_c"], x["epochs"], x["tracker"], x["obs"][:, :, sl])
        got = eng.od_bls_batch(*args, st, cs, ep)
        got["n_steps"] = got["details"]["n_steps"]
        kernel = eng.last_kernel()
        got["eval_rms"], got["eval_status"] = eng.od_bls_evaluate_batch(*args, st, cs, ep)
        assert eng.last_kernel() == kernel
        got["kernel"] = kernel
    else:
        obs = x["obs"][:, :, sl]
        sol = eng.od_position_batch(x["cfg"], len(x["names"]), x["dev_c"], x["epochs"], x["tracker"], obs, st, cs, ep, x["cov"][:, sl],
                                    estimates_capacity=x["cap"])
        got = dict(status=sol.status, epoch=sol.final_epoch_ns, n_steps=sol.details["n_steps"], state=sol.final_state_soa, covar=sol.covar,
                   dev=sol.state_deviation, flags=sol.msr_flags, prefit=sol.prefit, postfit=sol.postfit, ratio=sol.resid_ratio,
                   records=sol.records, kernel=eng.last_kernel())
        got["smooth"] = eng.od_position_smooth_batch(x["cfg"], len(x["names"]), x["dev_c"], x["tracker"], obs, sol.records, sol.status)
    return got, got["kernel"]


# ---- comparison --------------------------------------------------------------------------------------------------------
def cov_errors(a, b):
    """a, b: [..][9][9].  Per 3x3 block of the 6x6 and for the Cr row and column (rows 0..5 of column 6 and columns 0..5 of row 6):
    the largest |a - b| over the matrices, each relative to the largest entry of that block of its b (inf where that block of b is
    zero and a differs)."""
    a, b = np.asarray(a).reshape(-1, 9, 9), np.asarray(b).reshape(-1, 9, 9)
    parts = [(k, a[:, r, c].reshape(len(a), -1), b[:, r, c].reshape(len(b), -1)) for k, r, c in BLOCKS]
    parts.append(("P_cr", np.concatenate([a[:, :6, 6], a[:, 6, :6]], 1), np.concatenate([b[:, :6, 6], b[:, 6, :6]], 1)))
    out = {}
    for k, pa, pb in parts:
        d = np.abs(pa - pb).max(1)
        sc = np.abs(pb).max(1)
        out[k] = float(np.where(sc > 0, d / np.where(sc > 0, sc, 1.0), np.where(d > 0, np.inf, 0.0)).max(initial=0.0))
    return out


def _norm_max(a, b):
    return float(np.sqrt(((np.asarray(a) - np.asarray(b)) ** 2).sum(-1)).max(initial=0.0))


def _merge(e, more):
    for k, v in more.items():
        e[k] = max(e.get(k, 0.0), v)


def exact_mismatches(kind, got, refs, runs):
    """What must be equal: status, final epochs, step counts, record counts and epochs, msr_flags, BLS iterations and convergence,
    the Cr and mass entries of predicted states, and the NaN patterns of every per-measurement output.  Returns a list of mismatches."""
    bad = []
    for j, (i, r) in enumerate(zip(runs, refs)):
        def eq(name, a, b):
            if not np.array_equal(a, b):
                bad.append((i, name, a if np.ndim(a) == 0 else "arrays differ"))
        eq("status", got["status"][i], r["status"])
        eq("n_steps", got["n_steps"][i], r["n_steps"])
        if kind == "predict":
            eq("epoch", got["epoch"][i], r["epoch"])
            eq("count", got["count"][i], r["count"])
            eq("rec_epoch", got["sol"].record_epochs(i), r["rec_epoch"])
            K = int(r["count"])
            eq("rec_state[6:]", got["rec_state"][:K, 6:, i], r["rec_state"][:, 6:])
            if K < got["rec_state"].shape[0]:
                eq("NaN past count", np.isnan(got["rec_state"][K:, :, i]).all(), True)
        elif kind == "bls":
            eq("epoch", got["epoch"][i], r["epoch"])
            eq("iterations", got["iterations"][i], r["iterations"])
            eq("converged", bool(got["converged"][i]), r["converged"])
            eq("eval_status", got["eval_status"][i], r["eval_status"])
        else:
            eq("epoch", got["epoch"][i], r["epoch"])
            eq("flags", got["flags"][:, i], r["flags"])
            for f in ("prefit", "postfit", "ratio"):
                eq(f"NaN {f}", np.isnan(got[f][:, :, i]), np.isnan(r["resid_ratio" if f == "ratio" else f]))
            rec, sink = got["records"], r["records"]
            eq("record count", rec["count"][i], len(sink))
            L = min(int(rec["count"][i]), len(sink))
            eq("record tags", rec["tag"][:L, i], np.array([e["tag"] for e in sink[:L]], dtype=np.int64))
            eq("record epochs", rec["epoch"][:L, i], np.array([e["epoch"] for e in sink[:L]], dtype=np.int64))
    return bad


def errors(kind, got, refs, runs):
    """Per quantity, the largest difference over the runs (units: km, km/s; covariance blocks and STMs relative; RMS relative)."""
    e = {}
    for i, r in zip(runs, refs):
        if kind == "predict":
            K = int(r["count"])
            rs = np.vstack([got["rec_state"][:K, :, i], got["state"][:, i][None]])
            ws = np.vstack([r["rec_state"], r["state"][None]])
            _merge(e, dict(dr=_norm_max(rs[:, :3], ws[:, :3]), dv=_norm_max(rs[:, 3:6], ws[:, 3:6]),
                           state_dev_r=float(np.abs(got["dev"][:3, i] - r["state_dev"][:3]).max())))
            rc = got["rec_covar"][:K, :, i].reshape(K, 9, 9).transpose(0, 2, 1)
            _merge(e, cov_errors(np.concatenate([rc, got["covar"][i][None]]), np.concatenate([r["rec_covar"], r["covar"][None]])))
        elif kind == "bls":
            _merge(e, dict(dr=_norm_max(got["state"][:3, i], r["state"][:3]), dv=_norm_max(got["state"][3:6, i], r["state"][3:6]),
                           cr=abs(got["state"][6, i] - r["state"][6]), rms=abs(got["final_rms"][i] - r["final_rms"]) / r["final_rms"],
                           corr_km=abs(got["final_corr_pos_km"][i] - r["final_corr_pos_km"]),
                           eval_rms=abs(got["eval_rms"][i] - r["eval_rms"]) / r["eval_rms"]))
            _merge(e, cov_errors(got["covar"][i], r["covar"]))
        else:
            rec, sink = got["records"], r["records"]
            L = min(int(rec["count"][i]), len(sink))
            nom = np.vstack([rec["nominal"][:L, :, i], got["state"][:, i][None]])
            wnom = np.vstack([np.array([s["nominal"] for s in sink[:L]]).reshape(L, 9), r["state"][None]])
            dev = np.vstack([rec["deviation"][:L, :, i], got["dev"][:, i][None]])
            wdev = np.vstack([np.array([s["deviation"] for s in sink[:L]]).reshape(L, 9), r["state_dev"][None]])
            _merge(e, dict(dr=_norm_max(nom[:, :3], wnom[:, :3]), dv=_norm_max(nom[:, 3:6], wnom[:, 3:6]),
                           cr=float(np.abs(nom[:, 6] - wnom[:, 6]).max()), state_dev_r=float(np.abs(dev[:, :3] - wdev[:, :3]).max())))
            pc = np.concatenate([rec["covar"][:L, :, i].reshape(L, 9, 9).transpose(0, 2, 1), got["covar"][i][None]])
            wc = np.concatenate([np.array([s["covar"] for s in sink[:L]]).reshape(L, 9, 9), r["covar"][None]])
            _merge(e, cov_errors(pc, wc))
            if L:
                stm = rec["stm"][:L, :, i].reshape(L, 9, 9).transpose(0, 2, 1)
                wstm = np.array([s["stm"] for s in sink[:L]])
                _merge(e, dict(stm=float(np.abs(stm - wstm).max() / np.abs(wstm).max())))
            for f, rf in (("ratio", "resid_ratio"), ("prefit", "prefit"), ("postfit", "postfit")):
                key = f if f == "ratio" else f"{f}_km"
                _merge(e, {key: float(np.nanmax(np.abs(got[f][:, :, i] - r[rf]), initial=0.0))})
    return e


@functools.lru_cache(maxsize=None)
def spread(kind, config, setting, span, n, degree=21, order=None, runs=None):
    """The restatement against its own self-probes (FMA build of the C oracle; numpy products summed in reverse order)."""
    ref = restated(kind, config, setting, span, n, degree, order, runs)
    rr = tuple(range(n)) if runs is None else runs
    sp = {}
    for probe in ("fma", "reassoc"):
        pr = restated(kind, config, setting, span, n, degree, order, runs, probe=probe)
        _merge(sp, errors(kind, _as_got(kind, pr, rr, n), ref, rr))
    return sp


def bounds(kind, config, setting, span, n, degree=21, order=None, runs=None):
    return {k: max(om.SPREAD_FACTOR * v, FLOORS[k]) for k, v in spread(kind, config, setting, span, n, degree, order, runs).items()}


def _as_got(kind, refs, runs, n):
    """Restatement results laid out like run()'s outputs, so that errors() compares two restatements."""
    idx = {i: j for j, i in enumerate(runs)}
    pick = [refs[idx[i]] if i in idx else refs[0] for i in range(n)]
    st = np.stack([r["state"] for r in pick], axis=-1)
    g = dict(state=st, covar=np.stack([r["covar"] for r in pick]))
    if kind == "predict":
        K = max(int(r["count"]) for r in pick)
        rs, rc = np.full((K, 9, n), np.nan), np.full((K, 81, n), np.nan)
        for i, r in enumerate(pick):
            k = int(r["count"])
            rs[:k, :, i] = r["rec_state"]
            rc[:k, :, i] = r["rec_covar"].transpose(0, 2, 1).reshape(k, 81)
        g.update(dev=np.stack([r["state_dev"] for r in pick], axis=-1), rec_state=rs, rec_covar=rc)
    elif kind == "bls":
        for f in ("final_rms", "final_corr_pos_km", "eval_rms"):
            g[f] = np.array([r[f] for r in pick])
    else:
        L = max(len(r["records"]) for r in pick)
        rec = {k: np.full((L, 9, n), np.nan) for k in ("nominal", "deviation")}
        rec.update(covar=np.full((L, 81, n), np.nan), stm=np.full((L, 81, n), np.nan), count=np.array([len(r["records"]) for r in pick]))
        for i, r in enumerate(pick):
            for k, s in enumerate(r["records"]):
                rec["nominal"][k, :, i], rec["deviation"][k, :, i] = s["nominal"], s["deviation"]
                rec["covar"][k, :, i], rec["stm"][k, :, i] = s["covar"].T.reshape(81), s["stm"].T.reshape(81)
        g.update(dev=np.stack([r["state_dev"] for r in pick], axis=-1), records=rec)
        for f, rf in (("ratio", "resid_ratio"), ("prefit", "prefit"), ("postfit", "postfit")):
            g[f] = np.stack([r[rf] for r in pick], axis=-1)
    return g
