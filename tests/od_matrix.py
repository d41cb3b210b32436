"""Inputs of the orbit-determination parity matrix (tests/test_gpu_od_matrix.py) and of its CPU companion
(tests/test_od_matrix_inputs.py): the filter ensemble, the two tracking arcs, the force-model configurations, the filter settings,
the STM ensemble, and the oracle results every kernel family is compared with.

Filters.  13 filters (three full blocks of the warp-cooperative kernel's 4 warps plus one partial block).  Each has its own dispersed
start state, its own initial covariance (position-velocity correlations, a Cr variance), dry / extra / propellant mass, SRP area and
Cr (2 is the upper clamp of the EKF state update), and its own noise realisation; blunders are injected into chosen filters at
chosen measurements.

Arcs.  The filters step at a fixed 45.5 s (DP78) under the 60 s max_step of KalmanODProcess, and the measurements are 60 s apart, so
every interval ends on a short step.
  regular  48 range + Doppler measurements over the three DSN stations, 10 per station in turn.  Goldstone's mask is raised to 20 deg
           in the filter, so its block is NOT_VISIBLE; one measurement of one filter is absent; the blunders are 50 sigma in range.
  edge     the arc of test_gpu_stm_od.test_filter_edge_cases_match_oracle: 150 s cadence (gaps longer than max_step), two
           measurements at the same epoch, an unknown tracker, a station whose mask hides every pass, a missing Doppler.

Configurations: "field" (JGM-3), "third_body" (+ Moon / Sun point masses), "srp" (+ SRP with Cr estimated, Earth and Moon shadows;
the orbit crosses penumbra and umbra during the arc), "lunar" (Moon-centred: lunar field + Earth / Sun point masses + SRP, Earth
stations; BASELINE configs[4] in small).

Field shapes where the code paths switch.  The warp-cooperative filter deals the columns m = 0..min(M, N) of the Legendre triangle
to 32 lanes (nyxb_api.cu, nyxb_od_ekf_batch) and builds its z^j / rho^j power table in ceil((N + 1) / 32) passes: one column per
lane and one pass up to N = 31, two for N = 32..63, three for N = 64..95 and four at N = 96 (coop_columns_per_lane below restates
the deal).  Only the full 96x96 field gives a lane four columns (ODC_KMAX); 96x95 has 96 columns, three per lane, with four passes.
Above the fixtures' top degrees (JGM-3 70, Luna 80) `gravity` takes the degree-96 fields of tests/high_degree.py, whose extra rows
are seeded draws; those shapes run in tests/test_gpu_high_degree.py."""
import functools

import numpy as np

import nyx_b200 as nb
from nyx_b200.frames import EARTH
from tests import fast_matrix as fm
from tests import high_degree as hd

S = 10**9
N_F = 13
N_MSR, CADENCE_S = 48, 60
N_EDGE, EDGE_CADENCE_S = 24, 150
METHOD = nb.IntegratorMethod.DormandPrince78
STEP_S = 45.5
CONFIGS = ("field", "third_body", "srp", "lunar")
CR_VALUES = (0.3, 0.9, 1.5, 2.0)
BLUNDERS = ((5, 1), (33, 6), (41, 11))          # (measurement, filter): +0.5 km in range
ABSENT = (17, 3)                                 # (measurement, filter): both types missing

# filter settings: (variant, msr_size, reject sigmas or None, SNC frame, SNC disable time in s)
EKF, CKF = nb.KalmanVariant.ReferenceUpdate, nb.KalmanVariant.DeviationTracking
RIC = nb.LocalFrame.RIC
VARIANTS = {
    "ekf": (EKF, 2, 3.0, RIC, 7200),
    "ekf_scalar_noreject": (EKF, 1, None, RIC, 50),    # 50 s: both SNC branches, see below
    "ckf_reject": (CKF, 2, 3.0, None, 7200),
    "ckf_scalar": (CKF, 1, None, None, 50),
}

# Short SNC disable time: the filter time-updates after every integration step, so the time since the previous update is 45.5 s or 14.5 s
# on a processed interval and 60 s after a measurement that was not visible (no update at its epoch).  A 50 s disable time therefore
# takes both branches of the SNC code (nyxb_od_arc.cuh od_covar_bar, snc.rs:188-196, 264-266).

# Field shapes: (config, degree, order).  Columns per lane of the warp-cooperative kernel: 1 up to degree 31, 2 for 32..63, 3 from 64.
SHAPES = [("field", 8, 0), ("field", 8, 1), ("field", 8, 8), ("field", 21, 4), ("field", 31, 31), ("field", 32, 32),
          ("field", 63, 63), ("field", 64, 64), ("field", 70, 70), ("lunar", 80, 80)]


def coop_columns_per_lane(degree, order):
    """Largest number of columns a lane gets from the host's longest-processing-time deal (nyxb_api.cu, nyxb_od_ekf_batch)."""
    mtop = min(order, degree)
    load, cnt = [0] * 32, [0] * 32
    for m in range(mtop + 1):
        best = min(range(32), key=lambda l: (load[l], cnt[l]))
        cnt[best] += 1
        load[best] += degree - max(m, 1) + 1 + 6
    return max(cnt)


def frame(config):
    return nb.MOON_J2000 if config == "lunar" else nb.EARTH_J2000


@functools.lru_cache(maxsize=None)
def almanac(config):
    if config == "lunar":
        return nb.Almanac.synthetic(nb.MOON_J2000, 0, 1.0, bodies=(EARTH, nb.SUN), pad_days=1.0)
    return fm.almanac()


def gravity(config, degree, order):
    if config == "lunar":
        if degree > 80:
            return nb.GravityField.new(hd.field_data("moon", degree, order))
        return nb.GravityField.new(nb.GravityFieldData.from_fixture("luna_jggrx_80x80", degree, order, nb.IAU_MOON_FRAME))
    if degree > 70:
        return nb.GravityField.new(hd.field_data("earth", degree, order))
    return fm.field(degree, order)


@functools.lru_cache(maxsize=None)
def dynamics(config, degree=21, order=None, drop=None):
    """`drop` removes one model ("field", "point_masses", "srp") to show that the configuration can see it."""
    order = degree if order is None else order
    alm = almanac(config)
    grav = [] if drop == "field" else [gravity(config, degree, order)]
    srp = [] if drop == "srp" else [nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)]
    pm = [] if drop == "point_masses" else [nb.PointMasses.new([EARTH, nb.SUN] if config == "lunar" else [nb.MOON, nb.SUN])]
    models, forces = {"field": (grav, []), "third_body": (pm + grav, []), "srp": (pm + grav, srp), "lunar": (pm + grav, srp)}[config]
    return nb.SpacecraftDynamics.from_models(nb.OrbitalDynamics.new(models), forces)


def propagator(config, mode, degree=21, order=None, drop=None, method=METHOD, step_s=STEP_S):
    return nb.Propagator.new(dynamics(config, degree, order, drop), method, nb.IntegratorOptions.with_fixed_step_s(step_s), mode=mode)


def devices(goldstone_mask_deg):
    rn, dn = nb.StochasticNoise(1e-2), nb.StochasticNoise(1e-5)          # 10 m, 1 cm/s
    return {"Madrid": nb.GroundStation.dss65_madrid(-90.0, rn, dn), "Canberra": nb.GroundStation.dss34_canberra(-90.0, rn, dn),
            "Goldstone": nb.GroundStation.dss13_goldstone(goldstone_mask_deg, rn, dn)}


def truth_orbit(config):
    if config == "lunar":
        return nb.Orbit.keplerian(1737.4 + 120.0, 0.002, 88.0, 20.0, 10.0, 0.0, 0, nb.MOON_J2000)
    return nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, nb.EARTH_J2000)


@functools.lru_cache(maxsize=None)
def truth(config, arc_kind):
    """(epochs[m], truth[m][6]) on the oracle (RK89 at 10 s, recorded) with the configuration's 21x21 dynamics."""
    from oracle import pyoracle

    m, cad = (N_MSR, CADENCE_S) if arc_kind == "regular" else (N_EDGE, EDGE_CADENCE_S)
    epochs = (np.arange(1, m + 1) * cad * S).astype(np.int64)
    sc = nb.Spacecraft(orbit=truth_orbit(config), mass=nb.Mass(500.0, 20.0, 50.0), srp=nb.SRPData(8.0, 1.3))
    st, cs, ep = nb.pack_spacecraft([sc])
    packed = dynamics(config).pack(frame(config), almanac(config))
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0).to_c(nb.IntegratorMethod.RungeKutta89)
    _, _, _, status, (t_ep, t_st, t_cnt) = pyoracle.propagate_batch(packed.c, topts, st, cs, ep, int(epochs[-1]), traj_capacity=m * cad // 10 + 2)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    assert np.array_equal(t_ep[idx, 0], epochs)
    return epochs, t_st[:, idx, 0].T.copy(), sc.to_vector()


@functools.lru_cache(maxsize=None)
def filters(config, seed=71):
    """(state[9][n], consts[4][n], epoch0[n], covar0[81][n] column-major): the 13 initial estimates."""
    _, _, y0 = truth(config, "regular")
    rng = np.random.default_rng(seed)
    n = N_F
    st = np.repeat(y0[:, None], n, axis=1)
    st[:3] += rng.normal(0.0, 0.3, (3, n))
    st[3:6] += rng.normal(0.0, 3e-4, (3, n))
    st[6] = np.array(CR_VALUES)[rng.permutation(n) % len(CR_VALUES)]
    st[8] = rng.uniform(10.0, 80.0, n)                       # propellant
    cs = np.vstack([rng.uniform(300.0, 700.0, n), rng.uniform(0.0, 40.0, n), np.where(np.arange(n) % 2 == 0, rng.uniform(12.0, 20.0, n), rng.uniform(30.0, 40.0, n)),
                    np.zeros(n)])
    ep = np.zeros(n, dtype=np.int64)
    cov = np.empty((81, n))
    sig = np.array([0.4, 0.4, 0.4, 4e-4, 4e-4, 4e-4, 0.2, 0.0, 0.0])
    for i in range(n):
        corr = np.eye(9)
        for a in range(3):                                   # position-velocity and velocity-Cr correlations
            corr[a, a + 3] = corr[a + 3, a] = rng.uniform(-0.6, 0.6)
            corr[a + 3, 6] = corr[6, a + 3] = rng.uniform(-0.3, 0.3)
        corr[:7, :7] = corr[:7, :7] @ corr[:7, :7].T        # keep it positive definite
        d = 1.0 / np.sqrt(np.diag(corr[:7, :7]))
        corr[:7, :7] *= np.outer(d, d)
        cov[:, i] = (corr * np.outer(sig, sig) * rng.uniform(0.5, 1.5)).T.reshape(81)
    for a in (st, cs, ep, cov):
        a.setflags(write=False)
    return st, cs, ep, cov


@functools.lru_cache(maxsize=None)
def arc(config, arc_kind, seed=72):
    """(epochs[m], tracker names[m], obs[m][2][n], filter devices)"""
    epochs, tr, _ = truth(config, arc_kind)
    m = len(epochs)
    names = ["Madrid", "Canberra", "Goldstone"]
    schedule = [names[(k // 10) % 3] for k in range(m)]
    rng = np.random.default_rng(seed)
    sim_dev = devices(-90.0)
    truth_n = np.repeat(tr[:, :, None], N_F, axis=2)
    obs = nb.simulate_tracking(epochs, truth_n, sim_dev, schedule, frame(config), almanac(config), rng).obs
    if arc_kind == "regular":
        for k, i in BLUNDERS:
            obs[k, 0, i] += 0.5
        obs[ABSENT[0], :, ABSENT[1]] = np.nan
        dev = devices(20.0)
    else:
        epochs = epochs.copy()
        epochs[5] = epochs[4]                                # same epoch, other station
        schedule[5] = "Canberra" if schedule[4] != "Canberra" else "Madrid"
        schedule[7] = "Atlantis"                             # not in the devices
        obs[5] = nb.simulate_tracking(epochs[5:6], truth_n[4:5], sim_dev, [schedule[5]], frame(config), almanac(config), None).obs[0]
        obs[9, 1, :] = np.nan                                # Doppler missing
        dev = devices(89.0)                                  # Goldstone never sees the spacecraft
    obs.setflags(write=False)
    return epochs, tuple(schedule), obs, dev


def od_process(prop, config, variant):
    var, msr_size, reject, snc_frame, disable_s = VARIANTS[variant]
    dev = arc(config, "regular")[3]
    odp = nb.KalmanODProcess(prop, var, nb.SigmaRejection(reject) if reject is not None else None, dev, almanac(config), msr_size=msr_size)
    return odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12, 1e-12, 1e-12], disable_s * S, snc_frame))


def od_inputs(config, variant, arc_kind, prop):
    """Everything nyxb_od_ekf_batch / process_arc take, for the 13 filters."""
    epochs, schedule, obs, dev = arc(config, arc_kind)
    odp = od_process(prop, config, variant)
    odp.devices = dict(dev)
    names, st_c = odp.stations_c(frame(config))
    tracker = np.array([names.index(t) if t in names else -1 for t in schedule], dtype=np.int32)
    st, cs, ep, cov = filters(config)
    if VARIANTS[variant][0] == CKF:                          # a linearised filter needs a start close to the truth
        y0 = truth(config, "regular")[2]
        st = st.copy()
        st[:6] = y0[:6, None] + 0.1 * (st[:6] - y0[:6, None])
    return odp, odp.config_c(), names, st_c, epochs, tracker, obs, st, cs, ep, cov


@functools.lru_cache(maxsize=None)
def oracle_filters(config, variant="ekf", arc_kind="regular", degree=21, order=None, drop=None, swap_areas=False, probe=None):
    """The oracle's results for the 13 filters, stacked like nyxb_od_outputs.  `probe`: "fma" runs the C oracle's FMA-contraction
    build, "reassoc" the numpy filter with every matrix product summed in reverse order (the spread of the oracle against itself)."""
    from oracle import pyoracle_od

    prop = propagator(config, nb.MODE_STRICT, degree, order, drop)
    odp, cfg, _, st_c, epochs, tracker, obs, st, cs, ep, cov = od_inputs(config, variant, arc_kind, prop)
    if swap_areas:
        cs = cs.copy()
        cs[2, : N_F - 1] = cs[2, : N_F - 1].reshape(-1, 2)[:, ::-1].reshape(-1)
    packed = prop.dynamics.pack(frame(config), almanac(config))
    oc = prop.opts.to_c(prop.method)
    res = []
    with _probe(probe):
        for i in range(N_F):
            y9 = st[:, i].copy()
            res.append(pyoracle_od.process_arc(packed.c, oc, cfg, st_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]), y9,
                                               cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy()))
    out = {k: np.stack([r[k] for r in res], axis=-1) for k in res[0] if k not in ("covar",)}
    out["covar"] = np.stack([r["covar"] for r in res])        # [n][9][9]
    return out


# ---- self-probes of the oracle -------------------------------------------------------------------------------------------
class _Reassoc(np.ndarray):
    """Every matmul with an operand of this type sums its inner index in reverse order."""

    def __array_ufunc__(self, ufunc, method, *inputs, **kw):
        args = [np.asarray(a) if isinstance(a, _Reassoc) else a for a in inputs]
        if ufunc is np.matmul and method == "__call__":
            a, b = args
            a2 = a[..., ::-1] if a.ndim > 1 else a[::-1]
            b2 = b[..., ::-1, :] if b.ndim > 1 else b[::-1]
            r = np.matmul(np.ascontiguousarray(a2), np.ascontiguousarray(b2))
        else:
            r = getattr(ufunc, method)(*args, **kw)
        return r.view(_Reassoc) if isinstance(r, np.ndarray) else r


class _probe:
    def __init__(self, kind):
        self.kind = kind

    def __enter__(self):
        from oracle import pyoracle

        self.saved = (pyoracle._LIB, pyoracle.Inst.get)
        if self.kind == "fma":
            pyoracle._LIB = _speed_lib_with_od()
        elif self.kind == "reassoc":
            get = pyoracle.Inst.get

            def get_reassoc(inst):
                y, *rest = get(inst)
                return (y.view(_Reassoc), *rest)

            pyoracle.Inst.get = get_reassoc
        return self

    def __exit__(self, *exc):
        from oracle import pyoracle

        pyoracle._LIB, pyoracle.Inst.get = self.saved


@functools.lru_cache(maxsize=None)
def _speed_lib_with_od():
    """The oracle's speed build (-ffp-contract=fast, FMA) with the argument types of every entry point of the parity build."""
    import ctypes as C

    from oracle import pyoracle

    par = pyoracle.lib()
    pyoracle.build()
    L = C.CDLL(str(pyoracle._DIR / "libnyx_oracle_speed.so"))
    for name in dir(par):
        if name.startswith("nyx_oracle_"):
            f = getattr(L, name)
            f.restype, f.argtypes = getattr(par, name).restype, getattr(par, name).argtypes
    return L


# ---- STM propagation -----------------------------------------------------------------------------------------------------
STM_N = 32
STM_END = 3600 * S
STM_CONFIGS = ("field", "third_body", "srp", "lunar")


@functools.lru_cache(maxsize=None)
def stm_ensemble(config):
    """32 trajectories of tests/fast_matrix.ensemble (per-trajectory epochs, masses, SRP areas, Cr), 24 LEO + 8 eccentric; for
    "lunar", the same dispersions around a 120 km lunar orbit."""
    st, cs, ep = fm.ensemble()
    idx = np.r_[0:24, 64:72]
    st, cs, ep = st[:, idx].copy(), cs[:, idx].copy(), ep[idx].copy()
    if config == "lunar":
        y0 = nb.Spacecraft(orbit=truth_orbit("lunar")).to_vector()
        st[:6] = y0[:6, None] + 0.01 * (st[:6] - st[:6].mean(axis=1, keepdims=True))
    st[6] = np.where(st[6] < 0.0, 0.3, np.minimum(st[6], 2.0))   # Cr in (0, 2]: with SRP, Cr = 0 gives a NaN STM (oracle and kernels)
    for a in (st, cs, ep):
        a.setflags(write=False)
    return st, cs, ep


def stm_step(method):
    return 10.0 if method == nb.IntegratorMethod.RungeKutta4 else STEP_S


@functools.lru_cache(maxsize=None)
def oracle_stm(config, method=METHOD, degree=21, order=None, end=STM_END, backward=False, probe=None):
    """The oracle's fixed-step STM result.  backward: from the oracle's forward state at `end` back to epoch 0."""
    from oracle import pyoracle

    prop = propagator(config, nb.MODE_STRICT, degree, order, method=method, step_s=stm_step(method))
    st, cs, ep = stm_ensemble(config)
    target = end
    if backward:
        st, ep = oracle_stm(config, method, degree, order, end)[:2]
        target = 0
    packed = prop.dynamics.pack(frame(config), almanac(config))
    with _probe(probe):
        out = pyoracle.propagate_batch_stm(packed.c, prop.opts.to_c(prop.method), st, cs, ep, target)
    for a in out[:3]:
        a.setflags(write=False)
    return out


STM_BLOCKS = (("rr", slice(0, 3), slice(0, 3)), ("rv", slice(0, 3), slice(3, 6)), ("vr", slice(3, 6), slice(0, 3)),
              ("vv", slice(3, 6), slice(3, 6)), ("cr", slice(0, 6), slice(6, 7)))


def stm_block_errors(a, b):
    """{block: max over trajectories of max|a - b| / max|b| within that trajectory's block}; a, b: [81][n] column-major."""
    A = a.T.reshape(-1, 9, 9).transpose(0, 2, 1)
    B = b.T.reshape(-1, 9, 9).transpose(0, 2, 1)
    out = {}
    for name, rs, cs in STM_BLOCKS:
        da = np.abs(A[:, rs, cs] - B[:, rs, cs]).reshape(len(A), -1).max(1)
        sc = np.abs(B[:, rs, cs]).reshape(len(B), -1).max(1)
        out[name] = float(np.where(sc > 0, da / np.where(sc > 0, sc, 1.0), np.where(da > 0, np.inf, 0.0)).max())
    return out


# ---- filter comparison ---------------------------------------------------------------------------------------------------
def filter_errors(got, ref):
    """Per quantity, the largest difference over the 13 filters and every measurement.  got: ODSolution-like dict or object with the
    attributes of nyx_b200.od.ODSolution; ref: oracle_filters(..).  Position-like entries in km, velocity-like in km/s, the
    covariance at correlation scale |dP_ij| / sqrt(P_ii P_jj), est_covar_diag relative."""
    g = got if isinstance(got, dict) else {
        "state": got.final_state_soa, "covar": got.covar, "state_dev": got.state_deviation, "resid_ratio": got.resid_ratio,
        "prefit": got.prefit, "postfit": got.postfit, "est_state": got.est_state, "est_covar_diag": got.est_covar_diag}
    e = {}
    e["dr"], e["dv"] = _dr_dv(g["state"], ref["state"])
    es_g, es_r = g["est_state"], ref["est_state"]                  # [m][9][n]
    e["est_dr"] = float(np.nanmax(np.sqrt(((es_g[:, :3] - es_r[:, :3]) ** 2).sum(1)), initial=0.0))
    e["est_dv"] = float(np.nanmax(np.sqrt(((es_g[:, 3:6] - es_r[:, 3:6]) ** 2).sum(1)), initial=0.0))
    e["cr"] = float(np.nanmax(np.abs(es_g[:, 6] - es_r[:, 6]), initial=0.0))
    P, Pr = g["covar"], ref["covar"]
    d = np.sqrt(np.abs(np.einsum("nii->ni", Pr)))
    scale = d[:, :, None] * d[:, None, :]
    live = scale > 0
    e["covar"] = float((np.abs(P - Pr)[live] / scale[live]).max())
    ecg, ecr = g["est_covar_diag"], ref["est_covar_diag"]
    live = np.isfinite(ecr) & (ecr > 0)
    e["est_covar"] = float((np.abs(ecg - ecr)[live] / ecr[live]).max(initial=0.0))
    e["state_dev_r"] = float(np.abs(g["state_dev"][:3] - ref["state_dev"][:3]).max())
    e["ratio"] = float(np.nanmax(np.abs(g["resid_ratio"] - ref["resid_ratio"]), initial=0.0))
    for q, unit in ((0, "km"), (1, "km_s")):
        e[f"prefit_{unit}"] = float(np.nanmax(np.abs(g["prefit"][:, q] - ref["prefit"][:, q]), initial=0.0))
        e[f"postfit_{unit}"] = float(np.nanmax(np.abs(g["postfit"][:, q] - ref["postfit"][:, q]), initial=0.0))
    return e


def _dr_dv(a, b):
    d = a - b
    return float(np.sqrt((d[:3] ** 2).sum(0)).max()), float(np.sqrt((d[3:6] ** 2).sum(0)).max())


# ---- bounds --------------------------------------------------------------------------------------------------------------
# Fixed step removes controller feedback: what separates two correct implementations is rounding, amplified by the filter's gain.
# The spread of a case is the largest difference between the oracle and its two self-probes ("fma", "reassoc"); the bound of every
# quantity is SPREAD_FACTOR x that spread, with a floor for quantities the probes leave (nearly) unmoved.
SPREAD_FACTOR = 10.0
FLOORS = {"dr": 1e-10, "dv": 1e-13, "est_dr": 1e-10, "est_dv": 1e-13, "cr": 1e-11, "covar": 1e-13, "est_covar": 1e-12,
          "state_dev_r": 1e-11, "ratio": 1e-9, "prefit_km": 1e-11, "postfit_km": 1e-11, "prefit_km_s": 1e-14, "postfit_km_s": 1e-14}
STM_FLOORS = {"dr": 1e-10, "dv": 1e-13, "rr": 1e-13, "rv": 1e-13, "vr": 1e-13, "vv": 1e-13, "cr": 1e-12}


@functools.lru_cache(maxsize=None)
def filter_spread(*case):
    ref = oracle_filters(*case)
    spread = {}
    for probe in ("fma", "reassoc"):
        for k, v in filter_errors(oracle_filters(*case, probe=probe), ref).items():
            spread[k] = max(spread.get(k, 0.0), v)
    return spread


def filter_bounds(*case):
    return {k: max(SPREAD_FACTOR * v, FLOORS[k]) for k, v in filter_spread(*case).items()}


def stm_errors(got, ref):
    e = dict(zip(("dr", "dv"), _dr_dv(got[0], ref[0])))
    e.update(stm_block_errors(got[2], ref[2]))
    return e


@functools.lru_cache(maxsize=None)
def stm_spread(*case):
    return stm_errors(oracle_stm(*case, probe="fma"), oracle_stm(*case))


def stm_bounds(*case):
    return {k: max(SPREAD_FACTOR * v, STM_FLOORS[k]) for k, v in stm_spread(*case).items()}
