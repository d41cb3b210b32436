"""Inputs of the parity matrix of angle tracking (nyxb_od_aer_batch + nyxb_od_aer_smooth_batch, tests/test_gpu_aer_matrix.py) and of
its CPU companion (tests/test_aer_matrix_inputs.py).

Everything is built from tests/od_matrix.py and tests/od_kernels_matrix.py: the four force-model configurations at fixed 45.5 s DP78,
their truth orbits, the 13 initial estimates (km.estimates), the field shapes, the ragged ensemble and the comparison helpers.

Settings
  "m2"  EKF at msr_size 2, sigma rejection at 3, SNC in RIC.  Madrid, Canberra and Goldstone carry [R, D, Az, El] (windows [R, D] and
        [Az, El]); Goldstone has a 20 deg mask in the filter, so its windows are NOT_VISIBLE on the Earth arcs.
  "m1"  CKF at msr_size 1, no rejection, started at a tenth of the dispersion (as om.od_inputs).  Madrid carries [Az, El], Canberra
        [El, R, Az], Goldstone [D, Az]: the output slot (the list position) is not the observation slot (the type value).

Arcs
  "long" / "short"  the truth of tests/od_matrix.py at 60 s (48 / 8 measurements), ten per station in turn, observed with every type
        and white noise of SIGMA.  An azimuth blunder of 50 sigma (BLUNDER: rejected under "m2"), one missing elevation
        (ABSENT_ANGLE), one measurement missing altogether (ABSENT_MSR) and one unknown tracker (UNKNOWN_MSR).  On "lunar" the Earth
        stations track the 120 km lunar orbiter in the Moon-centred frame, and the Moon hides it for part of the arc (Vallado's SIGHT in
        od_window_setup), which no mask does.
  "edges"  noise-free tracking of the "field" or "srp" truth by four stations placed from the truth itself (EDGE_TIMES):
        North     a pass that crosses due north between two measurements, measured on both sides of the cut; under "m2" one observation
                  straddles it (359.999 deg against a computed azimuth near 0.002 deg: a prefit near 360 deg, REJECTED)
        Zenith    a pass that peaks at about 89.9 deg (ZENITH_DEG)
        Mask      the Zenith site with its mask at the truth's elevation 240 s before the peak, measured just before and after the
                  pass crosses it (MASK_MARGIN_DEG below and above)
        Polar     the line of sight nearly along the integration frame's -Z: (dx^2 + dy^2) / |dr|^2 about 1e-11 (POLAR_CONDITION)
                  drives the azimuth row's 1 / (dx^2 + dy^2) and the cancellation in the elevation row's sqrt(r^2 - dz^2)
        The 13 filters start 1e-4 of the dispersion away from the truth, with its masses and areas, and weight angles at
        0.05 deg, so that every filter's nominal state sees the geometry above (tests/test_aer_matrix_inputs.py checks the margins on
        the restatement's own states).

Bounds: as tests/od_kernels_matrix.py (10 x the spread of the restatement against the C oracle's FMA build and reversed numpy sums), with
the residuals compared per unit of the slot's type: *_km (range), *_km_s (Doppler), *_deg (azimuth and elevation).  The FMA probe also
fuses the dot products of the window geometry (_fused_dots): a range of 384 000 km (Earth stations, lunar orbiter) has an ulp of 5.8e-11
km, and a contracting build moves it by that much, which the filter then carries into the states."""
import functools
import math

import numpy as np

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import aer_oracle as ao
from tests import od_kernels_matrix as km
from tests import od_matrix as om

S = om.S
SETTINGS = ("m2", "m1")
ALL = (MT.Range, MT.Doppler, MT.Azimuth, MT.Elevation)
AZ, EL = int(MT.Azimuth), int(MT.Elevation)
SIGMA = {MT.Range: 1e-2, MT.Doppler: 1e-5, MT.Azimuth: 1e-2, MT.Elevation: 1e-2}       # km, km/s, deg, deg
EDGE_SIGMA = {**SIGMA, MT.Azimuth: 5e-2, MT.Elevation: 5e-2}
POLAR_SIGMA = {**EDGE_SIGMA, MT.Elevation: 1e-6}     # the polar elevation decides its update: its row's rounding shows in the state
TYPES = {"m2": {"Madrid": ALL, "Canberra": ALL, "Goldstone": ALL},
         "m1": {"Madrid": (MT.Azimuth, MT.Elevation), "Canberra": (MT.Elevation, MT.Range, MT.Azimuth),
                "Goldstone": (MT.Doppler, MT.Azimuth)}}
MASKS = {"m2": {"Goldstone": 20.0}, "m1": {}}
BLUNDER = (33, 6)             # (measurement, filter): +0.5 deg in azimuth (Madrid)
ABSENT_ANGLE = (14, 2)        # (measurement, filter): elevation missing (Canberra)
ABSENT_MSR = (35, 9)          # (measurement, filter): every type missing
UNKNOWN_MSR = 27              # not a station of the filter

UNITS = {abi.MSR_RANGE: "km", abi.MSR_DOPPLER: "km_s", abi.MSR_AZIMUTH: "deg", abi.MSR_ELEVATION: "deg"}
# Floor of the angle residuals, in degrees.  A computed azimuth is fmod(atan2(..) * 180/pi, 360) + 360 when negative: CUDA's atan2 and
# asin are within 2 ulp (of a value below pi), the scaling adds one rounding and the +360 rounds to ulp(360) = 2^-44 deg = 5.7e-14 deg.
# Four ulp of 360 cover that sum for either angle (the elevation is below 90 deg, its ulps are smaller).
DEG_FLOOR = 4 * float(np.spacing(360.0))
FLOORS = dict(km.FLOORS, prefit_deg=DEG_FLOOR, postfit_deg=DEG_FLOOR)
# the smoother on the GPU's own records: od_kernels_matrix.SMOOTH_BOUNDS, and a postfit bound per unit.  The angle bound is 1e-10 deg:
# an H100 measured 2.2e-11 deg, on the "srp" edges arc on every family (the same smoothed states through the same window).
SMOOTH_BOUNDS = dict(km.SMOOTH_BOUNDS, sm_postfit_km_s=1e-14, sm_postfit_deg=1e-10)

# ---- the "edges" arc: epochs (s) of the geometry, on the configuration's truth
EDGE_TIMES = dict(north=1020, mask=1800, zenith=2040, polar=3540)
NORTH_AZ = 0.002               # truth azimuth (deg) at the straddling epoch
STRADDLE_OBS = 359.999
MASK_MARGIN_DEG = 1e-3         # the truth's elevation at the two mask measurements: the mask -/+ about this
ZENITH_DEG = 89.9
POLAR_CONDITION = 1e-11        # (dx^2 + dy^2) / |dr|^2 of the truth at the polar epoch


def case_id(config, degree, order, setting, span, n):
    return f"aer-{setting}-{config}-{degree}x{order}-{span}-n{n}"


# ---- truth and stations of the "edges" arc ---------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def truth_at(config, epochs):
    """The truth of tests/od_matrix.py (RK89 at a fixed 10 s on the oracle, 21x21) at arbitrary sorted epochs (ns): [len][9]."""
    from oracle import pyoracle

    sc = nb.Spacecraft(orbit=om.truth_orbit(config), mass=nb.Mass(500.0, 20.0, 50.0), srp=nb.SRPData(8.0, 1.3))
    st, cs, ep = nb.pack_spacecraft([sc])
    packed = om.dynamics(config).pack(om.frame(config), om.almanac(config))
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0).to_c(nb.IntegratorMethod.RungeKutta89)
    out = []
    for t in epochs:
        y, e, _, status = pyoracle.propagate_batch(packed.c, topts, st, cs, ep, int(t))
        assert status[0] == 0 and e[0] == t
        out.append(y[:, 0].copy())
        st, ep = y, e
    return np.array(out)


def truth_consts(config):
    sc = nb.Spacecraft(orbit=om.truth_orbit(config), mass=nb.Mass(500.0, 20.0, 50.0), srp=nb.SRPData(8.0, 1.3))
    return nb.pack_spacecraft([sc])[1][:, 0]


def _geodetic(p, frame=nb.IAU_EARTH_FRAME):
    """Body-fixed position -> (latitude deg, longitude deg, height km) on the frame's ellipsoid (inverse of GroundStation.body_fixed)."""
    a = frame.mean_equatorial_radius_km()
    b = frame.polar_radius_km
    e2 = 1.0 - (b * b) / (a * a)
    lon = math.atan2(p[1], p[0])
    rho = math.hypot(p[0], p[1])
    lat = math.atan2(p[2], rho * (1.0 - e2))
    for _ in range(50):
        nu = a / math.sqrt(1.0 - e2 * math.sin(lat) ** 2)
        h = rho / math.cos(lat) - nu
        lat = math.atan2(p[2], rho * (1.0 - e2 * nu / (nu + h)))
    nu = a / math.sqrt(1.0 - e2 * math.sin(lat) ** 2)
    return math.degrees(lat), math.degrees(lon), rho / math.cos(lat) - nu


def _station(name, lat, lon, h, mask=-90.0, types=ALL, sigma=EDGE_SIGMA):
    gs = nb.GroundStation(name, lat, lon, h, nb.IAU_EARTH_FRAME, mask, measurement_types=[],
                          stochastic_noises={MT.Range: nb.StochasticNoise(sigma[MT.Range]), MT.Doppler: nb.StochasticNoise(sigma[MT.Doppler])})
    for t in types:
        gs.with_msr_type(t, nb.StochasticNoise(sigma[t]))
    return gs


def _look(gs, t, y):
    """(azimuth, elevation, dr) of state y from station gs at t (ns), as the kernels compute them."""
    g = ao.geometry(gs.to_aer_c(nb.EARTH_J2000, None), None, int(t), y)
    return g["az"], g["elev"], np.array(g["dr"])


def _bf(t):
    return nb.od._rotation_matrix(nb.IAU_EARTH_FRAME.rotation, int(t))


def _brent(f, a, b):
    from scipy.optimize import brentq

    return brentq(f, a, b, xtol=1e-15, rtol=4 * np.finfo(float).eps, maxiter=200)


@functools.lru_cache(maxsize=None)
def edge_geometry(config):
    """The four stations (geodetic coordinates solved from the truth) and the epochs of the "edges" arc.
    Returns (stations {name: (lat, lon, h, mask)}, epochs (ns), schedule, the straddling measurement's index)."""
    T = {k: v * S for k, v in EDGE_TIMES.items()}
    # North: 8 deg south of the sub-satellite point at T["north"], its longitude solved for a truth azimuth of NORTH_AZ there
    y = truth_at(config, (T["north"],))[0]
    lat_s, lon_s, _ = _geodetic(_bf(T["north"]) @ y[:3])

    def az_north(lon):
        az = _look(_station("North", lat_s - 8.0, lon, 0.0), T["north"], y)[0]
        return (az + 180.0) % 360.0 - 180.0 - NORTH_AZ
    north = (lat_s - 8.0, _brent(az_north, lon_s - 5.0, lon_s + 5.0), 0.0, -90.0)
    # Zenith: on the sub-satellite meridian at T["zenith"], its latitude solved for a truth elevation of ZENITH_DEG there
    y = truth_at(config, (T["zenith"],))[0]
    lat_z, lon_z, _ = _geodetic(_bf(T["zenith"]) @ y[:3])
    dlat = _brent(lambda d: _look(_station("Zenith", lat_z + d, lon_z, 0.0), T["zenith"], y)[1] - ZENITH_DEG, 1e-6, 2.0)
    zenith = (lat_z + dlat, lon_z, 0.0, -90.0)
    # Mask: the zenith station's site, its mask at the truth's elevation at T["mask"], on the rising part of the same pass
    y = truth_at(config, (T["mask"],))[0]
    mask = (*zenith[:3], _look(_station("Mask", *zenith[:3]), T["mask"], y)[1])
    # Polar: on the ellipsoid below the spacecraft along -Z at T["polar"], offset horizontally for POLAR_CONDITION
    y = truth_at(config, (T["polar"],))[0]
    assert y[2] < 0.0
    fr = nb.IAU_EARTH_FRAME
    a, b = fr.mean_equatorial_radius_km(), fr.polar_radius_km
    z_s = -b * math.sqrt(1.0 - (y[0] ** 2 + y[1] ** 2) / a ** 2)
    eps = math.sqrt(POLAR_CONDITION) * abs(y[2] - z_s) / math.sqrt(2.0)
    polar = (*_geodetic(_bf(T["polar"]) @ np.array([y[0] - eps, y[1] - eps, z_s])), -90.0)
    stations = {"North": north, "Mask": mask, "Zenith": zenith, "Polar": polar}
    # epochs: North every 60 s around the straddle, Mask on either side of its crossing, Zenith at and after its peak, Polar last
    el_rate = (_look(_station("Mask", *mask[:3]), T["mask"] + S, truth_at(config, (T["mask"] + S,))[0])[1]
               - _look(_station("Mask", *mask[:3]), T["mask"] - S, truth_at(config, (T["mask"] - S,))[0])[1]) / 2.0
    dt_mask = int(round(MASK_MARGIN_DEG / abs(el_rate) * S))
    sched = [(T["north"] + d * S, "North") for d in (-180, -120, -60, 0, 60, 120)]
    sched += [(T["mask"] - dt_mask, "Mask"), (T["mask"] + dt_mask, "Mask")]
    sched += [(T["zenith"] - 60 * S, "Zenith"), (T["zenith"], "Zenith"), (T["zenith"] + 60 * S, "Zenith")]
    sched += [(T["polar"], "Polar")]
    sched.sort()
    epochs = tuple(int(t) for t, _ in sched)
    return stations, epochs, tuple(s for _, s in sched), epochs.index(T["north"])


EDGE_TYPES = {"m2": {s: ALL for s in ("North", "Mask", "Zenith", "Polar")},
              "m1": {"North": (MT.Azimuth, MT.Range), "Mask": (MT.Elevation, MT.Doppler), "Zenith": (MT.Elevation, MT.Azimuth, MT.Doppler),
                     "Polar": (MT.Elevation, MT.Azimuth, MT.Range)}}


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _process(prop, config, setting, devices):
    if setting == "m2":
        odp = nb.KalmanODProcess(prop, om.EKF, nb.SigmaRejection(3.0), devices, om.almanac(config), msr_size=2)
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-12, 1e-12, 1e-12], 7200 * S, om.RIC))
    else:
        odp = nb.KalmanODProcess(prop, om.CKF, None, devices, om.almanac(config), msr_size=1)
    return odp


def dsn(setting):
    out = {}
    for nm, ctor in (("Madrid", nb.GroundStation.dss65_madrid), ("Canberra", nb.GroundStation.dss34_canberra),
                     ("Goldstone", nb.GroundStation.dss13_goldstone)):
        gs = ctor(MASKS[setting].get(nm, -90.0), nb.StochasticNoise(SIGMA[MT.Range]), nb.StochasticNoise(SIGMA[MT.Doppler]))
        gs.measurement_types = []
        for t in TYPES[setting][nm]:
            gs.with_msr_type(t, nb.StochasticNoise(SIGMA[t]))
        out[nm] = gs
    return out


def schedule(n_msr):
    names = ["Madrid", "Canberra", "Goldstone"]
    return ["nobody" if k == UNKNOWN_MSR else names[(k // 10) % 3] for k in range(n_msr)]


def observe(config, epochs, truth, stations, sched, n, rng=None):
    """Range, Doppler, azimuth and elevation of the truth ([m][>=6]) from each scheduled station (all four types, whether it sees the
    spacecraft or not: the filter's mask and line-of-sight test decide), computed as the kernels do; white noise of SIGMA when `rng`
    is given.  obs [m][4][n]."""
    obs = np.empty((len(epochs), 4, n))
    for k, (t, nm) in enumerate(zip(epochs, sched)):
        g = ao.geometry(stations[nm].to_aer_c(om.frame(config), om.almanac(config)), packed(config).c, int(t), truth[k])
        for q in range(4):
            v = ao.computed(q, g)
            obs[k, q] = v + (rng.normal(0.0, SIGMA[ALL[q]], n) if rng is not None else 0.0)
    return obs


def _all_types_dsn():
    sim = dsn("m2")
    for gs in sim.values():
        gs.elevation_mask_deg = -90.0
    return list(sim.values())


@functools.lru_cache(maxsize=None)
def _regular_obs(config, n_msr, n):
    """Every type from every station (white noise of SIGMA), with the blunder and the missing observations; obs [m][4][n]."""
    epochs, tr, _ = om.truth(config, "regular")
    epochs, tr = epochs[:n_msr], tr[:n_msr]
    sim = dict(zip(("Madrid", "Canberra", "Goldstone"), _all_types_dsn()))
    sim["nobody"] = sim["Madrid"]
    obs = observe(config, epochs, tr, sim, schedule(n_msr), n, np.random.default_rng(91))
    f = np.arange(n) % om.N_F
    for (k, i), fill in ((BLUNDER, None), (ABSENT_ANGLE, EL), (ABSENT_MSR, slice(None))):
        if k >= n_msr:
            continue
        if fill is None:
            obs[k, AZ, f == i] += 0.5
        else:
            obs[k, fill, f == i] = np.nan
    obs.setflags(write=False)
    return epochs, obs


@functools.lru_cache(maxsize=None)
def _edge_obs(config, setting):
    stations, epochs, sched, k_s = edge_geometry(config)
    tr = truth_at(config, epochs)
    sim = {nm: _station(nm, *c[:3]) for nm, c in stations.items()}
    obs = observe(config, epochs, tr, sim, sched, om.N_F)
    if setting == "m2":
        obs[k_s, AZ, :] = STRADDLE_OBS
    obs.setflags(write=False)
    return obs


@functools.lru_cache(maxsize=None)
def inputs(config, setting, span, n, degree=21, order=None, drop=None):
    """Everything nyxb_od_aer_batch and the restatement take for n runs of one case."""
    prop = om.propagator(config, nb.MODE_STRICT, degree, order, drop)
    if span == "edges":
        assert n == om.N_F and config in ("field", "srp")
        stations, epochs, sched, _ = edge_geometry(config)
        devices = {nm: _station(nm, *c, types=EDGE_TYPES[setting][nm], sigma=POLAR_SIGMA if nm == "Polar" else EDGE_SIGMA)
                   for nm, c in stations.items()}
        epochs, obs = np.array(epochs, dtype=np.int64), _edge_obs(config, setting)
        st, _, cov = km.estimates(config, n)
        y0 = om.truth(config, "regular")[2]
        st = y0[:, None] + 1e-4 * (st - y0[:, None])
        cs = np.repeat(truth_consts(config)[:, None], n, axis=1)
    else:
        devices = dsn(setting)
        sched = schedule(om.N_MSR if span == "long" else 8)
        epochs, obs = _regular_obs(config, len(sched), n)
        st, cs, cov = km.estimates(config, n)
        if setting == "m1":                                     # a linearised filter needs a start close to the truth
            y0 = om.truth(config, "regular")[2]
            st = st.copy()
            st[:6] = y0[:6, None] + 0.1 * (st[:6] - y0[:6, None])
    odp = _process(prop, config, setting, devices)
    names, st_c = odp.aer_stations_c(om.frame(config))
    tracker = np.array([names.index(t) if t in names else -1 for t in sched], dtype=np.int32)
    types = [tuple(int(t) for t in devices[nm].measurement_types) for nm in names]
    for a in (st, cs):
        a.setflags(write=False)
    return dict(prop=prop, odp=odp, cfg=odp.config_c(), M=odp.msr_size, names=names, st_c=st_c, types=types, epochs=epochs, tracker=tracker,
                obs=obs, st=st, cs=cs, ep=np.zeros(n, dtype=np.int64), cov=cov,
                cap=int(epochs[-1] // int(om.STEP_S * S)) + 6 * len(epochs) + 2)


def slot_units(x):
    """[m][4]: the unit of the type at each output slot (the list position of the measurement's station), '' where there is none."""
    u = np.full((len(x["tracker"]), 4), "", dtype=object)
    for k, t in enumerate(x["tracker"]):
        if t >= 0:
            for q, typ in enumerate(x["types"][t]):
                u[k, q] = UNITS[typ]
    return u


_PACKED = {}


def packed(config, degree=21, order=None, drop=None):
    """The STRICT dynamics packed for the oracle (kept alive: the C struct points into its arrays)."""
    key = (config, degree, order, drop)
    if key not in _PACKED:
        _PACKED[key] = om.propagator(config, nb.MODE_STRICT, degree, order, drop).dynamics.pack(om.frame(config), om.almanac(config))
    return _PACKED[key]


# ---- the restatement ----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def restated(config, setting, span, n, degree=21, order=None, runs=None, drop=None, probe=None, sight=True):
    """tests/aer_oracle.process_arc of each run in `runs` (default all) with its estimate records.  probe: a self-probe of
    tests/od_matrix.py ("fma", "reassoc").  sight=False: the stations' line-of-sight test is switched off (body_radius_km = -1)."""
    from oracle import pyoracle  # noqa: F401  (builds the oracle)

    x = inputs(config, setting, span, n, degree, order, drop)
    prop = x["prop"]
    oc = prop.opts.to_c(prop.method)
    st_c = x["st_c"]
    if not sight:
        st_c = (abi.AerStationC * len(x["names"]))(*[st_c[j] for j in range(len(x["names"]))])
        for j in range(len(x["names"])):
            st_c[j].body_radius_km = -1.0
    dyn = packed(config, degree, order, drop)
    out = []
    with om._probe(probe), _fused_dots(probe == "fma"):
        for i in (range(n) if runs is None else runs):
            sink = []
            r = ao.process_arc(dyn.c, oc, x["cfg"], st_c, x["epochs"], x["tracker"], np.ascontiguousarray(x["obs"][:, :, i]),
                               x["st"][:, i].copy(), x["cs"][:, i].copy(), int(x["ep"][i]), x["cov"][:, i].reshape(9, 9).T.copy(), sink=sink)
            r["records"] = sink
            out.append(r)
    return out


def _fma(a, b, c):
    """a * b + c rounded once."""
    from fractions import Fraction

    return float(Fraction(a) * Fraction(b) + Fraction(c))


class _fused_dots:
    """The "fma" self-probe also fuses the window's dot products (range, range rate, elevation, azimuth components), as a contracting
    build of the kernels may: fma(a2, b2, fma(a1, b1, a0 * b0))."""

    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.saved = ao._dot
        if self.on:
            ao._dot = lambda a, b: _fma(a[2], b[2], _fma(a[1], b[1], a[0] * b[0]))
        return self

    def __exit__(self, *exc):
        ao._dot = self.saved


# ---- comparison ---------------------------------------------------------------------------------------------------------
def errors(got, refs, runs, units):
    """od_kernels_matrix.errors of the position kind (states, deviation, covariance blocks, STMs, ratio), with the residuals per unit."""
    e = km.errors("position", got, refs, runs)
    for k in ("prefit_km", "postfit_km"):
        e.pop(k)
    for i, r in zip(runs, refs):
        for f in ("prefit", "postfit"):
            d = np.abs(got[f][:, :, i] - r[f])
            for u in ("km", "km_s", "deg"):
                km._merge(e, {f"{f}_{u}": float(np.nanmax(d[units == u], initial=0.0))})
    return e


@functools.lru_cache(maxsize=None)
def spread(config, setting, span, n, degree=21, order=None, runs=None):
    ref = restated(config, setting, span, n, degree, order, runs)
    rr = tuple(range(n)) if runs is None else runs
    units = slot_units(inputs(config, setting, span, n, degree, order))
    sp = {}
    for probe in ("fma", "reassoc"):
        pr = restated(config, setting, span, n, degree, order, runs, probe=probe)
        km._merge(sp, errors(km._as_got("position", pr, rr, n), ref, rr, units))
    return sp


def bounds(config, setting, span, n, degree=21, order=None, runs=None):
    return {k: max(om.SPREAD_FACTOR * v, FLOORS[k]) for k, v in spread(config, setting, span, n, degree, order, runs).items()}


def nominals(x, ref, k):
    """The nominal states run i's windows of measurement k were computed from: the records of that measurement (written with the
    state before its update), else the state at its epoch (nothing was processed there)."""
    ys = [s["nominal"] for s in ref["records"] if s["tag"] >= 0 and abi.od_pos_tag_fields(s["tag"])[0] == k]
    return ys or [ref["est_state"][k]]


# ---- the GPU side --------------------------------------------------------------------------------------------------------
def run(family, config, setting, span, n, degree=21, order=None, only=None):
    """One launch of nyxb_od_aer_batch on `family` for all n runs (only=i: run i alone), then nyxb_od_aer_smooth_batch on its records.
    Returns (dict of outputs, the kernel family that ran the filter)."""
    x = inputs(config, setting, span, n, degree, order)
    mode = nb.MODE_STRICT if family == "STRICT" else nb.MODE_FAST
    eng = om.propagator(config, mode, degree, order).engine(om.frame(config), om.almanac(config))
    eng.set_kernel(nb.KERNEL_THREAD if family == "FAST-thread" else nb.KERNEL_AUTO)
    sl = slice(None) if only is None else slice(only, only + 1)
    obs = x["obs"][:, :, sl]
    sol = eng.od_aer_batch(x["cfg"], len(x["names"]), x["st_c"], x["epochs"], x["tracker"], obs, x["st"][:, sl], x["cs"][:, sl], x["ep"][sl],
                           x["cov"][:, sl], estimates_capacity=x["cap"])
    got = dict(status=sol.status, epoch=sol.final_epoch_ns, n_steps=sol.details["n_steps"], state=sol.final_state_soa, covar=sol.covar,
               dev=sol.state_deviation, flags=sol.msr_flags, prefit=sol.prefit, postfit=sol.postfit, ratio=sol.resid_ratio,
               records=sol.records, kernel=eng.last_kernel())
    got["smooth"] = eng.od_aer_smooth_batch(x["cfg"], len(x["names"]), x["st_c"], x["tracker"], obs, sol.records, sol.status)
    return got, got["kernel"]
