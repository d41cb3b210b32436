"""Inputs of the degree-71..96 parity tests (tests/test_gpu_high_degree.py) and of their CPU companion
(tests/test_high_degree_inputs.py): gravity fields of degree 96, the top of the range the C ABI accepts (NYXB_MAX_DEGREE), two
ensembles that make the top degrees visible, and the oracle results the kernels are compared with.

Fields.  No degree-96 data file ships with the project, so the fields are built in memory:
  earth  JGM-3 rows 0..70 from data/jgm3_70x70.npz, rows 71..96 drawn (seed 9671)
  moon   GRAIL JGGRX rows 0..80 from data/luna_jggrx_80x80.npz, rows 81..96 drawn (seed 9681)
Above the fixture's top degree every C̄nm (m = 0..n) and S̄nm (m = 1..n) is an independent normal draw of
np.random.default_rng(seed) with standard deviation sigma_n, the degree RMS sqrt(sum_m (C̄nm^2 + S̄nm^2) / (2n + 1)) of a power law
log sigma_n = a + b log n fitted by least squares over the fixture's top ten degrees (61..70 and 71..80): a Kaula-like continuation
without a step in the spectrum.  Draws are made row by row, C before S, m ascending.

Ensembles (RK89 at a fixed 60 s, to END = 3 h; start epochs spread over the first 40 min at the nanosecond, per-trajectory masses):
  moon   40 lunar orbits, periapsis altitude 30..60 km (there rho^96 ~ 0.2), apoapsis 80..200 km, about 1.5 revolutions
  earth  24 LEO orbits at 250..300 km (rho^96 ~ 0.01), about two revolutions
Inclinations include exactly polar and near-polar orbits (|sin phi| -> 1 is sampled on every revolution), retrograde ones and a
few low ones."""
import functools

import numpy as np

import nyx_b200 as nb
from tests.util import S

TOP = 96
FIXTURE = {"earth": ("jgm3_70x70", 70, nb.IAU_EARTH_FRAME, 9671), "moon": ("luna_jggrx_80x80", 80, nb.IAU_MOON_FRAME, 9681)}
FRAME = {"earth": nb.EARTH_J2000, "moon": nb.MOON_J2000}
END = 3 * 3600 * S
STEP_S = 60.0
RK89 = nb.IntegratorMethod.RungeKutta89
INCLINATIONS = (90.0, 89.7, 88.0, 92.5, 85.0, 97.0, 70.0, 120.0, 30.0, 60.0)
# Field changes that each touch only coefficients above degree 80 (tests/test_high_degree_inputs.py)
DROPS = ("truncate_95", "sectoral_96", "zonal_above_80", "s_row_96")


def degree_rms(c, s, n):
    return float(np.sqrt((c[n, : n + 1] ** 2 + s[n, : n + 1] ** 2).sum() / (2 * n + 1)))


@functools.lru_cache(maxsize=None)
def _full(body):
    """(c[97][97], s[97][97], power-law coefficients (a, b)) of the degree-96 field of `body`."""
    name, top, frame, seed = FIXTURE[body]
    fx = nb.GravityFieldData.from_fixture(name, top, top, frame)
    c, s = np.zeros((TOP + 1, TOP + 1)), np.zeros((TOP + 1, TOP + 1))
    c[: top + 1, : top + 1], s[: top + 1, : top + 1] = fx.c_nm, fx.s_nm
    ns = np.arange(top - 9, top + 1)
    b, a = np.polyfit(np.log(ns), np.log([degree_rms(c, s, n) for n in ns]), 1)
    rng = np.random.default_rng(seed)
    for n in range(top + 1, TOP + 1):
        sigma = np.exp(a + b * np.log(n))
        c[n, : n + 1] = rng.normal(0.0, sigma, n + 1)
        s[n, 1: n + 1] = rng.normal(0.0, sigma, n)
    for x in (c, s):
        x.setflags(write=False)
    return c, s, (a, b)


def field_data(body, degree=TOP, order=None, drop=None):
    """GravityFieldData of `body` truncated to degree x order (rows above `degree` removed, orders above `order` zero), with one
    of DROPS applied."""
    order = degree if order is None else order
    c, s, _ = _full(body)
    if drop == "truncate_95":
        degree, order = 95, min(order, 95)
    c, s = c[: degree + 1, : degree + 1].copy(), s[: degree + 1, : degree + 1].copy()
    c[:, order + 1:] = 0.0
    s[:, order + 1:] = 0.0
    if drop == "sectoral_96":
        c[96, 96] = s[96, 96] = 0.0
    elif drop == "zonal_above_80":
        c[81:, 0] = 0.0
    elif drop == "s_row_96":
        s[96, :] = 0.0
    else:
        assert drop in (None, "truncate_95"), drop
    return nb.GravityFieldData(degree, order, c, s, FIXTURE[body][2])


@functools.lru_cache(maxsize=None)
def dynamics(body, degree=TOP, order=None, drop=None):
    return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(field_data(body, degree, order, drop))))


def propagator(body, mode, degree=TOP, order=None, drop=None, opts=None):
    return nb.Propagator.new(dynamics(body, degree, order, drop), RK89, opts or nb.IntegratorOptions.with_fixed_step_s(STEP_S), mode=mode)


@functools.lru_cache(maxsize=None)
def ensemble(body, seed=96):
    """(state[9][n], consts[4][n], epoch0[n])"""
    n, r_eq, (lo, hi), (alo, ahi) = {"moon": (40, 1737.4, (30.0, 60.0), (80.0, 200.0)),
                                     "earth": (24, 6378.1363, (250.0, 300.0), (250.0, 300.0))}[body]
    rng = np.random.default_rng(seed + (body == "earth"))
    scs = []
    for i in range(n):
        hp = rng.uniform(lo, hi)
        ha = max(hp, rng.uniform(alo, ahi))
        sma = r_eq + (hp + ha) / 2
        orbit = nb.Orbit.keplerian(sma, (ha - hp) / (2 * sma), INCLINATIONS[i % len(INCLINATIONS)], rng.uniform(0, 360),
                                   rng.uniform(0, 360), rng.uniform(0, 360), 0, FRAME[body])
        scs.append(nb.Spacecraft(orbit=orbit, mass=nb.Mass(rng.uniform(60.0, 300.0), rng.uniform(5.0, 40.0), rng.uniform(0.0, 25.0))))
    st, cs, _ = nb.pack_spacecraft(scs)
    ep = rng.integers(0, 2400 * S, n).astype(np.int64)
    for a in (st, cs, ep):
        a.setflags(write=False)
    return st, cs, ep


@functools.lru_cache(maxsize=None)
def oracle_fixed(body, degree=TOP, order=None, drop=None, speed_build=False):
    """The oracle's fixed-step result for the ensemble of `body` (speed_build: its FMA-contraction build)."""
    from oracle import pyoracle

    prop = propagator(body, nb.MODE_STRICT, degree, order, drop)
    st, cs, ep = ensemble(body)
    packed = prop.dynamics.pack(FRAME[body], None)
    out = pyoracle.propagate_batch(packed.c, prop.opts.to_c(prop.method), st, cs, ep, END, speed_build=speed_build)
    assert (out[3] == 0).all(), out[3]
    for a in out[:4]:
        a.setflags(write=False)
    return out


FIXED_DR, FIXED_DV = 5e-9, 5e-12


@functools.lru_cache(maxsize=None)
def fixed_bounds(body, degree=TOP, order=None):
    """(|dr| km, |dv| km/s) bound of a fixed-step FAST comparison: max(5e-9 km, 10 x the oracle's spread against its FMA build)
    and the same for velocity."""
    from tests.util import max_dr_dv

    dr, dv = max_dr_dv(oracle_fixed(body, degree, order, speed_build=True)[0], oracle_fixed(body, degree, order)[0])
    return max(FIXED_DR, 10.0 * dr), max(FIXED_DV, 10.0 * dv)
