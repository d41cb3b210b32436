"""Inputs of the FAST-mode parity matrix (tests/test_gpu_fast_matrix.py) and of its CPU companion (tests/test_fast_matrix_inputs.py):
one ensemble, the force-model configurations, and the oracle results every kernel family is compared with.

The ensemble is built so that a kernel that mixes up lanes or stage epochs gives a different answer: start epochs differ at
the nanosecond, every trajectory has its own dry / extra / propellant mass, SRP area, drag area and Cd, and Cr is drawn from
{-0.3, 0.7, 1.8, 2.5} (both clamps of cosmic/spacecraft.rs:494).  A third of it flies a 300 x 1 500 km orbit, which crosses the
1 000 km branch altitude of the StdAtm density model on every revolution; the rest is the dispersed 300 km circular LEO of
tests/util.leo_ensemble, which passes through the Earth's penumbra and umbra on every revolution."""
import functools

import numpy as np

import nyx_b200 as nb
from tests.util import S, leo_ensemble

N_LEO, N_ECC = 64, 32            # 96 trajectories: three sets of 32 for the transposed kernel
END = 6 * 3600 * S               # absolute end epoch of the fixed-step runs
CR_VALUES = (-0.3, 0.7, 1.8, 2.5)
STDATM_BRANCH_KM = 1000.0        # AtmDensity.StdAtm(1e6 m): pow law above, polynomial below (drag.rs:251-270)
FIXED_DR, FIXED_DV = 5e-9, 5e-12             # bounds of the fixed-step comparisons over 6 h (km, km/s)
FIXED_DR_RK4, FIXED_DV_RK4 = 5e-8, 5e-11     # RK4 at 10 s: 2 160 steps, ten times the round-off of the others

CONFIGS = ("field", "third_body", "srp", "drag_constant", "drag_exponential", "drag_stdatm", "all")
METHODS = tuple(nb.IntegratorMethod)


def method_step_s(method):
    """Step of the all-methods sweep: RK4 at 10 s, the others at 45.5 s, so that every run ends on a shorter final step (the
    F_LAST path).  The configuration sweep runs RK89 at 60 s."""
    return 10.0 if method == nb.IntegratorMethod.RungeKutta4 else 45.5


def bounds(method):
    return (FIXED_DR_RK4, FIXED_DV_RK4) if method == nb.IntegratorMethod.RungeKutta4 else (FIXED_DR, FIXED_DV)


@functools.lru_cache(maxsize=None)
def almanac():
    return nb.Almanac.synthetic(nb.EARTH_J2000, 0, 1.0, pad_days=1.0)


@functools.lru_cache(maxsize=None)
def ensemble(seed=61):
    """(state[9][96], consts[4][96], epoch0[96]); columns 0..63 LEO, 64..95 on the 300 x 1 500 km orbit."""
    _, (st1, cs1, ep1) = leo_ensemble(N_LEO, seed=seed)
    r_eq = 6378.1363
    sma = r_eq + (300.0 + 1500.0) / 2
    orbit = nb.Orbit.keplerian(sma, 600.0 / sma, 51.6, 30.0, 40.0, 0.0, 0, nb.EARTH_J2000)
    template = nb.Spacecraft(orbit=orbit, mass=nb.Mass(100.0, 20.0, 0.0))
    mc = nb.MonteCarlo(template, nb.MvnSpacecraft.from_cartesian_std(template, 1.0, 1e-3), "ecc", seed=seed + 1)
    st2, cs2, ep2 = nb.pack_spacecraft(ds.state for _, ds in mc.generate_states(0, N_ECC))
    st, cs, ep = np.concatenate([st1, st2], axis=1), np.concatenate([cs1, cs2], axis=1), np.concatenate([ep1, ep2])
    n = st.shape[1]
    rng = np.random.default_rng(seed)
    st[6] = np.array(CR_VALUES)[rng.permutation(n) % len(CR_VALUES)]
    st[7] = rng.uniform(1.6, 2.8, n)          # Cd
    st[8] = rng.uniform(5.0, 40.0, n)         # propellant mass
    cs[0] = rng.uniform(60.0, 300.0, n)       # dry mass
    cs[1] = rng.uniform(0.0, 25.0, n)         # extra mass
    cs[2] = rng.uniform(2.0, 14.0, n)         # SRP area (m^2): A/m ~ 0.01 - 0.2 m^2/kg
    cs[3] = rng.uniform(2.0, 14.0, n)         # drag area
    ep = rng.integers(0, 2400 * S, n).astype(np.int64)   # start epochs over the first 40 min, at the nanosecond
    for a in (st, cs, ep):
        a.setflags(write=False)
    return st, cs, ep


def field(degree=21, order=None):
    return nb.GravityField.new(nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree if order is None else order,
                                                                nb.IAU_EARTH_FRAME))


def density(kind):
    return {"drag_constant": nb.AtmDensity.Constant(2e-12), "drag_exponential": nb.AtmDensity.earth_exponential(),
            "drag_stdatm": nb.AtmDensity.StdAtm(1_000_000.0)}[kind]


@functools.lru_cache(maxsize=None)
def dynamics(config, degree=21, order=None, drop=None):
    """SpacecraftDynamics of one configuration with a primary JGM-3 field of degree x order.  `drop` removes one model
    ("field", "point_masses", "srp", "drag" or "second_field") to show that the configuration can see it."""
    alm = almanac()
    primary = [] if drop == "field" else [field(degree, order)]
    pm = [] if drop == "point_masses" else [nb.PointMasses.new([nb.MOON, nb.SUN])]
    srp = [] if drop == "srp" else [nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)]
    if config == "field":
        models, forces = primary, []
    elif config == "third_body":
        models, forces = pm + primary, []
    elif config == "srp":
        models, forces = primary, srp
    elif config.startswith("drag_"):
        models, forces = primary, ([] if drop == "drag" else [nb.Drag(density(config), nb.IAU_EARTH_FRAME)])
    elif config == "all":
        # a second field of the central body (e.g. a low-degree correction model summed after the main one): the lane-cooperative
        # kernel takes its several-fields template and the transposed kernel calls accel_extra_fields
        second = [] if drop == "second_field" else [field(6)]
        drag = [] if drop == "drag" else [nb.Drag(density("drag_stdatm"), nb.IAU_EARTH_FRAME)]
        models, forces = pm + primary + second, srp + drag
    else:
        raise ValueError(config)
    return nb.SpacecraftDynamics.from_models(nb.OrbitalDynamics.new(models), forces)


def propagator(config, method=nb.IntegratorMethod.RungeKutta89, opts=None, degree=21, order=None, drop=None):
    return nb.Propagator.new(dynamics(config, degree, order, drop), method, opts or nb.IntegratorOptions.with_fixed_step_s(60.0),
                             mode=nb.MODE_FAST)


@functools.lru_cache(maxsize=None)
def oracle_fixed(config, method=nb.IntegratorMethod.RungeKutta89, step_s=60.0, degree=21, order=None, drop=None, start=None,
                 end=END, traj_capacity=0):
    """The oracle's fixed-step result for the ensemble (or for `start` = (state, epoch) of an earlier oracle result)."""
    from oracle import pyoracle

    prop = propagator(config, method, nb.IntegratorOptions.with_fixed_step_s(step_s), degree, order, drop)
    st, cs, ep = ensemble()
    if start is not None:
        st, ep = oracle_fixed(*start)[:2]
    packed = prop.dynamics.pack(nb.EARTH_J2000, almanac())
    out = pyoracle.propagate_batch(packed.c, prop.opts.to_c(prop.method), st, cs, ep, end, traj_capacity=traj_capacity)
    for a in out[:4]:
        a.setflags(write=False)
    return out
