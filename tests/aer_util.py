"""Scenario builders of the angle-tracking filter tests (CPU restatement and GPU parity): ground stations that measure azimuth and
elevation next to range and Doppler (nyxb_od_aer_batch)."""
import numpy as np

import nyx_b200 as nb
from nyx_b200.od import MeasurementType as MT
from tests import aer_oracle as ao

S = 10**9
ALL = (MT.Range, MT.Doppler, MT.Azimuth, MT.Elevation)
NOISE = {MT.Range: 2e-3, MT.Doppler: 3e-6, MT.Azimuth: 1e-3, MT.Elevation: 1e-3}   # km, km/s, deg, deg


def dsn(mask_deg=-90.0, types=ALL, sigma=None, bias=0.0, names=("Madrid", "Canberra", "Goldstone")):
    """The three DSN stations of the reference's builtins, each with `types` in that list order (with_msr_type)."""
    sigma = dict(NOISE if sigma is None else sigma)
    ctor = {"Madrid": nb.GroundStation.dss65_madrid, "Canberra": nb.GroundStation.dss34_canberra,
            "Goldstone": nb.GroundStation.dss13_goldstone}
    out = {}
    for nm in names:
        gs = ctor[nm](mask_deg, nb.StochasticNoise(sigma[MT.Range]), nb.StochasticNoise(sigma[MT.Doppler]))
        gs.measurement_types = []
        for t in types:
            gs.with_msr_type(t, nb.StochasticNoise(sigma[t], bias))
        out[nm] = gs
    return out


def truth_states(dyn, frame, truth0, epochs):
    """The truth at `epochs` from the C oracle's RK89 at a fixed 10 s step ([m][9])."""
    from oracle import pyoracle as oracle

    packed = dyn.pack(frame, None)
    st, cs, ep = nb.pack_spacecraft([truth0])
    cap = int((epochs[-1] - truth0.epoch()) // (10 * S)) + 4
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0)
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(packed.c, topts.to_c(nb.IntegratorMethod.RungeKutta89), st, cs, ep,
                                                                  int(epochs[-1]), traj_capacity=cap)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    return t_st[:, idx, 0].T


def scenario(n=4, n_msr=30, degree=8, fixed=False, types=ALL, mask_deg=-90.0, bias=0.0, seed=0, sigma=None, pos_err=0.5, vel_err=5e-4,
             cadence_s=60, orbit=None):
    """n filters around a 7 000 km orbit, tracked every `cadence_s` by Madrid, Canberra and Goldstone in turn (noisy, seeded)."""
    frame = nb.EARTH_J2000
    if degree:
        gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    else:
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    orbit = orbit or nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame)
    truth0 = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    epochs = (orbit.epoch + np.arange(1, n_msr + 1) * cadence_s * S).astype(np.int64)
    truth = np.repeat(truth_states(dyn, frame, truth0, epochs)[:, :, None], n, axis=2)
    devices = dsn(mask_deg, types, sigma, bias)
    names = list(devices)
    schedule = [names[k % len(names)] for k in range(n_msr)]
    rng = np.random.default_rng(seed)
    arc = nb.simulate_tracking(epochs, truth, devices, schedule, frame, None, rng)
    ests = []
    for _ in range(n):
        v = truth0.to_vector()
        v[:3] += rng.normal(0, pos_err, 3)
        v[3:6] += rng.normal(0, vel_err, 3)
        ests.append(nb.KfEstimate.from_diag(truth0.with_vector(orbit.epoch, v), [pos_err ** 2] * 3 + [vel_err ** 2] * 3 + [0.0] * 3))
    opts = nb.IntegratorOptions.with_fixed_step_s(10.0) if fixed else nb.IntegratorOptions.default()
    return dict(dyn=dyn, opts=opts, frame=frame, packed=dyn.pack(frame, None), arc=arc, ests=ests, devices=devices, truth=truth,
                truth0=truth0)


def oracle_run(sc, odp, i, sink=None):
    """The restatement (tests/aer_oracle.py) of filter i of a scenario under the process odp."""
    names, st_c = odp.aer_stations_c(sc["frame"])
    arc = sc["arc"]
    tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
    est = sc["ests"][i]
    m = est.nominal_state.mass
    cs = np.array([m.dry_mass_kg, m.extra_mass_kg, est.nominal_state.srp.area_m2, est.nominal_state.drag.area_m2])
    prop = odp.prop
    return ao.process_arc(sc["packed"].c, prop.opts.to_c(prop.method), odp.config_c(), st_c, arc.epoch_ns, tracker,
                          np.ascontiguousarray(arc.obs[:, :, i]), est.nominal_state.to_vector(), cs, est.nominal_state.epoch(), est.covar,
                          sink=sink)
