"""Scenario builders of the interlink filter tests (CPU restatement and GPU parity): a transmitter on a Moon-centred, NRHO-like orbit
tracks low lunar orbiters (nyxb_od_interlink_batch)."""
import math

import numpy as np

import nyx_b200 as nb
from nyx_b200.od import MeasurementType as MT
from nyx_b200.trajectory import Traj
from tests import interlink_oracle as io

S = 10**9
FRAME = nb.MOON_J2000
C_KM_S = 299_792.458
# from_hardware_range_km / from_hardware_doppler_km_s (od/noise/link_specific.rs:179-222) of the reference's interlink test: an
# Allan deviation of 1e-11 over 10 s, T4B chips, average S/N0, an S-band carrier and average C/N0
SIGMA_R = math.sqrt((C_KM_S * 1e-11 * 10.0 / math.sqrt(3.0)) ** 2 + (C_KM_S / (2 * math.pi * 1e6 * math.sqrt(2.0 * 1e5))) ** 2)
SIGMA_D = math.sqrt((C_KM_S * 1e-11) ** 2 + (C_KM_S / (2 * math.pi * 2.2e9 * math.sqrt(2.0 * 10 ** 5.5 * 10.0))) ** 2)


def nrho_orbit():
    """A Moon-centred orbit of the NRHO's shape (periapsis 3 300 km over the north pole, apoapsis 70 000 km), started near apoapsis.  Its
    plane is 60 deg from the LLO's: a transmitter in the receiver's orbital plane would leave the out-of-plane component unobserved."""
    rp, ra = 3_300.0, 70_000.0
    return nb.Orbit.keplerian((rp + ra) / 2.0, (ra - rp) / (ra + rp), 90.0, 60.0, 90.0, 160.0, 0, FRAME)


def llo_orbit():
    """The reference test's low lunar orbit: 110 km altitude, e = 1e-4, polar; started where the transmitter sees it."""
    return nb.Orbit.keplerian(1737.4 + 110.0, 1e-4, 90.0, 0.0, 0.0, 220.0, 0, FRAME)


def dynamics(degree=8):
    if degree:
        gd = nb.GravityFieldData.from_fixture("luna_jggrx_80x80", degree, degree, nb.IAU_MOON_FRAME)
        return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())


def record(dyn, orbit, end_ns, step_s=10.0, name=None):
    """Traj of `orbit` from its epoch to end_ns on the C oracle (RK89 at a fixed step, every step recorded)."""
    from oracle import pyoracle as oracle

    sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    st, cs, ep = nb.pack_spacecraft([sc])
    cap = int((end_ns - orbit.epoch) // int(step_s * S)) + 4
    topts = nb.IntegratorOptions.with_fixed_step_s(step_s)
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(dyn.pack(FRAME, None).c, topts.to_c(nb.IntegratorMethod.RungeKutta89),
                                                                  st, cs, ep, int(end_ns), traj_capacity=cap)
    assert status[0] == 0
    k = int(t_cnt[0])
    return Traj(sc, t_ep[:k, 0].copy(), np.ascontiguousarray(t_st[:, :k, 0].T), name).finalize()


def device(traj, types=(MT.Range, MT.Doppler), sigma=(1e-3, 1e-6), bias=0.0):
    noises = {MT.Range: nb.StochasticNoise(sigma[0], bias), MT.Doppler: nb.StochasticNoise(sigma[1], bias)}
    return nb.InterlinkTxSpacecraft(traj, list(types), noises)


def scenario(n=4, n_msr=30, degree=8, types=(MT.Range, MT.Doppler), cadence_s=60, tx_span_s=None, seed=0, pos_err=0.5, vel_err=5e-4,
             sigma=(1e-3, 1e-6), bias=0.0, tx_start_s=None):
    """n filters of the LLO, tracked every `cadence_s` by the NRHO transmitter (noisy, seeded); the filter's transmitter recording
    spans [tx_start_s, tx_span_s] seconds (default: the whole arc, as the simulation's)."""
    dyn = dynamics(degree)
    orbit = llo_orbit()
    epochs = (orbit.epoch + np.arange(1, n_msr + 1) * cadence_s * S).astype(np.int64)
    traj = record(dyn, nrho_orbit(), orbit.epoch + (n_msr + 1) * cadence_s * S, name="NRHO Tx SC")
    truth_tr = record(dyn, orbit, int(epochs[-1]))
    truth = np.stack([truth_tr.at(int(e)).orbit.to_cartesian_pos_vel() for e in epochs])          # [m][6]
    truth = np.repeat(truth[:, :, None], n, axis=2)
    devices = {"NRHO": device(traj, types, sigma, bias)}
    arc = nb.simulate_interlink(epochs, truth, devices, ["NRHO"] * n_msr, FRAME, np.random.default_rng(seed))
    if tx_span_s is not None or tx_start_s is not None:    # the filter's transmitter recording covers part of the arc only
        traj = traj.filter_by_epoch(orbit.epoch + int((tx_start_s or 0) * S),
                                    int(traj.epochs_ns[-1]) if tx_span_s is None else orbit.epoch + int(tx_span_s * S))
        devices = {"NRHO": device(traj, types, sigma, bias)}
    truth0 = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    rng = np.random.default_rng(seed + 1)
    ests = []
    for _ in range(n):
        v = truth0.to_vector()
        v[:3] += rng.normal(0, pos_err, 3)
        v[3:6] += rng.normal(0, vel_err, 3)
        ests.append(nb.KfEstimate.from_diag(truth0.with_vector(orbit.epoch, v), [pos_err ** 2] * 3 + [vel_err ** 2] * 3 + [0.0] * 3))
    return dict(dyn=dyn, opts=nb.IntegratorOptions.with_fixed_step_s(10.0), frame=FRAME, packed=dyn.pack(FRAME, None), arc=arc, ests=ests,
                devices=devices, truth=truth, truth0=truth0, traj=traj)


def oracle_run(sc, odp, i, sink=None):
    """The restatement (tests/interlink_oracle.py) of filter i of a scenario under the process odp."""
    names, dev_c, (_sink, _n_tx, _keep) = odp.interlink_c(sc["frame"])
    trajs = []
    for nm in names:
        t = odp.devices[nm].traj
        if all(u is not t for u in trajs):
            trajs.append(t)
    arc = sc["arc"]
    tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
    est = sc["ests"][i]
    m = est.nominal_state.mass
    cs = np.array([m.dry_mass_kg, m.extra_mass_kg, est.nominal_state.srp.area_m2, est.nominal_state.drag.area_m2])
    prop = odp.prop
    return io.process_arc(sc["packed"].c, prop.opts.to_c(prop.method), odp.config_c(), [dev_c[s] for s in range(len(names))], trajs,
                          arc.epoch_ns, tracker, np.ascontiguousarray(arc.obs[:, :, i]), est.nominal_state.to_vector(), cs,
                          est.nominal_state.epoch(), est.covar, sink=sink)
