"""Scenario builders of the position-fix filter tests (CPU restatement and GPU parity)."""
import numpy as np

import nyx_b200 as nb
from nyx_b200.od import MeasurementType as MT
from tests import position_oracle as po

S = 10**9


def scenario(n=4, n_msr=30, degree=8, fixed=False, sigma=1e-3, bias=0.0, types=(MT.X, MT.Y, MT.Z), seed=0, two_devices=False,
             orbit=None, pos_err=1.0, vel_err=1e-3, cadence_s=60):
    frame = nb.EARTH_J2000
    if degree:
        gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    else:
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
    orbit = orbit or nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame)
    truth0 = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    epochs = (orbit.epoch + np.arange(1, n_msr + 1) * cadence_s * S).astype(np.int64)
    from oracle import pyoracle as oracle
    packed = dyn.pack(frame, None)
    st, cs, ep = nb.pack_spacecraft([truth0])
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0)
    cap = n_msr * cadence_s // 10 + 2
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(packed.c, topts.to_c(nb.IntegratorMethod.RungeKutta89), st, cs, ep,
                                                                  int(epochs[-1]), traj_capacity=cap)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    truth = np.repeat(t_st[:, idx, 0].T[:, :, None], n, axis=2)
    devices = {"gnss": nb.PositionDevice("gnss")}
    for t in types:
        devices["gnss"].with_noise(t, nb.StochasticNoise(sigma, bias))
    names = ["gnss"]
    if two_devices:
        devices["gnss2"] = nb.PositionDevice("gnss2")
        for t in (MT.Z, MT.X):
            devices["gnss2"].with_noise(t, nb.StochasticNoise(2 * sigma))
        names.append("gnss2")
    schedule = [names[k % len(names)] for k in range(n_msr)]
    rng = np.random.default_rng(seed)
    arc = nb.simulate_position_fixes(epochs, truth, devices, schedule, rng)
    ests = []
    for i in range(n):
        v = truth0.to_vector()
        v[:3] += rng.normal(0, pos_err, 3)
        v[3:6] += rng.normal(0, vel_err, 3)
        ests.append(nb.KfEstimate.from_diag(truth0.with_vector(orbit.epoch, v),
                                            [pos_err ** 2] * 3 + [vel_err ** 2] * 3 + [0.0, 0.0, 0.0]))
    opts = nb.IntegratorOptions.with_fixed_step_s(10.0) if fixed else nb.IntegratorOptions.default()
    return dict(dyn=dyn, opts=opts, frame=frame, packed=packed, arc=arc, ests=ests, devices=devices, truth=truth, truth0=truth0)


def oracle_run(sc, odp, i, sink=None):
    names, dev_c = odp.position_devices_c()
    arc = sc["arc"]
    tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
    est = sc["ests"][i]
    m = est.nominal_state.mass
    cs = np.array([m.dry_mass_kg, m.extra_mass_kg, est.nominal_state.srp.area_m2, est.nominal_state.drag.area_m2])
    prop = odp.prop
    return po.process_arc(sc["packed"].c, prop.opts.to_c(prop.method), odp.config_c(), dev_c, arc.epoch_ns, tracker,
                          np.ascontiguousarray(arc.obs[:, :, i]), est.nominal_state.to_vector(), cs, est.nominal_state.epoch(), est.covar,
                          sink=sink)


def gps_scenario(n_seeds):
    """tests/orbit_determination/gps_position.rs: SMA 22 000 km, e 0.01, i 30, RAAN 80, AoP 40, TA 170 at 2020-01-01 04:00 UTC,
    two-body Earth, RK89 defaults, 6 h of fixes every minute with sigma = 1 m, initial error (+1, -1, +1) km and (+1, -1, +1) m/s."""
    t0 = nb.utc_iso_to_epochs(["2020-01-01T04:00:00"])[0]
    orbit = nb.Orbit.keplerian(22000.0, 0.01, 30.0, 80.0, 40.0, 170.0, int(t0), nb.EARTH_J2000)
    sc = scenario(n=n_seeds, n_msr=360, degree=0, orbit=orbit, sigma=1e-3, pos_err=0.0, vel_err=0.0)
    arcs = [scenario(n=1, n_msr=360, degree=0, orbit=orbit, sigma=1e-3, pos_err=0.0, vel_err=0.0, seed=s)["arc"] for s in range(n_seeds)]
    sc["arc"] = nb.TrackingDataArc(arcs[0].epoch_ns, arcs[0].tracker, np.concatenate([a.obs for a in arcs], axis=2), arcs[0].types)
    ests = []
    for _ in range(n_seeds):
        v = sc["truth0"].to_vector()
        v[:6] += [1.0, -1.0, 1.0, 1e-3, -1e-3, 1e-3]
        ests.append(nb.KfEstimate.from_diag(sc["truth0"].with_vector(orbit.epoch, v), [1.0] * 3 + [1e-6] * 3 + [0.0] * 3))
    sc["ests"] = ests
    return sc


def gps_errors_restatement(n_seeds):
    """Final position error (m, RIC norm) of the reference's GPS scenario on the CPU restatement, one per noise stream.  As the
    reference (gps_position.rs:93-99) it takes the LAST ESTIMATE's nominal state, the pre-update nominal of the last fix."""
    sc = gps_scenario(n_seeds)
    prop = nb.Propagator.new(sc["dyn"], nb.IntegratorMethod.RungeKutta89, sc["opts"], mode=nb.MODE_STRICT)
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, sc["devices"], None, msr_size=3)
    truth = sc["truth"][-1, :3, 0]
    errs = []
    for i in range(n_seeds):
        sink = []
        oracle_run(sc, odp, i, sink=sink)
        errs.append(ric_error_m(sc, sink[-1]["nominal"], truth))
    return errs


def ric_error_m(sc, y, truth_pos):
    sc_f = sc["truth0"].with_vector(sc["truth0"].orbit.epoch, np.asarray(y, dtype=np.float64))
    dcm = nb.od.dcm_ric_to_inertial(sc_f.orbit)
    return float(np.linalg.norm(dcm[:3, :3].T @ (np.asarray(y[:3]) - truth_pos)) * 1e3)
