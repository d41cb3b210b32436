"""Scenario builder for the batch least-squares tests (CPU restatement and GPU parity)."""
import numpy as np

import nyx_b200 as nb
from nyx_b200 import abi

S = 10**9


def blse_scenario(oracle, n=4, n_msr=20, cadence_s=60, seed=3, degree=4, stepping="fixed", mode=None, pos_err_km=1.0, vel_err_km_s=1e-3,
                  noise=False, bias_km=0.0, types=(nb.MeasurementType.Range, nb.MeasurementType.Doppler), mask_deg=-90.0,
                  truth_method=nb.IntegratorMethod.RungeKutta89):
    """LEO spacecraft tracked by two Earth stations.  The truth is propagated with the CPU oracle (truth_method, 10 s); the tracking is
    noise-free unless `noise`; each problem starts from its own guess, dispersed by about pos_err_km / vel_err_km_s."""
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    kw = {} if mode is None else dict(mode=mode)
    if stepping == "fixed":
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(10.0), **kw)
    else:
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions(init_step=7 * S), **kw)
    orbit = nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame)
    truth0 = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
    rn, dn = nb.StochasticNoise(1e-2, bias_km), nb.StochasticNoise(1e-5)
    devices = {"Madrid": nb.GroundStation.dss65_madrid(mask_deg, rn, dn), "Canberra": nb.GroundStation.dss34_canberra(mask_deg, rn, dn)}
    for d in devices.values():
        d.measurement_types = tuple(types)
    names = list(devices)
    epochs = (np.arange(1, n_msr + 1) * cadence_s * S).astype(np.int64)
    schedule = [names[(k // 5) % 2] for k in range(n_msr)]
    packed = dyn.pack(frame, None)
    st, cs, ep = nb.pack_spacecraft([truth0])
    cap = n_msr * cadence_s // 10 + 2
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0)
    _, _, _, status, (t_ep, t_st, t_cnt) = oracle.propagate_batch(packed.c, topts.to_c(truth_method), st, cs, ep,
                                                                  int(epochs[-1]), traj_capacity=cap)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    truth = np.repeat(t_st[:, idx, 0].T[:, :, None], n, axis=2)
    rng = np.random.default_rng(seed)
    arc = nb.simulate_tracking(epochs, truth, devices, schedule, frame, None, rng if noise else None)
    guesses = []
    for i in range(n):
        v = truth0.to_vector()
        v[:6] += np.concatenate([rng.normal(0, pos_err_km, 3), rng.normal(0, vel_err_km_s, 3)])
        guesses.append(truth0.with_vector(0, v))
    return dict(frame=frame, dyn=dyn, prop=prop, devices=devices, arc=arc, guesses=guesses, truth0=truth0, packed=packed,
                opts_c=prop.opts.to_c(prop.method))


def bls(sc, **kw):
    return nb.BatchLeastSquares(sc["prop"], sc["devices"], None, **kw)


def oracle_cfg(b):
    from .blse_oracle import Config

    return Config(int(b.solver), b.tolerance_pos_km, b.max_iterations, b.max_step, b.epoch_precision, b.lm_lambda_init, b.lm_lambda_decrease,
                  b.lm_lambda_increase, b.lm_lambda_min, b.lm_lambda_max, b.lm_use_diag_scaling)


def consts(g):
    return np.array([g.mass.dry_mass_kg, g.mass.extra_mass_kg, g.srp.area_m2, g.drag.area_m2])


def oracle_args(sc, b, i, guess=None, arc=None):
    """The arguments of blse_oracle.estimate / evaluate for problem i."""
    arc = arc or sc["arc"]
    g = guess or sc["guesses"][i]
    names = list(b.devices)
    st_c = (abi.GroundStationC * max(len(names), 1))()
    for j, nme in enumerate(names):
        st_c[j] = b.devices[nme].to_c(sc["frame"], None)
    tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
    return (sc["packed"].c, sc["opts_c"], oracle_cfg(b), st_c, arc.epoch_ns, tracker, np.ascontiguousarray(arc.obs[:, :, i]), g.to_vector(),
            consts(g), g.epoch())
