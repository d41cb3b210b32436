"""Batch least-squares benchmark (`BatchLeastSquares::estimate` through nyxb_od_bls_batch), timed with CUDA events:

  ref   the geometry of the reference's blse_robust_large_disp test: 22 000 km orbit from 2020-01-01T04:00 UTC, Moon / Sun / Jupiter
        point masses, default RK89, Canberra alone (0 deg mask, default noises), 10 s sampling cut to the first 10 minutes of
        visibility, Levenberg-Marquardt; n = 10 000 guesses dispersed in SMA / RAAN / inclination / eccentricity; per-thread kernel
  c5    lunar 70x70 + Earth/Sun point masses + SRP (warp-cooperative kernel), Madrid / Canberra / Goldstone every 10 minutes over
        1 day, Levenberg-Marquardt with 3 iterations; n = 1 000 guesses dispersed by 100 m / 10 cm/s

Each line reports the kernel time, iterations/s, STM steps/s, the status counts, the GPU name and power limit read in the same call,
and the largest difference from the restatement (tests/blse_oracle.py) on a sample.  Needs a GPU.
Run from the repository root:  python scripts/blse_bench.py [--only ref,c5] [--sample 2]
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

import nyx_b200 as nb  # noqa: E402
from nyx_b200 import abi  # noqa: E402

from predict_bench import c5 as c5_predict, gpu_info  # noqa: E402

S = 10**9


def _arc(frame, alm, dyn, truth0, devices, cadence_s, span_s):
    from oracle import pyoracle

    epochs = truth0.epoch() + (np.arange(1, int(span_s // cadence_s) + 1) * cadence_s * S).astype(np.int64)
    st, cs, ep = nb.pack_spacecraft([truth0])
    topts = nb.IntegratorOptions.with_fixed_step_s(10.0).to_c(nb.IntegratorMethod.RungeKutta89)
    _, _, _, status, (t_ep, t_st, t_cnt) = pyoracle.propagate_batch(dyn.pack(frame, alm).c, topts, st, cs, ep, int(epochs[-1]),
                                                                    traj_capacity=int(span_s // 10) + 2)
    assert status[0] == 0
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    names = list(devices)
    sched = [names[k % len(names)] for k in range(len(epochs))]
    return nb.simulate_tracking(epochs, t_st[:, idx, 0].T[:, :, None], devices, sched, frame, alm, np.random.default_rng(0))


def ref(n, rng):
    from nyx_b200.cosmic import utc_iso_to_epochs

    t0 = int(utc_iso_to_epochs(["2020-01-01T04:00:00"])[0])
    frame = nb.EARTH_J2000
    alm = nb.Almanac.synthetic(frame, t0, 1.0, bodies=(nb.MOON, nb.SUN, nb.JUPITER_BARYCENTER), pad_days=1.0)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.point_masses([nb.MOON, nb.SUN, nb.JUPITER_BARYCENTER]))
    truth0 = nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0, 0.01, 30.0, 80.0, 40.0, 170.0, t0, frame))
    devices = {"Canberra": nb.GroundStation.dss34_canberra(0.0, nb.StochasticNoise.default_range_km(), nb.StochasticNoise.default_doppler_km_s())}
    arc = _arc(frame, alm, dyn, truth0, devices, 10, 6 * 3600)
    vis = ~np.isnan(arc.obs[:, 0, 0])
    arc = nb.TrackingDataArc(arc.epoch_ns[vis], [t for t, v in zip(arc.tracker, vis) if v], arc.obs[vis]).filter_by_offset(None, 600 * S)
    guesses = [nb.Spacecraft(orbit=nb.Orbit.keplerian(22000.0 + rng.normal(0, 0.02), 0.01 + rng.normal(0, 2e-4), 30.0 + rng.normal(0, 0.02),
                                                      80.0 + rng.normal(0, 0.02), 40.0, 170.0, t0, frame)) for _ in range(n)]
    b = nb.BatchLeastSquares(nb.Propagator.default(dyn, mode=nb.MODE_FAST), devices, alm, solver=nb.BLSSolver.LevenbergMarquardt)
    return frame, alm, dyn, b, guesses, arc, nb.KERNEL_THREAD


def c5(n, rng):
    frame, alm, dyn, prop, ests, _ = c5_predict(n, rng)
    rn, dn = nb.StochasticNoise(1e-2), nb.StochasticNoise(1e-5)
    devices = {"Madrid": nb.GroundStation.dss65_madrid(0.0, rn, dn), "Canberra": nb.GroundStation.dss34_canberra(0.0, rn, dn),
               "Goldstone": nb.GroundStation.dss13_goldstone(0.0, rn, dn)}
    truth0 = ests[0].nominal_state.with_vector(0, ests[0].nominal_state.to_vector())
    arc = _arc(frame, alm, dyn, truth0, devices, 600, 86400)
    arc = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, np.repeat(arc.obs, n, axis=2))
    b = nb.BatchLeastSquares(prop, devices, alm, solver=nb.BLSSolver.LevenbergMarquardt, max_iterations=3)
    return frame, alm, dyn, b, [e.nominal_state for e in ests], arc, nb.KERNEL_AUTO


def run(name, builder, n, sample, gpu):
    from tests import blse_oracle
    from tests.blse_util import consts, oracle_cfg

    rng = np.random.default_rng(0)
    frame, alm, dyn, b, guesses, arc, kernel = builder(n, rng)
    arc_n = arc if arc.n == n else nb.TrackingDataArc(arc.epoch_ns, arc.tracker, np.repeat(arc.obs, n, axis=2))
    eng = b.prop.engine(frame, alm)
    eng.set_kernel(kernel)
    b.estimate_ensemble(guesses[:8], nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc_n.obs[:, :, :8]))   # module load, allocator
    t0 = time.perf_counter()
    sol = b.estimate_ensemble(guesses, arc_n)
    wall = time.perf_counter() - t0
    kms = eng.last_kernel_ms()
    family = {nb.KERNEL_THREAD: "thread", nb.KERNEL_COOP: "coop"}.get(eng.last_kernel(), str(eng.last_kernel()))
    iters = int(sol.iterations.sum())
    steps = int(sol.details["n_steps"].sum())
    statuses = {int(k): int(v) for k, v in zip(*np.unique(sol.status, return_counts=True))}
    names = list(b.devices)
    st_c = (abi.GroundStationC * len(names))(*[b.devices[k].to_c(frame, alm) for k in names])
    trk = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
    dyn_c, opts_c = dyn.pack(frame, alm).c, b.prop.opts.to_c(b.prop.method)
    worst = 0.0
    for i in range(sample):
        g = guesses[i]
        r = blse_oracle.estimate(dyn_c, opts_c, oracle_cfg(b), st_c, arc.epoch_ns, trk, np.ascontiguousarray(arc_n.obs[:, :, i]), g.to_vector(),
                                 consts(g), g.epoch())
        assert r["status"] == sol.status[i] and r["iterations"] == sol.iterations[i]
        worst = max(worst, float(np.abs(r["state"][:3] - sol.state_soa[:3, i]).max()))
    line = dict(workload=name, n=n, msrs=len(arc), kernel_family=family, kernel_ms=kms, call_wall_s=wall, iterations=iters,
                iterations_per_s=iters / (kms * 1e-3), stm_steps=steps, stm_steps_per_s=steps / (kms * 1e-3), status_counts=statuses,
                converged=int(sol.converged.sum()), parity=dict(sample=sample, max_dr_km=worst), gpu=gpu[0], power_limit=gpu[1])
    print(json.dumps(line), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="ref,c5")
    ap.add_argument("--sample", type=int, default=2)
    args = ap.parse_args()
    gpu = gpu_info()
    cases = {"ref": (ref, 10000), "c5": (c5, 1000)}
    for k in args.only.split(","):
        run(k, *cases[k], args.sample, gpu)


if __name__ == "__main__":
    main()
