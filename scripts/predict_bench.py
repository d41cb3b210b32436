"""Covariance mapping on the GPU (`nyxb_od_predict_batch`, KalmanODProcess::predict_for): one JSON line per workload.

  c3_full   C3 geometry (JWST-like, examples/02_jwst_covar_monte_carlo), RIC uncertainty of main.rs:77-86, CKF, max_step 1 min,
            6.5 days, n = 1 000, every record kept (9 361 records x 90 doubles per run)
  c3_final  the same with n = 10 000, final estimates only
  c5        lunar 70x70 + Earth/Sun point masses + SRP (warp-cooperative kernel), n = 1 000, 1 day, final estimates only

Each line: time updates/s and trajectory steps/s over the kernel time (CUDA events), the kernel family, record bytes, the STM
propagation of the same ensemble over the same span (`nyxb_propagate_batch_stm`) for comparison, parity against the oracle
restatement on a sample, the oracle's host rate with the core count, the GPU name and power limit.  Needs a GPU.
Run from the repository root:  python scripts/predict_bench.py [--only c3_full,c3_final,c5] [--sample 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import nyx_b200 as nb  # noqa: E402
from nyx_b200.frames import EARTH  # noqa: E402

S = 10**9


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True)
    name, power = (out.stdout.strip().split(", ") + ["?"])[:2] if out.returncode == 0 else ("unknown", "unknown")
    return name, power


def c3(n, rng):
    frame = nb.EARTH_J2000
    alm = nb.Almanac.synthetic(frame, 0, 8.5)
    srp = nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)
    dyn = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.point_masses([nb.MOON, nb.SUN]), srp)
    orbit = nb.Orbit.cartesian(119901.070276, -1389299.665421, -1041369.150539, 0.045956, -0.013168, 0.034535, 0, frame)
    jwst = nb.Spacecraft(orbit=orbit, mass=nb.Mass(6200.0, 0.0, 0.0), srp=nb.SRPData(21.197 * 14.162, 1.56))
    est = nb.SpacecraftUncertainty(jwst, nb.LocalFrame.RIC, x_km=0.5, y_km=0.3, z_km=1.5, vx_km_s=1e-4, vy_km_s=0.6e-3,
                                   vz_km_s=3e-3).to_estimate()
    # an ensemble of JWST-like estimates: the nominal state drawn from the estimate itself
    x = est.to_random_variable().sample_vectors(rng, n)
    ests = [nb.KfEstimate(jwst.with_vector(0, jwst.to_vector() + x[i]), est.covar) for i in range(n)]
    return frame, alm, dyn, nb.Propagator.default(dyn, mode=nb.MODE_FAST), ests, int(6.5 * 86400) * S


def c5(n, rng):
    frame = nb.MOON_J2000
    alm = nb.Almanac.synthetic(frame, 0, 3.0, bodies=(EARTH, nb.SUN))
    gd = nb.GravityFieldData.from_fixture("luna_jggrx_80x80", 70, 70, nb.IAU_MOON_FRAME)
    srp = nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)
    dyn = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.new([nb.PointMasses.new([EARTH, nb.SUN]), nb.GravityField.new(gd)]), srp)
    orbit = nb.Orbit.keplerian(1737.4 + 100.0, 0.002, 88.0, 20.0, 10.0, 0.0, 0, frame)
    sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(1018.0, 900.0, 0.0), srp=nb.SRPData(3.9 * 2.7, 0.96))
    cov = np.diag([0.1, 0.1, 0.1, 1e-4, 1e-4, 1e-4, 0.0, 0.0, 0.0]) ** 2
    x = nb.MvnSpacecraft.from_spacecraft_cov(sc, cov).sample_vectors(rng, n)
    ests = [nb.KfEstimate(sc.with_vector(0, sc.to_vector() + x[i]), cov) for i in range(n)]
    return frame, alm, dyn, nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST), ests, 86400 * S


def run(name, builder, n, full_records, sample, gpu):
    from tests.predict_oracle import predict_until as oracle_predict

    rng = np.random.default_rng(0)
    frame, alm, dyn, prop, ests, span = builder(n, rng)
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.DeviationTracking, None, {}, alm)
    eng = prop.engine(frame, alm)
    warm = odp.predict_ensemble_for(ests[:8], 10 * 60 * S, capacity=0)   # module load, allocator
    assert (warm.status == 0).all()
    t0 = time.perf_counter()
    sol = odp.predict_ensemble_for(ests, span, capacity=None if full_records else 0)
    wall = time.perf_counter() - t0
    kms = eng.last_kernel_ms()
    family = {nb.KERNEL_THREAD: "thread", nb.KERNEL_COOP: "coop"}.get(eng.last_kernel(), str(eng.last_kernel()))
    assert (sol.status == 0).all(), np.unique(sol.status)
    tus = int((sol.rec_count - 1).sum())
    steps = int(sol.details["n_steps"].sum())
    rec_bytes = 0 if not full_records else int(sol.capacity) * 90 * 8 * n
    # STM propagation of the same ensemble over the same span, one launch, no time updates
    st, cs, ep = nb.pack_spacecraft(e.nominal_state for e in ests)
    out, oep, _, det, status = eng.propagate_batch_stm(st, cs, ep, int(span))
    stm_ms = eng.last_kernel_ms()
    stm_steps = int(det["n_steps"].sum())
    # parity on a sample, and the oracle's host rate
    dyn_c, opts_c = dyn.pack(frame, alm).c, prop.opts.to_c(prop.method)
    worst_r, worst_p, o_steps, o_time = 0.0, 0.0, 0, 0.0
    for i in range(sample):
        e = ests[i]
        sc = e.nominal_state
        c4 = np.array([sc.mass.dry_mass_kg, sc.mass.extra_mass_kg, sc.srp.area_m2, sc.drag.area_m2])
        t1 = time.perf_counter()
        ref = oracle_predict(dyn_c, opts_c, odp.config_c(), sc.to_vector(), c4, sc.epoch(), e.covar, sc.epoch() + span,
                             e.state_deviation)
        o_time += time.perf_counter() - t1
        o_steps += ref["n_steps"]
        assert ref["count"] == sol.rec_count[i] and ref["epoch"] == sol.final_epoch_ns[i]
        worst_r = max(worst_r, float(np.abs(ref["state"][:3] - sol.final_state_soa[:3, i]).max()))
        worst_p = max(worst_p, float(np.abs(ref["covar"][:6, :6] - sol.covar[i][:6, :6]).max() / np.abs(ref["covar"][:6, :6]).max()))
    line = dict(workload=name, n=n, span_s=span / S, max_step_s=odp.max_step / S, kernel_family=family, kernel_ms=kms,
                call_wall_s=wall, time_updates=tus, time_updates_per_s=tus / (kms * 1e-3), traj_steps=steps,
                traj_steps_per_s=steps / (kms * 1e-3), record_bytes=rec_bytes,
                stm_propagation=dict(kernel_ms=stm_ms, traj_steps=stm_steps, traj_steps_per_s=stm_steps / (stm_ms * 1e-3)),
                parity=dict(sample=sample, max_dr_km=worst_r, max_rel_dP=worst_p),
                oracle=dict(host_steps_per_s_one_core=o_steps / o_time if o_time else None, cores=os.cpu_count()),
                gpu=gpu[0], power_limit=gpu[1])
    print(json.dumps(line), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c3_full,c3_final,c5")
    ap.add_argument("--sample", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    gpu = gpu_info()
    cases = {"c3_full": (c3, 1000, True), "c3_final": (c3, 10000, False), "c5": (c5, 1000, False)}
    lines = [run(k, *cases[k], args.sample, gpu) for k in args.only.split(",")]
    if args.out:
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
