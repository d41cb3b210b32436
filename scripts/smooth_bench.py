"""Filter with every estimate recorded, then ODSolution::smooth, on the GPU: one JSON line per workload.
  c5   lunar 70x70 + Earth/Sun point masses + SRP (warp-cooperative filter kernel), n = 1 000 EKFs, 1 day, DSN range + Doppler every
       10 min, max_step 1 min
  leo  JGM-3 8x8 LEO (per-thread filter kernel, FAST, forced), n = 1 024 EKFs, 1 day, DSN range + Doppler every minute
Each line: the filter kernel time without and with recording, alternated in the same call (CUDA events), the records' bytes, the
smoothing kernel time and its fraction of the byte roof at 3.35 TB/s (bytes the kernel must move: every record read once, every
smoothed output written once), the wall time of the smooth() call (which uploads the records again), a parity sample of the smoothed
estimates against the restatement (tests/smooth_oracle.py) run on the GPU filter's own records, the GPU name and power limit.
Run from the repository root:  python scripts/smooth_bench.py [--only c5,leo] [--reps 2]
"""
import argparse
import json
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
HBM_BYTES_PER_S = 3.35e12
REC_BYTES = 1456            # per estimate: epoch, tag, 2 x 9 + 2 x 81 doubles


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True)
    name, power = (out.stdout.strip().split(", ") + ["?"])[:2] if out.returncode == 0 else ("unknown", "unknown")
    return name, power


def devices():
    rn, dn = nb.StochasticNoise(1e-2), nb.StochasticNoise(1e-5)
    return {"Madrid": nb.GroundStation.dss65_madrid(10.0, rn, dn), "Canberra": nb.GroundStation.dss34_canberra(10.0, rn, dn),
            "Goldstone": nb.GroundStation.dss13_goldstone(10.0, rn, dn)}


def c5(n, rng):
    frame = nb.MOON_J2000
    alm = nb.Almanac.synthetic(frame, 0, 3.0, bodies=(EARTH, nb.SUN))
    gd = nb.GravityFieldData.from_fixture("luna_jggrx_80x80", 70, 70, nb.IAU_MOON_FRAME)
    srp = nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)
    dyn = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.new([nb.PointMasses.new([EARTH, nb.SUN]), nb.GravityField.new(gd)]), srp)
    orbit = nb.Orbit.keplerian(1737.4 + 100.0, 0.002, 88.0, 20.0, 10.0, 0.0, 0, frame)
    sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(1018.0, 900.0, 0.0), srp=nb.SRPData(3.9 * 2.7, 0.96))
    return frame, alm, dyn, nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST), sc, 600


def leo(n, rng):
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", 8, 8, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    orbit = nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame)
    sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 0.0, 0.0))
    return frame, None, dyn, nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST), sc, 60


def run(name, builder, n, reps, sample, gpu):
    from tests import smooth_oracle

    rng = np.random.default_rng(0)
    frame, alm, dyn, prop, sc, cadence = builder(n, rng)
    span = 86400 * S
    dev = devices()
    epochs = (np.arange(1, span // (cadence * S) + 1) * cadence * S).astype(np.int64)
    # the truth of every filter is the template; the estimates start dispersed around it
    st1, cs1, ep1 = nb.pack_spacecraft([sc])
    _, _, _, tst, (t_ep, t_st, t_cnt) = nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST).engine(frame, alm).propagate_batch(
        st1, cs1, ep1, int(epochs[-1]), traj_capacity=200_000)
    from nyx_b200.trajectory import Traj
    tr = Traj(sc, t_ep[: t_cnt[0], 0].copy(), np.ascontiguousarray(t_st[:, : t_cnt[0], 0].T)).finalize()
    truth = np.stack([tr.at(int(t)).orbit.to_cartesian_pos_vel() for t in epochs])
    names = list(dev)
    schedule = [names[(k // 30) % 3] for k in range(len(epochs))]
    arc = nb.simulate_tracking(epochs, np.repeat(truth[:, :, None], n, axis=2), dev, schedule, frame, alm, np.random.default_rng(1))
    cov = np.diag([0.1, 0.1, 0.1, 1e-4, 1e-4, 1e-4, 0.0, 0.0, 0.0]) ** 2
    x = nb.MvnSpacecraft.from_spacecraft_cov(sc, cov).sample_vectors(rng, n)
    ests = [nb.KfEstimate(sc.with_vector(0, sc.to_vector() + x[i]), cov) for i in range(n)]
    odp = nb.SpacecraftKalmanOD(prop, nb.KalmanVariant.ReferenceUpdate, nb.SigmaRejection(3.0), dev, alm)
    eng = prop.engine(frame, alm)
    if name == "leo":
        eng.set_kernel(nb.KERNEL_THREAD)          # the per-thread filter kernel (FAST picks the warp kernel from degree 8)
    # capacity from a first recorded run; then plain and recorded runs alternate
    probe = odp.process_arcs(ests, arc, estimates_capacity=0)
    cap = int(probe.records["count"].max())
    times = {"plain": [], "recorded": []}
    sol = None
    for _ in range(reps):
        plain = odp.process_arcs(ests, arc)
        times["plain"].append(eng.last_kernel_ms())
        sol = odp.process_arcs(ests, arc, estimates_capacity=cap)
        times["recorded"].append(eng.last_kernel_ms())
        assert np.array_equal(plain.final_state_soa, sol.final_state_soa) and np.array_equal(plain.covar, sol.covar)
    family = {nb.KERNEL_THREAD: "thread", nb.KERNEL_COOP: "coop"}.get(eng.last_kernel(), str(eng.last_kernel()))
    t0 = time.perf_counter()
    sm = sol.smooth()
    smooth_wall = time.perf_counter() - t0
    smooth_ms = eng.last_kernel_ms()
    counts = np.minimum(sol.records["count"], cap)
    n_est = int(counts.sum())
    ok = sm.smoother["status"] == 0
    # bytes the smoothing kernel must move: per estimate k < l, records k and k+1 (nominal, deviation of both; covariance of both;
    # STM of k+1; epoch and tags) are read, and state / deviation / covariance / ratios / postfit written
    moved = int(((counts - 1) * (8 * (9 + 9 + 9 + 81 + 81 + 1 + 1 + 1 + 9) + 8 * (9 + 9 + 81 + 9 + 2))).clip(0).sum())
    worst = 0.0
    dyn_c = dyn.pack(frame, alm).c
    names_c, st_c = odp.stations_c(frame)
    tracker = np.array([names_c.index(t) for t in arc.tracker], dtype=np.int32)
    for i in range(sample):
        L = int(counts[i])
        stream = [dict(epoch=int(sol.records["epoch"][k, i]), tag=int(sol.records["tag"][k, i]), nominal=sol.records["nominal"][k, :, i].copy(),
                       deviation=sol.records["deviation"][k, :, i].copy(), covar=sol.records["covar"][k, :, i].reshape(9, 9).T.copy(),
                       stm=sol.records["stm"][k, :, i].reshape(9, 9).T.copy()) for k in range(L)]
        filt = dict(prefit=sol.prefit[:, :, i], postfit=sol.postfit[:, :, i], resid_ratio=sol.resid_ratio[:, :, i])
        ref, _, _ = smooth_oracle.smooth(stream, filt, 2, st_c, dyn_c, tracker, np.ascontiguousarray(arc.obs[:, :, i]))
        for k in range(L):
            worst = max(worst, float(np.abs(sm.smoother["state"][k, :3, i] - smooth_oracle.state_of(ref[k])[:3]).max()))
    line = dict(workload=name, n=n, span_s=span / S, msrs=len(epochs), kernel_family=family, capacity=cap, estimates=n_est,
                record_bytes=int(cap) * REC_BYTES * n, filter_kernel_ms=dict(plain=times["plain"], recorded=times["recorded"]),
                recording_overhead=float(np.median(times["recorded"]) / np.median(times["plain"]) - 1.0),
                smooth_kernel_ms=smooth_ms, smooth_bytes=moved, smooth_roof_fraction=moved / HBM_BYTES_PER_S / (smooth_ms * 1e-3),
                smooth_call_wall_s=smooth_wall, smooth_status_ok=int(ok.sum()),
                filter_status_ok=int((sol.status == 0).sum()), parity=dict(sample=sample, max_dr_km_vs_restatement=worst),
                gpu=gpu[0], power_limit=gpu[1])
    print(json.dumps(line), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c5,leo")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sample", type=int, default=2)
    a = ap.parse_args()
    gpu = gpu_info()
    work = {"c5": (c5, 1000), "leo": (leo, 1024)}
    for name in a.only.split(","):
        b, n = work[name]
        run(name, b, n, a.reps, a.sample, gpu)


if __name__ == "__main__":
    main()
