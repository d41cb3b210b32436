"""Position-fix filter ensemble (PositionDevice, nyxb_od_position_batch) on the GPU: one JSON line per workload.
  A constellation: n LEO filters (default 1 024), one day of 1-minute X/Y/Z fixes (sigma 1 m), EKF, each filter with its own fixes
  and initial error.  One field shape per filter kernel family the dispatch picks:
    thread  JGM-3 8x8, FAST, per-thread kernel forced        coop  JGM-3 21x21, FAST, warp-cooperative kernel (degree >= 8)
Each line: filter kernel time by CUDA events for msr_size 3 and msr_size 1 and with the estimate records (alternated in the same call),
measurement updates/s, STM steps/s, the smoothing kernel time, a two-filter parity sample against the restatement
(tests/position_oracle.py) on STRICT, the GPU name and power limit.
Run from the repository root:  python scripts/position_bench.py [--n 1024] [--hours 24] [--reps 2]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import nyx_b200 as nb  # noqa: E402
from nyx_b200.od import MeasurementType as MT  # noqa: E402

S = 10**9


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return (out.stdout.strip().split(", ") + ["?"])[:2] if out.returncode == 0 else ("unknown", "unknown")


def workload(n, hours, degree, seed=0):
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    rng = np.random.default_rng(seed)
    # constellation: 32 planes, satellites spread in RAAN and true anomaly; the truth of each is propagated on the GPU (STRICT)
    tmpl = [nb.Spacecraft(orbit=nb.Orbit.keplerian(7000.0 + 10 * (i % 7), 0.001, 53.0, (i % 32) * 11.25, 0.0, (i // 32) * 360.0 / max(n // 32, 1),
                                                   0, frame), mass=nb.Mass(300.0, 0.0, 0.0)) for i in range(n)]
    m = int(hours * 60)
    epochs = (np.arange(1, m + 1) * 60 * S).astype(np.int64)
    tprop = nb.Propagator.rk89(dyn, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=nb.MODE_STRICT)
    st, cs, ep = nb.pack_spacecraft(tmpl)
    teng = tprop.engine(frame, None)
    _, _, _, tstat, (t_ep, t_st, t_cnt) = teng.propagate_batch(st, cs, ep, int(epochs[-1]), traj_capacity=m * 6 + 2)
    assert (tstat == 0).all()
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    truth = np.ascontiguousarray(t_st[:, idx, :].transpose(1, 0, 2))          # [m][6][n]
    dev = nb.PositionDevice("gnss")
    for t in (MT.X, MT.Y, MT.Z):
        dev.with_noise(t, nb.StochasticNoise(1e-3))
    arc = nb.simulate_position_fixes(epochs, truth, {"gnss": dev}, ["gnss"] * m, rng)
    ests = []
    for sc in tmpl:
        v = sc.to_vector()
        v[:3] += rng.normal(0, 0.1, 3)
        v[3:6] += rng.normal(0, 1e-4, 3)
        ests.append(nb.KfEstimate.from_diag(sc.with_vector(0, v), [0.01] * 3 + [1e-8] * 3 + [0.0] * 3))
    return dyn, frame, dev, arc, ests


def run(family, n, hours, reps):
    degree = 8 if family == "thread" else 21
    dyn, frame, dev, arc, ests = workload(n, hours, degree)
    prop = nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST)
    eng = prop.engine(frame, None)
    eng.set_kernel(nb.KERNEL_THREAD if family == "thread" else nb.KERNEL_AUTO)
    times = {"m3": [], "m1": [], "m3_rec": []}
    sols = {}
    for _ in range(reps):
        for key in times:
            odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, {"gnss": dev}, None, msr_size=1 if key == "m1" else 3)
            sols[key] = odp.process_arcs(ests, arc, estimates_capacity=(len(arc) + 2) if key == "m3_rec" else None)
            times[key].append(eng.last_kernel_ms())
    assert (sols["m3"].status == 0).all(), np.unique(sols["m3"].status)
    assert np.array_equal(sols["m3"].final_state_soa, sols["m3_rec"].final_state_soa)
    kernel = "coop" if eng.last_kernel() == nb.KERNEL_COOP else "thread"
    sm = sols["m3_rec"].smooth()
    sm_ms = eng.last_kernel_ms()
    steps = float(sols["m3"].details["n_steps"].sum())
    ms3 = min(times["m3"])
    # parity sample: two filters on STRICT against the restatement
    from tests import position_oracle
    sprop = nb.Propagator.default_dp78(dyn, mode=nb.MODE_STRICT)
    sodp = nb.KalmanODProcess(sprop, nb.KalmanVariant.ReferenceUpdate, None, {"gnss": dev}, None, msr_size=3)
    sub = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc.obs[:, :, :2], arc.types)
    ssol = sodp.process_arcs(ests[:2], sub)
    _, dev_c = sodp.position_devices_c()
    worst = 0.0
    for i in range(2):
        e = ests[i].nominal_state
        ref = position_oracle.process_arc(dyn.pack(frame, None).c, sprop.opts.to_c(sprop.method), sodp.config_c(), dev_c, arc.epoch_ns,
                                          np.zeros(len(arc), dtype=np.int32), np.ascontiguousarray(arc.obs[:, :, i]), e.to_vector(),
                                          np.array([300.0, 0.0, 0.0, 0.0]), 0, ests[i].covar)
        worst = max(worst, float(np.abs(ssol.final_state_soa[:3, i] - ref["state"][:3]).max()))
    name, power = gpu_info()
    return dict(workload=f"position-{family}", kernel=kernel, n=n, fixes=len(arc), degree=degree, kernel_ms_m3=ms3,
                kernel_ms_m1=min(times["m1"]), m3_over_m1=ms3 / min(times["m1"]), kernel_ms_m3_records=min(times["m3_rec"]),
                recording_overhead=min(times["m3_rec"]) / ms3 - 1.0, msr_updates_per_s=n * len(arc) / (ms3 * 1e-3),
                stm_steps_per_s=steps / (ms3 * 1e-3), smooth_kernel_ms=sm_ms, smooth_ok=int((sm.smoother["status"] == 0).sum()),
                strict_parity_max_dr_km=worst, gpu=name, power_limit=power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--hours", type=float, default=24.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--only", default="thread,coop")
    a = ap.parse_args()
    for fam in a.only.split(","):
        print(json.dumps(run(fam, a.n, a.hours, a.reps)), flush=True)


if __name__ == "__main__":
    main()
