"""Angle-tracking filter ensemble (ground stations with azimuth and elevation, nyxb_od_aer_batch) on the GPU: one JSON line per workload.
  n filters (default 1 024) on 26 000 km orbits spread in RAAN and true anomaly, one day of 1-minute tracking by Madrid, Canberra and
  Goldstone in turn (0 deg mask, range 2 m, Doppler 3 mm/s, angles 1 mdeg), EKF, each filter with its own data and initial error.  One
  field shape per filter kernel family the dispatch picks:
    thread  JGM-3 8x8, FAST, per-thread kernel forced        coop  JGM-3 21x21, FAST, warp-cooperative kernel (degree >= 8)
Each line, from CUDA events, alternated in one call: the range/Doppler part of the arc through nyxb_od_ekf_batch against the same arc
through nyxb_od_aer_batch (msr_size 2); the four types at msr_size 2 and at msr_size 1; the four types with the estimate records and
the smoothing kernel.  Also: measurement updates/s, a two-filter STRICT parity sample against the restatement (tests/aer_oracle.py),
the GPU name and power limit.
Run from the repository root:  python scripts/aer_bench.py [--n 1024] [--hours 24] [--reps 2]
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
SIGMA = {MT.Range: 2e-3, MT.Doppler: 3e-6, MT.Azimuth: 1e-3, MT.Elevation: 1e-3}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return (out.stdout.strip().split(", ") + ["?"])[:2] if out.returncode == 0 else ("unknown", "unknown")


def stations(types):
    out = {}
    for name, ctor in (("Madrid", nb.GroundStation.dss65_madrid), ("Canberra", nb.GroundStation.dss34_canberra),
                       ("Goldstone", nb.GroundStation.dss13_goldstone)):
        gs = ctor(0.0, nb.StochasticNoise(SIGMA[MT.Range]), nb.StochasticNoise(SIGMA[MT.Doppler]))
        gs.measurement_types = []
        for t in types:
            gs.with_msr_type(t, nb.StochasticNoise(SIGMA[t]))
        out[name] = gs
    return out


def workload(n, hours, degree, seed=0):
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", degree, degree, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    rng = np.random.default_rng(seed)
    tmpl = [nb.Spacecraft(orbit=nb.Orbit.keplerian(26000.0 + 10 * (i % 7), 0.01, 55.0, (i % 32) * 11.25, 0.0,
                                                   (i // 32) * 360.0 / max(n // 32, 1), 0, frame), mass=nb.Mass(300.0, 0.0, 0.0))
            for i in range(n)]
    m = int(hours * 60)
    epochs = (np.arange(1, m + 1) * 60 * S).astype(np.int64)
    tprop = nb.Propagator.rk89(dyn, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=nb.MODE_STRICT)
    st, cs, ep = nb.pack_spacecraft(tmpl)
    _, _, _, tstat, (t_ep, t_st, t_cnt) = tprop.engine(frame, None).propagate_batch(st, cs, ep, int(epochs[-1]), traj_capacity=m * 6 + 2)
    assert (tstat == 0).all()
    idx = np.searchsorted(t_ep[: t_cnt[0], 0], epochs)
    truth = np.ascontiguousarray(t_st[:, idx, :].transpose(1, 0, 2))
    devs = stations((MT.Range, MT.Doppler, MT.Azimuth, MT.Elevation))
    names = list(devs)
    arc = nb.simulate_tracking(epochs, truth, devs, [names[k % 3] for k in range(m)], frame, None, rng)
    ests = []
    for sc in tmpl:
        v = sc.to_vector()
        v[:3] += rng.normal(0, 0.1, 3)
        v[3:6] += rng.normal(0, 1e-4, 3)
        ests.append(nb.KfEstimate.from_diag(sc.with_vector(0, v), [0.01] * 3 + [1e-8] * 3 + [0.0] * 3))
    return dyn, frame, devs, arc, ests


def run(family, n, hours, reps):
    degree = 8 if family == "thread" else 21
    dyn, frame, devs, arc, ests = workload(n, hours, degree)
    rd_devs = stations((MT.Range, MT.Doppler))
    rd_arc2 = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc.obs[:, :2, :])
    rd_arc4 = nb.TrackingDataArc(arc.epoch_ns, arc.tracker, np.concatenate([arc.obs[:, :2, :], np.full_like(arc.obs[:, 2:, :], np.nan)], 1),
                                 nb.AER_TYPES)
    prop = nb.Propagator.default_dp78(dyn, mode=nb.MODE_FAST)
    eng = prop.engine(frame, None)
    eng.set_kernel(nb.KERNEL_THREAD if family == "thread" else nb.KERNEL_AUTO)
    cases = {  # key: (devices, arc, msr_size, records)
        "rd_ekf_batch": (rd_devs, rd_arc2, 2, False),
        "rd_aer_batch": (rd_devs, rd_arc4, 2, False),
        "aer_m2": (devs, arc, 2, False),
        "aer_m1": (devs, arc, 1, False),
        "aer_m2_rec": (devs, arc, 2, True),
    }
    times = {k: [] for k in cases}
    sols = {}
    for _ in range(reps):
        for key, (dv, a, M, rec) in cases.items():
            odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, None, dv, None, msr_size=M)
            sols[key] = odp.process_arcs(ests, a, estimates_capacity=(2 * len(a) + 2) if rec else None)
            times[key].append(eng.last_kernel_ms())
    for key in cases:
        assert (sols[key].status == 0).all(), (key, np.unique(sols[key].status))
    assert np.array_equal(sols["aer_m2"].final_state_soa, sols["aer_m2_rec"].final_state_soa)
    rd_diff = float(np.abs(sols["rd_ekf_batch"].final_state_soa[:3] - sols["rd_aer_batch"].final_state_soa[:3]).max())
    kernel = "coop" if eng.last_kernel() == nb.KERNEL_COOP else "thread"
    sm = sols["aer_m2_rec"].smooth()
    sm_ms = eng.last_kernel_ms()
    updates = int(((sols["aer_m2"].msr_flags & nb.abi.MSRF_PROCESSED) != 0).sum())
    ms = {k: min(v) for k, v in times.items()}
    # parity sample: two filters on STRICT against the restatement
    from tests import aer_oracle
    sprop = nb.Propagator.default_dp78(dyn, mode=nb.MODE_STRICT)
    sodp = nb.KalmanODProcess(sprop, nb.KalmanVariant.ReferenceUpdate, None, devs, None, msr_size=2)
    ssol = sodp.process_arcs(ests[:2], nb.TrackingDataArc(arc.epoch_ns, arc.tracker, arc.obs[:, :, :2], arc.types))
    names, st_c = sodp.aer_stations_c(frame)
    tracker = np.array([names.index(t) for t in arc.tracker], dtype=np.int32)
    worst = 0.0
    for i in range(2):
        ref = aer_oracle.process_arc(dyn.pack(frame, None).c, sprop.opts.to_c(sprop.method), sodp.config_c(), st_c, arc.epoch_ns, tracker,
                                     np.ascontiguousarray(arc.obs[:, :, i]), ests[i].nominal_state.to_vector(), np.array([300.0, 0.0, 0.0, 0.0]),
                                     0, ests[i].covar)
        worst = max(worst, float(np.abs(ssol.final_state_soa[:3, i] - ref["state"][:3]).max()))
    name, power = gpu_info()
    return dict(workload=f"aer-{family}", kernel=kernel, n=n, measurements=len(arc), degree=degree,
                kernel_ms_rd_ekf_batch=ms["rd_ekf_batch"], kernel_ms_rd_aer_batch=ms["rd_aer_batch"],
                rd_aer_over_ekf=ms["rd_aer_batch"] / ms["rd_ekf_batch"], rd_max_dr_km=rd_diff,
                kernel_ms_aer_m2=ms["aer_m2"], kernel_ms_aer_m1=ms["aer_m1"], m1_over_m2=ms["aer_m1"] / ms["aer_m2"],
                kernel_ms_aer_m2_records=ms["aer_m2_rec"], processed_measurements=updates,
                msr_updates_per_s=updates / (ms["aer_m2"] * 1e-3), smooth_kernel_ms=sm_ms, smooth_ok=int((sm.smoother["status"] == 0).sum()),
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
