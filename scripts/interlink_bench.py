"""Interlink filter ensemble (nyxb_od_interlink_batch) on the GPU: one JSON line.
  1 000 filters of a 110 km polar lunar orbit (each with its own initial error and noise), tracked every minute for 2 h by one transmitter
  on a Moon-centred NRHO-like orbit (self-contained: no test helpers, no oracle), whose recording comes from nyxb_propagate_batch (range 0.11 m, Doppler 3 mm/s, EKF, msr_size 2),
  lunar 8x8 field.  Both filter kernel families in FAST mode, alternated in one call: the per-thread kernel (forced) and the
  warp-cooperative kernel the dispatch picks for degree >= 8.  Kernel time from CUDA events (Engine.last_kernel_ms), best of --reps;
  measurement updates/s; the GPU name and power limit.
Run from the repository root:  python scripts/interlink_bench.py [--n 1000] [--reps 3]
"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import nyx_b200 as nb  # noqa: E402
from nyx_b200 import abi  # noqa: E402
from nyx_b200.od import MeasurementType as MT  # noqa: E402

S = 10**9
FRAME = nb.MOON_J2000
C_KM_S = 299_792.458
# the reference interlink test's hardware noises (od/noise/link_specific.rs:179-222): Allan deviation 1e-11 over 10 s, T4B chips,
# average S/N0; S band, average C/N0
SIGMA_R = math.sqrt((C_KM_S * 1e-11 * 10.0 / math.sqrt(3.0)) ** 2 + (C_KM_S / (2 * math.pi * 1e6 * math.sqrt(2.0 * 1e5))) ** 2)
SIGMA_D = math.sqrt((C_KM_S * 1e-11) ** 2 + (C_KM_S / (2 * math.pi * 2.2e9 * math.sqrt(2.0 * 10 ** 5.5 * 10.0))) ** 2)


def nrho_orbit():
    rp, ra = 3_300.0, 70_000.0
    return nb.Orbit.keplerian((rp + ra) / 2.0, (ra - rp) / (ra + rp), 90.0, 60.0, 90.0, 160.0, 0, FRAME)


def llo_orbit():
    return nb.Orbit.keplerian(1737.4 + 110.0, 1e-4, 90.0, 0.0, 0.0, 220.0, 0, FRAME)


def lunar_dynamics():
    gd = nb.GravityFieldData.from_fixture("luna_jggrx_80x80", 8, 8, nb.IAU_MOON_FRAME)
    return nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return (out.stdout.strip().split(", ") + ["?"])[:2] if out.returncode == 0 else ("unknown", "unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    n, m = a.n, 120
    dyn = lunar_dynamics()
    rec = nb.Propagator.rk89(dyn, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=nb.MODE_FAST).engine(FRAME, None)
    tx_sc = nb.Spacecraft(orbit=nrho_orbit(), mass=nb.Mass(500.0, 50.0, 0.0))
    rx_sc = nb.Spacecraft(orbit=llo_orbit(), mass=nb.Mass(500.0, 50.0, 0.0))
    end = (m + 1) * 60 * S
    st, cs, ep = nb.pack_spacecraft([tx_sc, rx_sc])
    _, _, _, status, (t_ep, t_st, t_cnt) = rec.propagate_batch(st, cs, ep, end, traj_capacity=end // (10 * S) + 4)
    assert (status == 0).all(), status
    trajs = [nb.Traj(s, t_ep[:int(t_cnt[j]), j].copy(), np.ascontiguousarray(t_st[:, :int(t_cnt[j]), j].T), nm).finalize()
             for j, (s, nm) in enumerate(((tx_sc, "NRHO Tx SC"), (rx_sc, "LLO")))]
    epochs = (np.arange(1, m + 1) * 60 * S).astype(np.int64)
    truth = np.repeat(np.stack([trajs[1].at(int(e)).orbit.to_cartesian_pos_vel() for e in epochs])[:, :, None], n, axis=2)
    devices = {"NRHO": nb.InterlinkTxSpacecraft(trajs[0], [MT.Range, MT.Doppler],
                                                {MT.Range: nb.StochasticNoise(SIGMA_R), MT.Doppler: nb.StochasticNoise(SIGMA_D)})}
    arc = nb.simulate_interlink(epochs, truth, devices, ["NRHO"] * m, FRAME, np.random.default_rng(0))
    rng = np.random.default_rng(1)
    ests = []
    for _ in range(n):
        v = rx_sc.to_vector()
        v[:3] += rng.normal(0, 0.1, 3)
        v[3:6] += rng.normal(0, 1e-4, 3)
        ests.append(nb.KfEstimate.from_diag(rx_sc.with_vector(0, v), [1e-2] * 3 + [1e-8] * 3 + [0.0] * 3))
    out = {"workload": "interlink_llo_nrho", "n": n, "n_msr": m}
    times = {"thread": [], "coop": []}
    sols = {}
    for _ in range(a.reps):
        for fam in ("thread", "coop"):
            prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions.default(), mode=nb.MODE_FAST)
            eng = prop.engine(FRAME, None)
            eng.set_kernel(nb.KERNEL_THREAD if fam == "thread" else nb.KERNEL_AUTO)
            odp = nb.KalmanODProcess(prop, nb.KalmanVariant.ReferenceUpdate, nb.SigmaRejection(), devices, None)
            sols[fam] = odp.process_arcs(ests, arc)
            times[fam].append(eng.last_kernel_ms())
            out[f"kernel_{fam}"] = eng.last_kernel()
    updates = int(((sols["thread"].msr_flags & abi.MSRF_PROCESSED) != 0).sum())
    for fam in times:
        best = min(times[fam])
        out[f"{fam}_ms"] = round(best, 3)
        out[f"{fam}_updates_per_s"] = float(f"{updates / (best * 1e-3):.4g}")
        out[f"{fam}_status_ok"] = int((sols[fam].status == 0).sum())
    out["measurement_updates"] = updates
    out["thread_vs_coop_max_dr_km"] = float(np.abs(sols["thread"].final_state_soa[:3] - sols["coop"].final_state_soa[:3]).max())
    out["gpu"], out["power_limit"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
