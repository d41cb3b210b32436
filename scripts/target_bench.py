"""Ensemble targeting benchmark (nyxb_target_batch): one JSON line per workload.

  ref  10 000 dispersions of the reference targeter tests' 8 000 km orbit, two-body DP78, SMA target at half a period, per-thread
  c2   10 000 LEO runs on BASELINE C2's dynamics (JGM-3 21x21, RK89), delta-v to SMA + ECC + INC one orbit later, FAST (n (V + 1) =
       40 000 trajectories per launch: the transposed kernel)

Each line reports problems/s, the iteration histogram, the device time of one profiled call split into propagation kernels and the
targeting loop's own kernels (update share), the share of the wall time spent on the host and the per-iteration read-back, the
propagation kernels' time against rounds x the kernel time of a plain nyxb_propagate_batch of the first iteration's n (V + 1) start
states over the same span (later rounds carry fewer problems, so < 1), a STRICT parity sample against the restatement, and the
restatement's own time on the host cores for that sample.  The GPU name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import nyx_b200 as nb  # noqa: E402
from nyx_b200 import abi  # noqa: E402
from tests import target_oracle as T  # noqa: E402

S = 10**9


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def workload(name, n, rng):
    frame = nb.EARTH_J2000
    mu = frame.mu_km3_s2()
    if name == "ref":
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.two_body())
        mk = lambda mode: nb.Propagator.default_dp78(dyn, mode=mode)
        kernel = abi.KERNEL_THREAD
        base = np.array(nb.Orbit.keplerian(8000.0, 0.2, 30.0, 60.0, 60.0, 180.0, 0, frame).to_cartesian_pos_vel())
        span = int(round(math.pi * math.sqrt(8000.0**3 / mu) * S))
        cfg = T.config([(c, 1e-4, 0.0, 0.2, 5.0, -5.0) for c in (3, 4, 5)], [(T.SMA, 8100.0, 1e-3)])
        mode = nb.MODE_FAST
    else:
        gd = nb.GravityFieldData.from_fixture("jgm3_70x70", 21, 21, nb.IAU_EARTH_FRAME)
        dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
        mk = lambda mode: nb.Propagator.default(dyn, mode=mode)
        kernel = abi.KERNEL_AUTO
        base = np.array(nb.Orbit.keplerian(6878.0, 0.01, 51.6, 30.0, 40.0, 0.0, 0, frame).to_cartesian_pos_vel())
        span = int(round(2 * math.pi * math.sqrt(6878.0**3 / mu) * S))
        cfg = T.config([(c, 1e-4, 0.0, 0.2, 5.0, -5.0) for c in (3, 4, 5)], [(T.SMA, 6880.0, 1e-3), (T.ECC, 0.011, 1e-4), (T.INC, 51.62, 1e-3)])
        mode = nb.MODE_FAST
    st = np.zeros((9, n))
    st[:6] = base[:, None] + np.concatenate([rng.normal(0, 1.0, (3, n)), rng.normal(0, 1e-3, (3, n))])
    cs = np.tile(np.array([[100.0], [0.0], [0.0], [0.0]]), (1, n))
    ep = np.zeros(n, dtype=np.int64)
    return mk, kernel, mode, cfg, st, cs, ep, span


def run(name, n, sample, steps):
    rng = np.random.default_rng(1)
    mk, kernel, mode, cfg, st, cs, ep, span = workload(name, n, rng)
    p = mk(mode)
    eng = p.engine(nb.EARTH_J2000, None)
    eng.set_kernel(kernel)
    eng.target_batch(cfg, st[:, :64], cs[:, :64], ep[:64], 0, span)   # warm-up of every shape's tables
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = eng.target_batch(cfg, st, cs, ep, 0, span)
        times.append(time.perf_counter() - t0)
    t_call = float(np.median(times))
    rounds = int(out["iterations"].max()) + 1
    # device time by kernel in one profiled call: propagation kernels against the targeting loop's own (stage / update / init /
    # finish and CUB's compaction); the rest of the wall time is host work and the per-iteration read-back
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.target_batch(cfg, st, cs, ep, 0, span)
    k_tgt = k_cub = k_prop = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if "nyxb_tgt_" in ev.key:
            k_tgt += t
        elif "cub" in ev.key.lower() or "DeviceSelect" in ev.key:
            k_cub += t
        elif "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
            k_prop += t
    k_all = k_tgt + k_cub + k_prop
    # plain nyxb_propagate_batch of the first iteration's launch (n (V + 1) start states) over the same span: kernel time (CUDA events)
    W = cfg.n_vars + 1
    pst, pcs, pep = np.tile(st, (1, W)), np.tile(cs, (1, W)), np.zeros(n * W, dtype=np.int64)
    plain_ms = []
    for _ in range(3):
        _, _, det, _ = eng.propagate_batch(pst, pcs, pep, span)
        plain_ms.append(eng.last_kernel_ms())
    t_plain = float(np.median(plain_ms)) * 1e-3
    # STRICT parity sample and the restatement on the host cores
    ps = mk(nb.MODE_STRICT)
    es = ps.engine(nb.EARTH_J2000, None)
    es.set_kernel(abi.KERNEL_THREAD)
    strict = es.target_batch(cfg, st[:, :sample], cs[:, :sample], ep[:sample], 0, span)
    t0 = time.perf_counter()
    ref = T.target_batch(ps.dynamics.pack(nb.EARTH_J2000, None).c, ps.opts.to_c(ps.method), cfg, st[:, :sample], cs[:, :sample], ep[:sample], 0, span)
    t_host = time.perf_counter() - t0
    ok = ref["status"] == 0
    parity = float(np.abs(strict["correction"][:, ok] - ref["correction"][:, ok]).max() / np.abs(ref["correction"][:, ok]).max()) if ok.any() else None
    hist = {int(k): int(v) for k, v in zip(*np.unique(out["iterations"], return_counts=True))}
    stat = {int(k): int(v) for k, v in zip(*np.unique(out["status"], return_counts=True))}
    gpu, power = gpu_info()
    return {
        "workload": name, "gpu": gpu, "power_limit": power, "n": n, "mode": "FAST", "kernel_family": eng.last_kernel(),
        "call_s": t_call, "problems_per_s": n / t_call, "rounds": rounds, "iteration_histogram": hist, "status_counts": stat,
        "device_s": k_all * 1e-6, "propagation_kernels_s": k_prop * 1e-6,
        "update_kernel_share": (k_tgt + k_cub) / k_all if k_all else None, "compaction_share": k_cub / k_all if k_all else None,
        "host_and_readback_share_of_wall": 1.0 - k_all * 1e-6 / t_call,
        "plain_first_launch_kernel_s": t_plain, "plain_steps_per_s": float(det["n_steps"].sum()) / t_plain,
        "propagation_kernels_over_rounds_x_plain": k_prop * 1e-6 / (t_plain * rounds),
        "strict_parity_sample": sample, "strict_parity_status_equal": bool(np.array_equal(strict["status"], ref["status"])),
        "strict_parity_max_rel_correction": parity, "host_restatement_s": t_host, "host_cores_used": 1, "host_cores": os.cpu_count(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ref,c2")
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--sample", type=int, default=8)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    for w in a.workloads.split(","):
        print(json.dumps(run(w, a.n, a.sample, a.steps)), flush=True)


if __name__ == "__main__":
    main()
