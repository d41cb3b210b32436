#!/usr/bin/env python
"""Small launches of every shared-memory-cooperating kernel, meant to run under compute-sanitizer (SURVEY.md section 5):

    compute-sanitizer --tool racecheck python scripts/sanitize_case.py coop|strict|tx|od|blse
    compute-sanitizer --tool memcheck  python scripts/sanitize_case.py all

Sizes are tiny (the tools slow kernels down ~100x): a few trajectories over a few steps, with rejections and a recording sink."""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import nyx_b200 as nb  # noqa: E402

S = 10**9


def ensemble(n, seed=1):
    frame = nb.EARTH_J2000
    orbit = nb.Orbit.keplerian(6678.0, 0.015, 68.5, 65.2, 75.0, 0.0, 0, frame)
    template = nb.Spacecraft(orbit=orbit, mass=nb.Mass(100.0, 20.0, 0.0))
    mvn = nb.MvnSpacecraft.from_cartesian_std(template, 1.0, 1e-3)
    mc = nb.MonteCarlo(template, mvn, "sanitize", seed=seed)
    return nb.pack_spacecraft(ds.state for _, ds in mc.generate_states(0, n))


def run(which):
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", 12, 12, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    opts = nb.IntegratorOptions(init_step=400 * nb.Unit.Second, tolerance=1e-12)   # the first attempts are rejected
    if which in ("coop", "tx", "thread"):
        st, cs, ep = ensemble(70)
        prop = nb.Propagator.rk89(dyn, opts, mode=nb.MODE_FAST)
        eng = prop.engine(nb.EARTH_J2000, None)
        eng.set_kernel({"coop": nb.KERNEL_COOP, "tx": nb.KERNEL_TRANSPOSED, "thread": nb.KERNEL_THREAD}[which])
        if which == "tx":
            eng.set_tx_tuning(3, 1)   # 3 sets on one CTA (two set contexts): parking and ticket hand-over are exercised
        out = eng.propagate_batch(st, cs, ep, 1500 * S, traj_capacity=40)
        assert (out[3] == 0).all(), out[3]
        print(which, "steps", int(out[2]["n_steps"].sum()), "rejected", int(out[2]["n_rejected"].sum()))
    elif which == "strict":
        st, cs, ep = ensemble(12)
        prop = nb.Propagator.rk89(dyn, opts, mode=nb.MODE_STRICT)
        eng = prop.engine(nb.EARTH_J2000, None)
        eng.set_lanes(8)
        out = eng.propagate_batch(st, cs, ep, 1500 * S, traj_capacity=40)
        assert (out[3] == 0).all()
        print(which, "steps", int(out[2]["n_steps"].sum()))
    elif which == "od":
        sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
        from oracle import pyoracle
        from tests.od_util import leo_od_scenario

        sc = leo_od_scenario(pyoracle, n=3, n_msr=6, seed=5, degree=8)
        sc["prop"].mode = nb.MODE_FAST
        sol = sc["odp"].process_arcs(sc["ests"], sc["arc"], record_estimates=True)
        assert (sol.status == 0).all()
        print(which, "filters", 3, "accepted", int(sol.accepted().sum()))
    elif which == "blse":   # nyxb_k_od_coop<OdBlsJob>: 3 problems, 4 measurements, LM with a rejected step (lambda0 = 1e-12)
        from oracle import pyoracle
        from tests.blse_util import blse_scenario

        sc = blse_scenario(pyoracle, n=3, n_msr=4, cadence_s=30, degree=12, mode=nb.MODE_FAST)
        b = nb.BatchLeastSquares(sc["prop"], sc["devices"], None, solver=nb.BLSSolver.LevenbergMarquardt, max_iterations=3,
                                 lm_lambda_init=1e-12)
        sol = b.estimate_ensemble(sc["guesses"], sc["arc"])
        assert sc["prop"].engine(sc["frame"], None).last_kernel() == nb.KERNEL_COOP and (sol.status == 0).all()
        print(which, "problems", 3, "iterations", sol.iterations.tolist())


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    for w in (["thread", "coop", "strict", "tx", "od", "blse"] if which == "all" else [which]):
        run(w)
