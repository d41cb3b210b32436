#!/usr/bin/env python
"""The oracle's `GravityField::eom` restatement (oracle/nyx_oracle.c, following gravity_field.rs:148-268) against an INDEPENDENT
arbiter: the textbook gradient of the normalised spherical-harmonic potential in spherical coordinates with closed-form associated
Legendre functions at 40 digits (tests/arbiters.py) — VERDICT r01 item 2.  Writes profiles/r02_arbiter_harmonics.json.
--points96 also checks the second arbiter (the Holmes & Featherstone recursion at 50 digits, which the degree-96 tests use against
the oracle) against the closed form on the degree-96 lunar field of tests/high_degree.py, at about 150 s per point; a run with
--points21 0 --points70 0 updates only that entry of the JSON.

    python scripts/arbiter_harmonics.py --points21 200 --points70 16 --points96 1"""
import argparse
import ctypes as C
import json
import multiprocessing as mp
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def oracle_field_accel(packed_c, rb):
    from nyx_b200 import abi
    from oracle import pyoracle

    L = pyoracle.lib()
    L.nyx_oracle_grav_new.restype = C.c_void_p
    L.nyx_oracle_grav_new.argtypes = [C.POINTER(abi.GravityFieldC)]
    L.nyx_oracle_grav_accel.restype = None
    L.nyx_oracle_grav_accel.argtypes = [C.c_void_p, C.c_int64, abi.c_double_p, abi.c_double_p, abi.c_double_p]
    L.nyx_oracle_grav_free.argtypes = [C.c_void_p]
    gf = packed_c.gravity[0]
    h = L.nyx_oracle_grav_new(C.byref(gf))
    scratch = np.zeros((gf.degree + 3) ** 2)
    out = np.zeros(3)
    r = np.ascontiguousarray(rb, dtype=np.float64)
    L.nyx_oracle_grav_accel(h, 0, abi.as_double_p(r), abi.as_double_p(scratch), abi.as_double_p(out))
    L.nyx_oracle_grav_free(h)
    return out


def _case(job):
    import nyx_b200 as nb
    from tests.arbiters import mp_harmonic_accel

    fixture, deg, seed = job
    moon = fixture.startswith("luna")
    gd = nb.GravityFieldData.from_fixture(fixture, deg, deg, nb.IAU_MOON_FRAME if moon else nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    packed = dyn.pack(nb.MOON_J2000 if moon else nb.EARTH_J2000, None)
    gf = packed.c.gravity[0]
    gf.rot.kind = 0
    rng = np.random.default_rng(seed)
    d = rng.normal(size=3)
    rb = d / np.linalg.norm(d) * gf.r_eq_km * rng.uniform(1.02, 1.5)
    got = oracle_field_accel(packed.c, rb)
    want = np.array(mp_harmonic_accel(gd.c_nm, gd.s_nm, deg, deg, gf.mu_km3_s2, gf.r_eq_km, rb))
    return float(np.abs(got - want).max() / np.abs(want).max()), float(np.linalg.norm(rb) / gf.r_eq_km)


def _case96(seed):
    import nyx_b200 as nb
    from tests import high_degree as hd
    from tests.arbiters import mp_harmonic_accel, mp_harmonic_accel_recursion

    gd = hd.field_data("moon")
    gf = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd))).pack(nb.MOON_J2000, None).c.gravity[0]
    rng = np.random.default_rng(seed)
    d = rng.normal(size=3)
    rb = d / np.linalg.norm(d) * gf.r_eq_km * 1.02
    args = (gd.c_nm, gd.s_nm, 96, 96, gf.mu_km3_s2, gf.r_eq_km, rb)
    closed = mp_harmonic_accel(*args, dps=40, as_mpf=True)
    rec = mp_harmonic_accel_recursion(*args, dps=50, as_mpf=True)
    scale = max(abs(v) for v in closed)
    return float(max(abs(a - b) for a, b in zip(closed, rec)) / scale), float(np.linalg.norm(rb) / gf.r_eq_km)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--points21", type=int, default=200)
    p.add_argument("--points70", type=int, default=16)
    p.add_argument("--points96", type=int, default=0)
    p.add_argument("--out", default="profiles/r02_arbiter_harmonics.json")
    a = p.parse_args()
    out = json.loads(Path(a.out).read_text()) if Path(a.out).exists() else {}
    jobs = [("jgm3_70x70", 21, s) for s in range(a.points21)] + [("jgm3_70x70", 70, 1000 + s) for s in range(a.points70)] + \
           [("luna_jggrx_80x80", 70, 2000 + s) for s in range(a.points70)]
    with mp.get_context("fork").Pool(mp.cpu_count()) as pool:
        res = pool.map(_case, jobs, chunksize=1)
        res96 = pool.map(_case96, range(3000, 3000 + a.points96), chunksize=1)
    for name, sl in (("jgm3_21x21", slice(0, a.points21)), ("jgm3_70x70", slice(a.points21, a.points21 + a.points70)),
                     ("grail_70x70", slice(a.points21 + a.points70, None))):
        e = np.array([r[0] for r in res[sl]])
        if e.size == 0:
            continue
        out[name] = {"points": int(e.size), "max_rel_err": float(e.max()), "median_rel_err": float(np.median(e)),
                     "radius_range_r_eq": [float(min(r[1] for r in res[sl])), float(max(r[1] for r in res[sl]))]}
    if res96:
        out["recursion_vs_closed_96x96"] = {
            "points": len(res96), "max_rel_diff": max(r[0] for r in res96), "radius_r_eq": [r[1] for r in res96],
            "field": "lunar 96x96 of tests/high_degree.py", "arbiters": "tests/arbiters.py: mp_harmonic_accel (closed form, 40 digits) "
            "against mp_harmonic_accel_recursion (Holmes & Featherstone forward-column recursion, 50 digits), compared unrounded"}
    out["arbiter"] = "textbook spherical-coordinate gradient, closed-form Legendre functions (mpmath.legenp), 40 digits: tests/arbiters.py"
    out["note"] = "relative to the largest component of the non-central acceleration; the oracle evaluates gravity_field.rs:148-268 in f64"
    txt = json.dumps(out, indent=1)
    print(txt)
    Path(a.out).write_text(txt + "\n")


if __name__ == "__main__":
    main()
