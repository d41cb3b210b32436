"""Parity of angle tracking (nyxb_od_aer_batch) and its smoother (nyxb_od_aer_smooth_batch) with their restatement
(tests/aer_oracle.process_arc and smooth_restated), at fixed step, across the filter matrix of tests/od_matrix.py.  Inputs:
tests/aer_matrix.py.

Families, each forced explicitly and checked with `last_kernel()`:
  STRICT       per-thread kernel nyxb_k_od<OdFilterJob<DevAerStation, true>>, STRICT arithmetic
  FAST-thread  the same kernel, FAST arithmetic                                     set_kernel(KERNEL_THREAD)
  FAST-coop    warp kernel nyxb_k_od_coop<OdFilterJob<DevAerStation, true>>, the FAST default at degree >= 8

Cases: both settings ("m2": EKF at msr_size 2 with rejection and SNC; "m1": CKF at msr_size 1, list order unlike the type values) on
every configuration at 21x21, Moon-centred with Earth stations the Moon hides included; the field shapes of od_kernels_matrix.SHAPE_CASES
(1 to 4 columns per lane, order 0, truncated orders, degree 96) on "m2"; a ragged ensemble of 37 runs, each equal bit for bit to the
same run launched alone (records and smoother outputs included), the runs at the block edges against the restatement; and the
"edges" arc: the azimuth cut at 0 / 360 (a straddling observation REJECTED under "m2"), elevations 1e-3 deg on either side of a mask,
a pass at 89.9 deg and a line of sight along the integration frame's -Z.

Exactly equal: status, final epochs, step counts, msr_flags (REJECTED and NOT_VISIBLE patterns), record counts, tags and epochs, and
the NaN pattern of every per-measurement output.  Within bounds: states, the CKF deviation, covariances per 3x3 block and on the Cr
row and column, recorded STMs, residual ratios, and prefit and postfit residuals per unit of the slot's type (km, km/s, deg).  The
bound of each quantity is 10 x the spread of the restatement against its two self-probes on the same case, with the floors of
aer_matrix.FLOORS (the degree floor: four ulp of 360).  The smoother runs on each family's own records against smooth_restated with the
configuration's dynamics (the station on the Earth seen from the Moon-centred frame), held to aer_matrix.SMOOTH_BOUNDS.

Each case prints an AERMATRIX line with the ratio of every difference to the restatement's spread.  Measured on an H100 80GB HBM3
(SXM, 700 W power limit), the largest ratio per family and quantity over the 57 cases (the bound is 10; the smoother's entries are
shares of their absolute bounds):

               dr   dv   Cr   state_dev  P_rr P_rv P_vr P_vv P_cr  STM     ratio  prefit km/km_s/deg  postfit km/km_s/deg
  STRICT       2.6  2.6  1.8  2.5        2.4  2.2  2.2  2.0  4.7   0.0037  2.3    1.9 / 1.5 / 2.0     1.1 / 0.62 / 1.9
  FAST-thread  2.7  2.3  2.1  2.1        4.1  1.5  1.5  1.8  3.2   0.0037  1.9    2.0 / 2.7 / 2.0     1.5 / 2.3 / 1.9
  FAST-coop    2.7  2.3  2.7  2.1        4.0  3.7  3.8  2.0  3.2   0.0037  2.0    2.0 / 2.7 / 2.2     2.0 / 2.3 / 2.2
The smoother, as a share of its bound: state 0.011, covariance 2e-9, postfit 0.18 (km), 0.40 (km/s), 0.22 (deg).  The 37-run
ensembles equal their single-run launches bit for bit on every family.  This file and tests/test_gpu_aer.py take 2.3 min together on
that card, most of it in the restatements.

Each of four one-line mutations of nyxb_od_device.cuh fails this file:
  - the elevation row with r^2 = dx^2 + dy^2 + dz^2 instead of (sqrt(sum))^2: test_geometry_edges under "m2" on "field" and "srp", on
    every family, and nowhere else (the polar window's elevation decides its update there);
  - the Moon's line-of-sight test dropped from od_window_setup: test_configurations on "lunar", both settings, every family;
  - AerTrk::ratio_slot back to the ground station's (M == 1) ? wno : 0: every "m2" case (configurations, field shapes, edges), every
    family;
  - the + 360 of the azimuth mapping removed: every case of test_configurations and test_geometry_edges and the lunar field shapes,
    every family (a negative azimuth comes out of every western pass, not only at the cut)."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import aer_matrix as am
from tests import aer_oracle as ao
from tests import od_kernels_matrix as km
from tests import od_matrix as om

pytestmark = pytest.mark.gpu

CONFIG_CASES = [(s, c) for s in am.SETTINGS for c in om.CONFIGS]
EDGE_CASES = [(s, c) for s in am.SETTINGS for c in ("field", "srp")]
SHAPE_SETTING = "m2"
RAGGED_SETTING = "m1"


def _kernel(family):
    return nb.KERNEL_COOP if family == "FAST-coop" else nb.KERNEL_THREAD


def check(family, config, setting, span="long", n=om.N_F, degree=21, order=None, runs=None):
    """Run the batch and its smoother on `family`, compare the runs in `runs` (default all) with the restatement; returns the outputs."""
    order = degree if order is None else order
    got, kernel = am.run(family, config, setting, span, n, degree, order)
    assert kernel == _kernel(family), (family, kernel)
    runs = tuple(range(n)) if runs is None else runs
    refs = am.restated(config, setting, span, n, degree, order, runs)
    x = am.inputs(config, setting, span, n, degree, order)
    tag = f"{family} {am.case_id(config, degree, order, setting, span, n)}"
    assert (np.array([r["status"] for r in refs]) == 0).any(), tag            # the case does something
    bad = km.exact_mismatches("position", got, refs, runs)
    err = am.errors(got, refs, runs, am.slot_units(x))
    bnd = am.bounds(config, setting, span, n, degree, order, runs)
    err.update(smoother_errors(got, x, config, degree, order, runs))
    bnd.update(am.SMOOTH_BOUNDS)
    ratios = {k: err[k] / (bnd[k] / (om.SPREAD_FACTOR if k in am.FLOORS else 1.0)) for k in err}
    worst = max(err, key=lambda k: err[k] / bnd[k])
    print(f"AERMATRIX {tag} worst={worst} ratio_to_spread=" + " ".join(f"{k}={v:.2g}" for k, v in ratios.items())
          + " abs=" + " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    assert not bad, (tag, bad[:5])
    over = {k: (err[k], bnd[k]) for k in err if not err[k] <= bnd[k]}
    assert not over, (tag, over)
    return got


def smoother_errors(got, x, config, degree, order, runs):
    """The smoother against ODSolution::smooth restated from the GPU's own records (filters with status 0), postfits per unit."""
    sm, rec = got["smooth"], got["records"]
    units = am.slot_units(x)
    dyn = am.packed(config, degree, order)
    e = {"sm_dr": 0.0, "sm_P": 0.0, "sm_postfit_km": 0.0, "sm_postfit_km_s": 0.0, "sm_postfit_deg": 0.0}
    for i in runs:
        if got["status"][i] != 0:
            assert sm["status"][i] != 0, i
            continue
        assert sm["status"][i] == 0, i
        want = ao.smooth_restated(rec, i, x["st_c"], dyn.c, x["M"], x["obs"], x["tracker"])
        assert len(want) == int(rec["count"][i]) - 1
        for k, (ys, Ps, post) in enumerate(want):
            e["sm_dr"] = max(e["sm_dr"], float(np.abs(sm["state"][k, :3, i] - ys[:3]).max()))
            e["sm_P"] = max(e["sm_P"], max(km.cov_errors(sm["covar"][k, :, i].reshape(9, 9).T, Ps).values()))
            g = sm["postfit"][k, :, i]
            assert np.array_equal(np.isnan(g), np.isnan(post)), (i, k, g, post)
            tg = int(rec["tag"][k + 1, i])
            if tg >= 0:
                d = np.abs(g - post)
                for u in ("km", "km_s", "deg"):
                    sel = units[abi.od_pos_tag_fields(tg)[0]] == u
                    e[f"sm_postfit_{u}"] = max(e[f"sm_postfit_{u}"], float(np.nanmax(d[sel], initial=0.0)))
    return e


# ---- every configuration at 21x21
@pytest.mark.parametrize("family", km.FAMILIES)
@pytest.mark.parametrize("setting,config", CONFIG_CASES, ids=[f"{s}-{c}" for s, c in CONFIG_CASES])
def test_configurations(oracle, setting, config, family):
    got = check(family, config, setting)
    flags = got["flags"]
    assert (flags & abi.MSRF_PROCESSED).any()
    if setting == "m2":
        assert (flags & abi.MSRF_REJECTED).any()
    if config == "lunar" or setting == "m2":
        assert (flags & abi.MSRF_NOT_VISIBLE).any()


# ---- field shapes
@pytest.mark.parametrize("family,config,degree,order", km.SHAPE_CASES, ids=[f"{f}-{c}-{d}x{o}" for f, c, d, o in km.SHAPE_CASES])
def test_field_shapes(oracle, family, config, degree, order):
    check(family, config, SHAPE_SETTING, "short", degree=degree, order=order)


# ---- an ensemble spanning several blocks
def _same_bits(batch, alone, i):
    """Every output of run i in the batch equals that of the run launched alone (records and smoother included), bit for bit."""
    def eq(a, b):
        return np.array_equal(np.ascontiguousarray(np.atleast_1d(a)).view(np.uint8), np.ascontiguousarray(np.atleast_1d(b)).view(np.uint8))

    bad = [k for k in ("status", "epoch", "n_steps", "state", "dev", "flags", "prefit", "postfit", "ratio")
           if not eq(np.asarray(batch[k])[..., i], np.asarray(alone[k])[..., 0])]
    if not eq(batch["covar"][i], alone["covar"][0]):
        bad.append("covar")
    L = int(batch["records"]["count"][i])
    if L != int(alone["records"]["count"][0]):
        bad.append("records.count")
    for k in ("epoch", "tag", "nominal", "deviation", "covar", "stm"):
        if not eq(batch["records"][k][:L, ..., i], alone["records"][k][:L, ..., 0]):
            bad.append(f"records.{k}")
    if not eq(batch["smooth"]["status"][i], alone["smooth"]["status"][0]):
        bad.append("smooth.status")
    for k in ("state", "deviation", "covar", "fs_ratio", "postfit"):
        if not eq(batch["smooth"][k][: L - 1, :, i], alone["smooth"][k][: L - 1, :, 0]):
            bad.append(f"smooth.{k}")
    return bad


@pytest.mark.parametrize("family", km.FAMILIES)
def test_ragged_ensemble(oracle, family):
    """37 runs: each equals its own launch bit for bit; the runs at the block edges match the restatement.  The smoother's (k, i) grid
    of records x filters is not a multiple of its block."""
    n = km.RAGGED
    batch = check(family, "field", RAGGED_SETTING, "short", n, runs=km.EDGE_RUNS)
    assert (batch["records"]["count"] >= 2).all()
    assert (batch["records"]["epoch"].shape[0] * n) % km.smooth_block() != 0
    bad = {}
    for i in range(n):
        alone, kernel = am.run(family, "field", RAGGED_SETTING, "short", n, only=i)
        assert kernel == _kernel(family)
        b = _same_bits(batch, alone, i)
        if b:
            bad[i] = b
    assert not bad, bad


# ---- the geometry edges
@pytest.mark.parametrize("family", km.FAMILIES)
@pytest.mark.parametrize("setting,config", EDGE_CASES, ids=[f"{s}-{c}" for s, c in EDGE_CASES])
def test_geometry_edges(oracle, setting, config, family):
    got = check(family, config, setting, "edges")
    _, epochs, sched, k_s = am.edge_geometry(config)
    assert (got["status"] == 0).all()
    k_mask = [k for k, s in enumerate(sched) if s == "Mask"]
    assert (got["flags"][k_mask[0]] == abi.MSRF_NOT_VISIBLE).all() and (got["flags"][k_mask[1]] & abi.MSRF_PROCESSED).all()
    if setting == "m2":
        assert (got["flags"][k_s] & abi.MSRF_REJECTED).all()                         # the straddling azimuth
        assert (np.abs(got["prefit"][k_s, 2] - 360.0) < 0.01).all()
    else:
        assert not (got["flags"] & abi.MSRF_REJECTED).any()
