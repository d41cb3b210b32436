"""Parity of covariance prediction (nyxb_od_predict_batch), batch least squares (nyxb_od_bls_batch / _evaluate_batch) and the
position-fix filter and smoother (nyxb_od_position_batch, nyxb_od_position_smooth_batch) with their restatements
(tests/predict_oracle.py, tests/blse_oracle.py, tests/position_oracle.py and tests/test_gpu_position._smooth_restated), at fixed step,
across the filter matrix of tests/od_matrix.py.  Inputs: tests/od_kernels_matrix.py.

Families, each forced explicitly and checked with `last_kernel()`:
  STRICT       per-thread kernels (nyxb_k_od<Job> of the prediction, BLS and position-fix jobs), STRICT arithmetic
  FAST-thread  the same kernels, FAST arithmetic                          set_kernel(KERNEL_THREAD)
  FAST-coop    warp kernels (nyxb_k_od_coop<Job> of the same jobs), the FAST default at degree >= 8

Cases: every configuration at 21x21 (predict EKF and CKF, BLS normal equations and Levenberg-Marquardt on "srp", the position filter
at msr_size 3 and 1); the field shapes where the warp kernels' column deal switches (1, 2, 3 and 4 columns per lane, order 0 and
truncated orders, degree 70 to 96), with 96x96 and a truncated field on the per-thread families; and a ragged ensemble of 37 runs
(two per-thread blocks, ten CTAs, the last holding one warp), where every run of the batch must equal the same run launched alone,
bit for bit, and the runs at the block edges must match the restatement.

Exactly equal: status, final epochs, step counts, record counts and epochs, msr_flags, BLS iterations and convergence flags, the Cr
and mass entries of predicted states, and the NaN pattern of every per-measurement output.  Within bounds: states (km, km/s), the
CKF deviation, covariances per 3x3 block and on the Cr row and column relative to the largest entry of that block, recorded STMs,
residuals, residual ratios and RMS values.  The bound of each quantity is 10 x the spread of the restatement against its two
self-probes (the C oracle's FMA build, and numpy products summed in reverse order) on the same case, with the floors of
od_kernels_matrix.FLOORS.  The smoother runs on the GPU's own records, so it is held to tests/test_gpu_position.py's bounds, tightened where the
measurements allow (od_kernels_matrix.SMOOTH_BOUNDS).

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), largest ratio of the GPU difference to the restatement's spread (the bound
is 10) per family and quantity, over every case of this file:

  predict      dr    dv    state_dev  P_rr  P_rv  P_vr  P_vv  P_cr
  STRICT       0.094 0.099 0.0011     0.17  0.20  0.22  0.25  0.22
  FAST-thread  1.3   1.2   0.0043     0.73  1.1   1.2   1.7   0.75
  FAST-coop    1.3   1.2   0.0043     0.73  1.1   1.2   1.7   0.75
  bls          dr    dv    Cr    rms   corr  evaluate  P_rr  P_rv  P_vr  P_vv  P_cr
  STRICT       0.97  1.4   1.2   2.5   2.0   0.94      1.1   0.99  0.99  0.97  1.2
  FAST-thread  1.6   2.6   3.6   8.2   1.2   3.0       1.5   1.5   1.5   1.5   2.3
  FAST-coop    1.8   2.9   3.6   8.2   1.8   3.0       1.8   1.9   1.9   1.8   1.9
  position     dr    dv    Cr     state_dev  P_rr P_rv P_vr P_vv P_cr  STM      ratio prefit postfit
  STRICT       0.052 0.081 0.0009 0.035      1.1  1.1  1.1  1.1  1.4   0.0001   0.081 0.078  0.046
  FAST-thread  1.3   1.2   1.0    1.6        1.1  1.1  1.1  1.1  1.6   0.0004   1.5   1.4    1.2
  FAST-coop    1.3   1.7   2.6    1.6        1.1  1.1  1.1  1.1  1.6   0.0004   1.5   1.5    1.2
The smoother, as a share of its bound: state 0.045 (4.5e-13 km), covariance 0.32, postfit 0.045.  The 37-run ensembles equal their
single-run launches bit for bit on every family.  The whole file takes about 3.2 min on that card, most of it in the restatements.
Each of three one-line arithmetic mutations of the kernels fails this file:
  - the lane's fourth column left out of the Z sums of grav_gradient_coop: test_field_shapes on FAST-coop at lunar 96x96, for
    predict, BLS and position, and nowhere else;
  - the sign of the SRP Cr partial flipped in the dual right-hand side: every predict and position case of test_configurations on
    "srp" and "lunar", on every family;
  - the Legendre recursion factor b scaled by 1 + 1e-3 above degree 80 (nyxb_api.cu): every lunar case of test_field_shapes from
    80x80 (whose column recursion reads row 81) to 96x96, on every family and kind."""
import numpy as np
import pytest

import nyx_b200 as nb
from tests import od_kernels_matrix as km
from tests import od_matrix as om

pytestmark = pytest.mark.gpu

CONFIG_CASES = ([("predict", s, c) for s in ("ekf", "ckf") for c in om.CONFIGS] + [("bls", "ne", c) for c in om.CONFIGS]
                + [("bls", "lm", "srp")] + [("position", s, c) for s in ("m3", "m1") for c in om.CONFIGS])
SHAPE_SETTING = {"predict": "ckf", "bls": "ne", "position": "m3"}
RAGGED_SETTING = {"predict": "ckf", "bls": "ne", "position": "m1"}


def _kernel(family):
    return nb.KERNEL_COOP if family == "FAST-coop" else nb.KERNEL_THREAD


def check(kind, family, config, setting, span="long", n=om.N_F, degree=21, order=None, runs=None):
    """Run the batch on `family`, compare the runs in `runs` (default all) with the restatement; returns the GPU outputs."""
    order = degree if order is None else order
    got, kernel = km.run(kind, family, config, setting, span, n, degree, order)
    assert kernel == _kernel(family), (family, kernel)
    runs = tuple(range(n)) if runs is None else runs
    refs = km.restated(kind, config, setting, span, n, degree, order, runs)
    tag = f"{family} {km.case_id(kind, config, degree, order, setting, span, n)}"
    assert (np.array([r["status"] for r in refs]) == 0).any(), tag            # the case does something
    bad = km.exact_mismatches(kind, got, refs, runs)
    err = km.errors(kind, got, refs, runs)
    bnd = km.bounds(kind, config, setting, span, n, degree, order, runs)
    if kind == "position":
        sm = smoother_errors(got, kind, config, setting, span, n, degree, order, runs)
        err.update(sm)
        bnd.update(km.SMOOTH_BOUNDS)
    ratios = {k: err[k] / (bnd[k] / (om.SPREAD_FACTOR if k in km.FLOORS else 1.0)) for k in err}
    worst = max(err, key=lambda k: err[k] / bnd[k])
    print(f"ODKMATRIX {tag} worst={worst} ratio_to_spread=" + " ".join(f"{k}={v:.2g}" for k, v in ratios.items())
          + " abs=" + " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    assert not bad, (tag, bad[:5])
    over = {k: (err[k], bnd[k]) for k in err if not err[k] <= bnd[k]}
    assert not over, (tag, over)
    return got


def smoother_errors(got, kind, config, setting, span, n, degree, order, runs):
    """The smoother against ODSolution::smooth restated from the GPU's own records (filters with status 0)."""
    from tests.test_gpu_position import _smooth_restated

    x = km.position_inputs(config, setting, span, n, degree, order)
    sm, rec = got["smooth"], got["records"]
    e = {"sm_dr": 0.0, "sm_P": 0.0, "sm_postfit_km": 0.0}
    for i in runs:
        if got["status"][i] != 0:
            assert sm["status"][i] != 0, i
            continue
        assert sm["status"][i] == 0, i
        want = _smooth_restated(rec, i, x["dev_c"], x["M"], x["obs"], x["tracker"])
        assert len(want) == int(rec["count"][i]) - 1
        for k, (ys, Ps, post) in enumerate(want):
            e["sm_dr"] = max(e["sm_dr"], float(np.abs(sm["state"][k, :3, i] - ys[:3]).max()))
            e["sm_P"] = max(e["sm_P"], max(km.cov_errors(sm["covar"][k, :, i].reshape(9, 9).T, Ps).values()))
            g = sm["postfit"][k, :, i]
            assert np.array_equal(np.isnan(g), np.isnan(post)), (i, k, g, post)
            e["sm_postfit_km"] = max(e["sm_postfit_km"], float(np.nanmax(np.abs(g - post), initial=0.0)))
    return e


# ---- every configuration at 21x21
@pytest.mark.parametrize("family", km.FAMILIES)
@pytest.mark.parametrize("kind,setting,config", CONFIG_CASES, ids=[f"{k}-{s}-{c}" for k, s, c in CONFIG_CASES])
def test_configurations(oracle, kind, setting, config, family):
    got = check(kind, family, config, setting)
    if kind == "predict" and config in ("srp", "lunar"):
        assert np.abs(got["covar"][:, :6, 6]).min() > 0.0                 # the Cr column is live
    if kind == "position":
        assert (got["status"] == 0).all() and (got["smooth"]["status"] == 0).all()


# ---- field shapes
@pytest.mark.parametrize("family,config,degree,order", km.SHAPE_CASES, ids=[f"{f}-{c}-{d}x{o}" for f, c, d, o in km.SHAPE_CASES])
@pytest.mark.parametrize("kind", km.KINDS)
def test_field_shapes(oracle, kind, family, config, degree, order):
    check(kind, family, config, SHAPE_SETTING[kind], "short", degree=degree, order=order)


# ---- an ensemble spanning several blocks
def _same_bits(kind, batch, alone, i):
    """Every output of run i in the batch equals that of the run launched alone (records included), bit for bit."""
    def eq(a, b):
        return np.array_equal(np.ascontiguousarray(np.atleast_1d(a)).view(np.uint8), np.ascontiguousarray(np.atleast_1d(b)).view(np.uint8))

    keys = {"predict": ("status", "epoch", "n_steps", "state", "dev", "count"),
            "bls": ("status", "epoch", "iterations", "converged", "final_rms", "final_corr_pos_km", "n_steps", "state", "eval_rms",
                    "eval_status"),
            "position": ("status", "epoch", "n_steps", "state", "dev", "flags", "prefit", "postfit", "ratio")}[kind]
    bad = [k for k in keys if not eq(np.asarray(batch[k])[..., i], np.asarray(alone[k])[..., 0])]
    if not eq(batch["covar"][i], alone["covar"][0]):
        bad.append("covar")
    if kind == "predict":
        K = int(batch["count"][i])
        for k in ("rec_state", "rec_covar"):
            if not eq(batch[k][:K, :, i], alone[k][:K, :, 0]):
                bad.append(k)
    if kind == "position":
        L = int(batch["records"]["count"][i])
        for k in ("epoch", "tag", "nominal", "deviation", "covar", "stm"):
            if not eq(batch["records"][k][:L, ..., i], alone["records"][k][:L, ..., 0]):
                bad.append(f"records.{k}")
        for k in ("status",):
            if not eq(batch["smooth"][k][i], alone["smooth"][k][0]):
                bad.append(f"smooth.{k}")
        for k in ("state", "deviation", "covar", "fs_ratio", "postfit"):
            if not eq(batch["smooth"][k][: L - 1, :, i], alone["smooth"][k][: L - 1, :, 0]):
                bad.append(f"smooth.{k}")
    return bad


@pytest.mark.parametrize("family", km.FAMILIES)
@pytest.mark.parametrize("kind", km.KINDS)
def test_ragged_ensemble(oracle, kind, family):
    """37 runs: each equals its own launch bit for bit; the runs at the block edges match the restatement.  For the smoother, the
    (k, i) grid of records x filters is not a multiple of its block."""
    setting, n = RAGGED_SETTING[kind], km.RAGGED
    batch = check(kind, family, "field", setting, "short", n, runs=km.EDGE_RUNS)
    if kind == "position":
        assert (batch["records"]["count"] >= 2).all()
        assert (batch["records"]["epoch"].shape[0] * n) % km.smooth_block() != 0
    bad = {}
    for i in range(n):
        alone, kernel = km.run(kind, family, "field", setting, "short", n, only=i)
        assert kernel == _kernel(family)
        b = _same_bits(kind, batch, alone, i)
        if b:
            bad[i] = b
    assert not bad, bad
