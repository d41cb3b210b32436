"""CPU companion of tests/test_gpu_od_kernels_matrix.py: the matrix can only catch a wrong column count, a wrong model, a wrong
covariance entry or a wrong index if its inputs make them matter.  Checked on the restatements alone."""
import numpy as np
import pytest

from nyx_b200 import abi
from tests import od_kernels_matrix as km
from tests import od_matrix as om

DROPS = [("field", "field"), ("third_body", "point_masses"), ("srp", "srp"), ("lunar", "field"), ("lunar", "point_masses"),
         ("lunar", "srp")]
DROP_SETTING = {"predict": "ekf", "bls": "ne", "position": "m3"}
COV_KEYS = ("P_rr", "P_rv", "P_vr", "P_vv", "P_cr")


def test_shape_grid_covers_every_column_count():
    """Every kernel runs the same shape grid: one to four columns per lane on the warp kernels, and a truncated field (order < degree)
    on each family."""
    coop = [(d, o) for f, _, d, o in km.SHAPE_CASES if f == "FAST-coop"]
    assert {om.coop_columns_per_lane(d, o) for d, o in coop} == {1, 2, 3, 4}
    assert {f for f, _, d, o in km.SHAPE_CASES if o < d} == set(km.FAMILIES)
    assert {f for f, _, d, o in km.SHAPE_CASES if d == 96 and o == 96} == set(km.FAMILIES)
    assert min(d for _, _, d, _ in km.SHAPE_CASES) == 8 and (8, 0) in coop


def test_ragged_size_spans_several_blocks():
    """37 runs: at least two blocks with a partial last one, in both launch geometries (sizes read from the kernel sources), and the
    runs compared with the restatement sit on both sides of every block edge."""
    n = km.RAGGED
    for per_block in (km.per_thread_block(), km.warps_per_cta()):
        blocks = -(-n // per_block)
        assert blocks >= 2 and n % per_block != 0, per_block
        edges = {b * per_block for b in range(1, blocks)} | {b * per_block - 1 for b in range(1, blocks)}
        if per_block == km.per_thread_block():
            assert edges <= set(km.EDGE_RUNS)
    assert km.per_thread_block() == 32 and km.warps_per_cta() == 4
    assert {0, n - 1} <= set(km.EDGE_RUNS) and {3, 4} <= set(km.EDGE_RUNS)
    st, _, _ = km.estimates("field", n)
    assert len({tuple(st[:3, i]) for i in range(n)}) == n                       # no two runs alike


def test_predict_ends_cover_every_chunk_edge():
    x = km.predict_inputs("field", "ckf", "long", om.N_F)
    span = x["end"] - x["ep"]
    assert (span % km.CHUNK == 0).any() and (span < 0).any() and ((span > 0) & (span % km.CHUNK != 0)).sum() >= 2
    assert (x["ep"] % om.S != 0).any() and len(set(x["ep"])) >= 3
    assert np.abs(x["dev0"][:7]).min() > 0.0


def _spanning_runs(kind):
    """The runs a dropped model must move.  A prediction whose end lies before its start maps one 60 s chunk, which the "srp" orbit
    spends in the Earth's shadow: those runs are left out."""
    if kind != "predict":
        return range(om.N_F)
    x = km.predict_inputs("field", "ekf", "long", om.N_F)
    return [i for i in range(om.N_F) if x["end"][i] > x["ep"][i]]


def _per_run(kind, config, setting, drop):
    """Per run: the largest position move and the largest covariance move (per block, relative) when the model is dropped."""
    base = km.restated(kind, config, setting, "long", om.N_F)
    moved = km.restated(kind, config, setting, "long", om.N_F, drop=drop)
    dr, dp = [], []
    for i in _spanning_runs(kind):
        e = km.errors(kind, km._as_got(kind, [moved[i]], (i,), om.N_F), [base[i]], (i,))
        dr.append(e["dr"])
        dp.append(max(e[k] for k in COV_KEYS))
    return np.array(dr), np.array(dp)


@pytest.mark.parametrize("config,drop", DROPS)
@pytest.mark.parametrize("kind", km.KINDS)
def test_every_model_moves_each_kernels_answer(oracle, kind, config, drop):
    """Dropping the model moves every run's states and covariance far beyond the bound they are compared at."""
    setting = DROP_SETTING[kind]
    b = km.bounds(kind, config, setting, "long", om.N_F)
    dr, dp = _per_run(kind, config, setting, drop)
    print(f"{kind} {config} -{drop}: min move dr {dr.min():.2e} (bound {b['dr']:.1e}), covariance {dp.min():.2e} "
          f"(bound {max(b[k] for k in COV_KEYS):.1e})")
    # The Moon-centred arc's oracle spread is 20 x the Earth arcs' and lunar SRP is weak: 1e2 x there (as tests/test_od_matrix_inputs.py)
    factor = 1e2 if config == "lunar" else 1e3
    assert dr.min() > factor * b["dr"], (kind, config, drop, dr.min(), b["dr"])
    assert dp.min() > factor * max(b[k] for k in COV_KEYS), (kind, config, drop, dp.min())


@pytest.mark.parametrize("config", ["srp", "lunar"])
def test_cr_entries_of_predicted_covariance_are_live(oracle, config):
    """The Cr row and column of every predicted covariance are nonzero, and the SRP Cr partial moves them far beyond their bound."""
    base = km.restated("predict", config, "ekf", "long", om.N_F)
    nosrp = km.restated("predict", config, "ekf", "long", om.N_F, drop="srp")
    bound = km.bounds("predict", config, "ekf", "long", om.N_F)["P_cr"]
    for i in _spanning_runs("predict"):
        r, q = base[i], nosrp[i]
        assert np.abs(r["rec_covar"][1:, :6, 6]).min() > 0.0
        cr = np.abs(r["covar"][:6, 6] - q["covar"][:6, 6]).max() / np.abs(r["covar"][:6, 6]).max()
        assert cr > 1e3 * bound, (config, cr, bound)


@pytest.mark.parametrize("kind", km.KINDS)
def test_compared_covariance_entries_are_not_negligible(oracle, kind):
    """The position-velocity correlations (above 1e-2) and the Cr correlations (above 1e-3) of every compared covariance are far from zero, so a relative bound
    per block sees them."""
    setting = DROP_SETTING[kind]
    for config in ("srp", "lunar"):
        for r in km.restated(kind, config, setting, "long", om.N_F):
            P = {"predict": lambda: r["rec_covar"], "bls": lambda: r["covar"][None],
                 "position": lambda: np.array([s["covar"] for s in r["records"]])}[kind]()
            d = np.sqrt(np.einsum("kii->ki", P)[:, :7])
            corr = P[:, :7, :7] / (d[:, :, None] * d[:, None, :])
            assert np.abs(corr[:, :3, 3:6]).max() > 1e-2 and np.abs(corr[:, :6, 6]).max() > 1e-3, (kind, config)


@pytest.mark.parametrize("setting", ["m3", "m1"])
def test_position_arcs_produce_every_flag(oracle, setting):
    refs = km.restated("position", "srp", setting, "long", om.N_F)
    flags = np.stack([r["flags"] for r in refs], axis=-1)
    sched = km.position_schedule(om.N_MSR)
    two = [k for k, s in enumerate(sched) if s == "gnss2"]
    assert (flags & abi.MSRF_PROCESSED).any(axis=0).all()
    assert flags[km.ABSENT_FIX] == abi.MSRF_ABSENT
    assert (flags[km.UNKNOWN_FIX] == 0).all()                                 # unknown tracker: nothing happens
    if setting == "m3":
        assert (flags[two] == 0).all()                                        # left out of the devices: unknown too
    else:
        assert (flags[two] & abi.MSRF_PROCESSED).all()
    k, q, f = km.PARTIAL_FIX
    assert flags[k, f] & abi.MSRF_PROCESSED and np.isnan(km.position_inputs("srp", setting, "long", om.N_F)["obs"][k, q, f])
    assert all(r["status"] == 0 for r in refs)
    assert all(len(r["records"]) >= 2 for r in refs)
