"""CPU companion of tests/test_gpu_aer_matrix.py: the matrix can only catch a wrong model, a wrong slot, a wrong visibility decision
or a wrong angle row if its inputs make them matter.  Checked on the restatement alone."""
import numpy as np
import pytest

from nyx_b200 import abi
from tests import aer_matrix as am
from tests import aer_oracle as ao
from tests import od_kernels_matrix as km
from tests import od_matrix as om

DROPS = [("field", "field"), ("third_body", "point_masses"), ("srp", "srp"), ("lunar", "field"), ("lunar", "point_masses"),
         ("lunar", "srp")]
COV_KEYS = ("P_rr", "P_rv", "P_vr", "P_vv", "P_cr")


def _flags(config, setting, span="long", **kw):
    return np.stack([r["flags"] for r in am.restated(config, setting, span, om.N_F, **kw)], axis=-1)


@pytest.mark.parametrize("config,drop", DROPS)
@pytest.mark.parametrize("setting", am.SETTINGS)
def test_every_model_moves_each_run(oracle, setting, config, drop):
    """Dropping the model moves every run's states and covariance far beyond the bound they are compared at."""
    b = am.bounds(config, setting, "long", om.N_F)
    base = am.restated(config, setting, "long", om.N_F)
    moved = am.restated(config, setting, "long", om.N_F, drop=drop)
    dr, dp = [], []
    for i in range(om.N_F):
        e = km.errors("position", km._as_got("position", [moved[i]], (i,), om.N_F), [base[i]], (i,))
        dr.append(e["dr"])
        dp.append(max(e[k] for k in COV_KEYS))
    dr, dp = np.array(dr), np.array(dp)
    print(f"aer {setting} {config} -{drop}: min move dr {dr.min():.2e} (bound {b['dr']:.1e}), covariance {dp.min():.2e} "
          f"(bound {max(b[k] for k in COV_KEYS):.1e})")
    factor = 1e2 if config == "lunar" else 1e3          # as tests/test_od_kernels_matrix_inputs.py
    assert dr.min() > factor * b["dr"], (setting, config, drop, dr.min(), b["dr"])
    assert dp.min() > factor * max(b[k] for k in COV_KEYS), (setting, config, drop, dp.min())


@pytest.mark.parametrize("setting", am.SETTINGS)
def test_arcs_produce_every_outcome(oracle, setting):
    """Processed, rejected (the blunder, under "m2"), not visible by the mask ("m2" Goldstone) and by the Moon ("lunar": the flags
    change when the line-of-sight test is switched off), absent, an unknown tracker, and the window layouts of the setting."""
    flags = _flags("srp", setting)
    sched = am.schedule(om.N_MSR)
    gold = [k for k, s in enumerate(sched) if s == "Goldstone"]
    assert (flags & abi.MSRF_PROCESSED).any(axis=0).all()
    assert flags[am.ABSENT_MSR] == abi.MSRF_ABSENT
    assert (flags[am.UNKNOWN_MSR] == 0).all()
    k, f = am.ABSENT_ANGLE
    assert flags[k, f] & abi.MSRF_PROCESSED and np.isnan(am.inputs("srp", setting, "long", om.N_F)["obs"][k, am.EL, f])
    k, f = am.BLUNDER
    if setting == "m2":
        assert flags[k, f] == abi.MSRF_PROCESSED | abi.MSRF_REJECTED
        assert ((flags[gold] & abi.MSRF_NOT_VISIBLE) != 0).sum(axis=0).min() >= 3       # below the mask
    else:
        assert flags[k, f] == abi.MSRF_PROCESSED and not (flags & abi.MSRF_REJECTED).any()
        assert not (flags & abi.MSRF_NOT_VISIBLE).any()
    lunar, open_sight = _flags("lunar", setting), _flags("lunar", setting, sight=False)
    hidden = ((lunar & abi.MSRF_NOT_VISIBLE) != 0) & ((open_sight & abi.MSRF_NOT_VISIBLE) == 0)     # by the Moon, not by a mask
    assert hidden.sum(axis=0).min() >= 5 and (open_sight[hidden] & abi.MSRF_PROCESSED).all()
    # window layouts: [R, D] + [Az, El] at msr_size 2 (the ratio of window w in slot w); one window per type at msr_size 1
    refs = am.restated("srp", setting, "long", om.N_F)
    x = am.inputs("srp", setting, "long", om.N_F)
    ratio = np.stack([r["resid_ratio"] for r in refs], axis=-1)
    for k in range(om.N_MSR):
        if x["tracker"][k] < 0 or k in (am.ABSENT_ANGLE[0], am.ABSENT_MSR[0]) or not (flags[k] & abi.MSRF_PROCESSED).all():
            continue
        n_win = -(-len(x["types"][x["tracker"][k]]) // x["M"])
        assert np.isfinite(ratio[k, :n_win]).all() and np.isnan(ratio[k, n_win:]).all(), k
    assert {len(t) for t in x["types"]} == ({4} if setting == "m2" else {2, 3})
    if setting == "m1":
        assert any(list(t) != sorted(t) for t in x["types"])              # list position differs from the type value
    assert all(r["status"] == 0 for r in refs) and all(len(r["records"]) >= 2 for r in refs)


def _looks(config, setting, k):
    """The geometry each run's windows of edges measurement k were computed from, on the restatement's own nominal states."""
    x = am.inputs(config, setting, "edges", om.N_F)
    gs = x["st_c"][x["tracker"][k]]
    out = []
    for r in am.restated(config, setting, "edges", om.N_F):
        for y in am.nominals(x, r, k):
            g = ao.geometry(gs, None, int(x["epochs"][k]), y)
            dr = np.array(g["dr"])
            out.append(dict(az=g["az"], el=g["elev"], mask=gs.elevation_mask_deg, cond=(dr[0] ** 2 + dr[1] ** 2) / (dr @ dr)))
    return out


@pytest.mark.parametrize("config", ["field", "srp"])
@pytest.mark.parametrize("setting", am.SETTINGS)
def test_edges_hold_their_margins(oracle, setting, config):
    """Every edge of the "edges" arc, on every run's nominal states, at least 1e3 x the angle spread from where rounding would decide."""
    _, epochs, sched, k_s = am.edge_geometry(config)
    sp = am.spread(config, setting, "edges", om.N_F)
    tol = 1e3 * max(sp["prefit_deg"], am.DEG_FLOOR)
    refs = am.restated(config, setting, "edges", om.N_F)
    assert all(r["status"] == 0 for r in refs)
    flags = np.stack([r["flags"] for r in refs], axis=-1)
    # azimuth cut: both sides measured, every computed azimuth clear of 0 and 360
    north = [k for k, s in enumerate(sched) if s == "North"]
    az = np.array([[g["az"] for g in _looks(config, setting, k)] for k in north])
    assert (np.minimum(az, 360.0 - az) > tol).all()
    assert (az > 180.0).all(axis=1).sum() >= 2 and (az < 180.0).all(axis=1).sum() >= 2
    straddle = np.array([g["az"] for g in _looks(config, setting, k_s)])
    assert (straddle > tol).all() and (straddle < 0.01).all()
    obs_s = am.inputs(config, setting, "edges", om.N_F)["obs"][k_s, am.AZ]
    if setting == "m2":
        assert (obs_s == am.STRADDLE_OBS).all() and (flags[k_s] == abi.MSRF_PROCESSED | abi.MSRF_REJECTED).all()
        pre = np.array([r["prefit"][k_s, 2] for r in refs])
        assert (np.abs(pre - 360.0) < 0.01).all()
    else:
        assert (obs_s < 0.01).all() and not (flags & abi.MSRF_REJECTED).any()
    # the mask: one measurement just below it, one just above, every margin in [1e-4, 1e-2] deg and far above the spread
    k0, k1 = [k for k, s in enumerate(sched) if s == "Mask"]
    for k, sign, flag in ((k0, -1.0, abi.MSRF_NOT_VISIBLE), (k1, 1.0, abi.MSRF_PROCESSED)):
        m = np.array([sign * (g["el"] - g["mask"]) for g in _looks(config, setting, k)])
        assert (m > max(1e-4, tol)).all() and (m < 1e-2).all(), (k, m.min(), m.max())
        assert (flags[k] == flag).all()
    # near zenith, not at it
    kz = epochs.index(am.EDGE_TIMES["zenith"] * om.S)
    el = np.array([g["el"] for g in _looks(config, setting, kz)])
    assert (np.abs(el - am.ZENITH_DEG) < 0.05).all() and (el < 90.0 - 0.01).all()
    # line of sight along -Z: the conditioning on every run, above the mask, and no NaN on the restatement or its probes
    kp = sched.index("Polar")
    looks = _looks(config, setting, kp)
    cond = np.array([g["cond"] for g in looks])
    assert (cond > 1e-12).all() and (cond < 1e-8).all(), (cond.min(), cond.max())
    assert all(g["el"] > g["mask"] for g in looks) and (flags[kp] == abi.MSRF_PROCESSED).all()
    n_types = len(am.EDGE_TYPES[setting]["Polar"])
    for probe in ("fma", "reassoc"):
        for r, q in zip(am.restated(config, setting, "edges", om.N_F, probe=probe), refs):
            for f in ("prefit", "postfit", "resid_ratio"):
                assert np.array_equal(np.isnan(r[f]), np.isnan(q[f])), (probe, f)
    for r in refs:
        assert np.isfinite(r["prefit"][kp, :n_types]).all() and np.isfinite(r["postfit"][kp, :n_types]).all()


def test_ragged_ensemble_spans_several_blocks():
    """37 runs: two per-thread blocks and ten warp CTAs with partial last ones (sizes read from the kernel sources), the compared runs on
    both sides of every per-thread block edge, and a smoother grid (records x filters) that is not a multiple of its block."""
    n = km.RAGGED
    for per_block in (km.per_thread_block(), km.warps_per_cta()):
        blocks = -(-n // per_block)
        assert blocks >= 2 and n % per_block != 0, per_block
    assert -(-n // km.per_thread_block()) == 2 and -(-n // km.warps_per_cta()) == 10
    edges = {km.per_thread_block() - 1, km.per_thread_block()}
    assert edges <= set(km.EDGE_RUNS) and {0, n - 1} <= set(km.EDGE_RUNS)
    x = am.inputs("field", "m1", "short", n)
    assert (x["cap"] * n) % km.smooth_block() != 0
    assert len({tuple(x["st"][:3, i]) for i in range(n)}) == n
