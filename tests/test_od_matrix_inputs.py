"""CPU companion of tests/test_gpu_od_matrix.py: the orbit-determination matrix can only catch a wrong model, a wrong filter branch
or a wrong covariance entry if its inputs make them matter.  Checked on the oracle alone."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import od_matrix as om

DROPS = [("field", "field"), ("third_body", "point_masses"), ("srp", "srp"), ("lunar", "field"), ("lunar", "point_masses"),
         ("lunar", "srp")]


def _per_filter_moves(a, b):
    """Per filter: the largest position move of the final state or of any recorded estimate, and of the final covariance."""
    dr = np.sqrt(((a["state"][:3] - b["state"][:3]) ** 2).sum(0))
    dr = np.maximum(dr, np.nanmax(np.sqrt(((a["est_state"][:, :3] - b["est_state"][:, :3]) ** 2).sum(1)), axis=0))
    d = np.sqrt(np.einsum("nii->ni", b["covar"]))
    live = d[:, :7]
    dp = np.abs(a["covar"][:, :7, :7] - b["covar"][:, :7, :7]) / (live[:, :, None] * live[:, None, :])
    return dr, dp.reshape(len(dp), -1).max(1)


@pytest.mark.parametrize("config,drop", DROPS)
def test_every_model_moves_the_filter_answer(oracle, config, drop):
    """Dropping the model moves every filter's estimates and final covariance by more than 1e3 x the matrix's bound."""
    bounds = om.filter_bounds(config, "ekf", "regular", 21, None)
    dr, dp = _per_filter_moves(om.oracle_filters(config, drop=drop), om.oracle_filters(config))
    # The Moon-centred arc's oracle spread is 20 x the Earth arcs' and lunar SRP is weak over 48 min: 1e2 x there (the Earth "srp"
    # configuration pins the SRP path at 1e3 x).
    factor = 1e2 if (config, drop) == ("lunar", "srp") else 1e3
    assert dr.min() > factor * max(bounds["dr"], bounds["est_dr"]), (config, drop, dr.min(), bounds["dr"])
    assert dp.min() > 1e3 * bounds["covar"], (config, drop, dp.min(), bounds["covar"])


def test_per_filter_srp_areas_matter(oracle):
    """Exchanging the SRP areas of neighbouring filters (what a kernel reading the wrong lane would do) moves every exchanged filter."""
    bounds = om.filter_bounds("srp", "ekf", "regular", 21, None)
    dr, dp = _per_filter_moves(om.oracle_filters("srp", swap_areas=True), om.oracle_filters("srp"))
    assert dr[: om.N_F - 1].min() > 1e3 * max(bounds["dr"], bounds["est_dr"]) and dp[: om.N_F - 1].min() > 1e3 * bounds["covar"]
    assert dr[-1] == 0.0
    assert 2.0 in set(om.filters("srp")[0][6])         # the EKF update clamps Cr at 2


def test_srp_arc_crosses_penumbra_and_umbra(oracle):
    """Earth shadow fraction along the filters' arc (truth recorded every 10 s): it flies through full sunlight, penumbra (a few
    seconds at this altitude) and umbra."""
    L = oracle.lib()
    packed = om.dynamics("srp").pack(nb.EARTH_J2000, om.almanac("srp"))
    sun = packed.c.bodies[packed.c.srp.contents.sun_body]
    t_ep = np.arange(0, om.N_MSR * om.CADENCE_S + 1, 10) * om.S
    prop = nb.Propagator.new(om.dynamics("srp"), nb.IntegratorMethod.RungeKutta89, nb.IntegratorOptions.with_fixed_step_s(10.0))
    st, cs, ep = nb.pack_spacecraft([nb.Spacecraft(orbit=om.truth_orbit("srp"), mass=nb.Mass(500.0, 20.0, 50.0), srp=nb.SRPData(8.0, 1.3))])
    rec = oracle.propagate_batch(packed.c, prop.opts.to_c(prop.method), st, cs, ep, int(t_ep[-1]), traj_capacity=len(t_ep) + 1)[4]
    fr = []
    for k in range(int(rec[2][0])):
        sp = np.zeros(3)
        assert L.nyx_oracle_body_position(C.byref(sun), int(rec[0][k, 0]), abi.as_double_p(sp)) == 0
        y = np.ascontiguousarray(rec[1][:3, k, 0])
        fr.append(L.nyx_oracle_occultation(abi.as_double_p(y), abi.as_double_p(np.ascontiguousarray(sp - y)), sun.radius_km,
                                           packed.c.central_radius_km))
    fr = np.array(fr)
    assert (fr == 0.0).sum() >= 20 and ((fr > 0.0) & (fr < 1.0)).sum() >= 1 and (fr == 1.0).sum() >= 20, fr


def test_arcs_produce_every_flag(oracle):
    reg = om.oracle_filters("srp")["msr_flags"]
    edge = om.oracle_filters("srp", arc_kind="edge")["msr_flags"]
    assert (reg & abi.MSRF_PROCESSED).any() and (reg & abi.MSRF_NOT_VISIBLE).any() and (reg & abi.MSRF_ABSENT).any()
    for k, i in om.BLUNDERS:
        assert reg[k, i] == abi.MSRF_PROCESSED | abi.MSRF_REJECTED
    assert reg[om.ABSENT] == abi.MSRF_ABSENT
    assert (edge[7] == 0).all()                                         # unknown tracker: nothing happens
    assert (edge & abi.MSRF_NOT_VISIBLE).any() and (edge[5] & abi.MSRF_PROCESSED).all() and (edge[9] & abi.MSRF_PROCESSED).all()
    assert (om.oracle_filters("srp", "ekf_scalar_noreject")["msr_flags"] & abi.MSRF_REJECTED).sum() == 0


@pytest.mark.parametrize("variant", ["ekf_scalar_noreject", "ckf_scalar"])
def test_short_snc_disable_takes_both_branches(oracle, monkeypatch, variant):
    from oracle import pyoracle_od

    taken = []
    snc = pyoracle_od._snc
    monkeypatch.setattr(pyoracle_od, "_snc", lambda *a: taken.append(snc(*a) is not None) or snc(*a))
    om.oracle_filters.__wrapped__("srp", variant)
    assert any(taken) and not all(taken), (sum(taken), len(taken))


def test_ckf_state_deviation_is_live(oracle):
    for variant in ("ckf_reject", "ckf_scalar"):
        dev = om.oracle_filters("srp", variant)["state_dev"]
        assert (np.abs(dev[:3]).max(0) > 1e-4).all() and (np.abs(dev[6]) > 0).all(), variant


def test_compared_covariance_entries_are_not_negligible(oracle):
    """The position-velocity and velocity-Cr correlations of every final covariance are far above the bound they are compared at."""
    for config in ("srp", "lunar"):
        P = om.oracle_filters(config)["covar"]
        d = np.sqrt(np.einsum("nii->ni", P))
        corr = P / (d[:, :, None] * d[:, None, :] + (d[:, :, None] * d[:, None, :] == 0))
        bound = om.filter_bounds(config, "ekf", "regular", 21, None)["covar"]
        assert (np.abs(corr[:, :3, 3:6]).reshape(om.N_F, -1).max(1) > 1e3 * bound).all(), config
        assert (np.abs(corr[:, 3:6, 6]).max(1) > 1e3 * bound).all(), config


def test_cooperative_column_deal():
    """The restated deal gives the thresholds the field shapes are chosen at."""
    assert [om.coop_columns_per_lane(n, n) for n in (8, 31, 32, 63, 64, 95, 96)] == [1, 1, 2, 2, 3, 3, 4]
    assert om.coop_columns_per_lane(8, 0) == om.coop_columns_per_lane(21, 4) == 1
