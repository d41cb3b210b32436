"""CPU companion of tests/test_gpu_fast_matrix.py: the FAST parity matrix can only catch a wrong force model if its inputs make
that model matter.  Checked on the oracle alone: every model of every configuration moves the 6 h fixed-step answer by far more
than the matrix's bound, the SRP ensemble flies through penumbra and umbra, and the eccentric orbits cross the StdAtm branch
altitude."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi
from tests import fast_matrix as fm
from tests.util import max_dr_dv

# the model each configuration adds to the one before it (or to two-body)
DROPS = [("field", "field"), ("third_body", "point_masses"), ("srp", "srp"), ("drag_constant", "drag"), ("drag_exponential", "drag"),
         ("drag_stdatm", "drag"), ("all", "second_field"), ("all", "srp"), ("all", "drag")]


@pytest.mark.parametrize("config,drop", DROPS)
def test_every_model_moves_the_fixed_step_answer(oracle, config, drop):
    """Dropping the model must move the answer by >= 1e3 x the fixed-step bound on every trajectory that the model acts on: a
    kernel that lost or garbled it could not stay inside the bound."""
    full = fm.oracle_fixed(config)[0]
    without = fm.oracle_fixed(config, drop=drop)[0]
    dr = np.sqrt(((full[:3] - without[:3]) ** 2).sum(0))
    if drop == "srp":   # Cr = -0.3 is clamped to 0: no SRP on those trajectories, in the oracle as in the kernels
        cr = fm.ensemble()[0][6]
        assert (dr[cr < 0] == 0).all()
        dr = dr[cr > 0]
    assert dr.min() > 1e3 * fm.FIXED_DR, (config, drop, dr.min())


def test_per_lane_constants_matter(oracle):
    """Exchanging the SRP areas of neighbouring trajectories (what a kernel reading lane ^ 1 would do) moves the answer by more
    than 1e3 x the bound on every trajectory that feels SRP.  Cr values below 0 and above 2 are in the ensemble, so both clamps
    act."""
    st, cs, ep = fm.ensemble()
    prop = fm.propagator("srp")
    packed, oc = prop.dynamics.pack(nb.EARTH_J2000, fm.almanac()), prop.opts.to_c(prop.method)
    ref = fm.oracle_fixed("srp")[0]
    swapped = cs.copy()
    swapped[2] = cs[2].reshape(-1, 2)[:, ::-1].reshape(-1)
    moved = np.sqrt(((oracle.propagate_batch(packed.c, oc, st, swapped, ep, fm.END)[0][:3] - ref[:3]) ** 2).sum(0))
    assert (moved[st[6] > 0] > 1e3 * fm.FIXED_DR).all()
    assert set(np.round(st[6], 6)) == set(fm.CR_VALUES)


def _records(config):
    ref = fm.oracle_fixed(config, traj_capacity=400)
    t_ep, t_st, t_cnt = ref[4]
    assert (t_cnt == ref[2]["n_steps"] + 1).all()
    return t_ep, t_st, t_cnt


def test_srp_ensemble_crosses_penumbra_and_umbra(oracle):
    """Earth shadow fraction of every recorded state (anise `occultation`, restated by the oracle): the ensemble spends steps in
    full sunlight, in penumbra (0 < f < 1) and in umbra (f = 1), so a wrong shadow path cannot hide."""
    L = oracle.lib()
    alm = fm.almanac()
    packed = fm.dynamics("srp").pack(nb.EARTH_J2000, alm)
    sun = packed.c.bodies[packed.c.srp.contents.sun_body]
    t_ep, t_st, t_cnt = _records("srp")
    fr = []
    for i in range(t_ep.shape[1]):
        for k in range(int(t_cnt[i])):
            sp = np.zeros(3)
            assert L.nyx_oracle_body_position(C.byref(sun), int(t_ep[k, i]), abi.as_double_p(sp)) == 0
            y = np.ascontiguousarray(t_st[:3, k, i])
            r_ls = np.ascontiguousarray(sp - y)
            fr.append(L.nyx_oracle_occultation(abi.as_double_p(y), abi.as_double_p(r_ls), sun.radius_km, packed.c.central_radius_km))
    fr = np.array(fr)
    assert (fr == 0.0).mean() > 0.4
    assert ((fr > 0.0) & (fr < 1.0)).sum() >= 20, ((fr > 0.0) & (fr < 1.0)).sum()
    assert (fr == 1.0).sum() >= 100


def test_eccentric_orbits_cross_the_stdatm_branch_altitude(oracle):
    t_ep, t_st, t_cnt = _records("drag_stdatm")
    r_eq = fm.dynamics("drag_stdatm").pack(nb.EARTH_J2000, fm.almanac()).c.drag.contents.r_eq_km
    for i in range(fm.N_LEO, fm.N_LEO + fm.N_ECC):
        alt = np.linalg.norm(t_st[:3, : int(t_cnt[i]), i], axis=0) - r_eq
        assert alt.min() < fm.STDATM_BRANCH_KM - 400 and alt.max() > fm.STDATM_BRANCH_KM + 300, (i, alt.min(), alt.max())
