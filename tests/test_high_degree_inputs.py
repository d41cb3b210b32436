"""CPU companion of tests/test_gpu_high_degree.py (degree 71..96), checked without a device:
  * the oracle's harmonic acceleration and its dual-number gradient at degree 96 against an independent 50-digit arbiter (the
    Holmes & Featherstone recursion of tests/arbiters.py, itself checked against the closed-form arbiter);
  * the inputs can see what they test: each change of the field above degree 80 moves the oracle's fixed-step answer by far more
    than the GPU bound;
  * the lane-cooperative FAST kernel's table (K2, three and four columns per lane) walked on the host reproduces the oracle."""
import multiprocessing as mp

import numpy as np
import pytest

import nyx_b200 as nb
from tests import high_degree as hd
from tests import od_matrix as om


def _packed(gd, body):
    packed = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd))).pack(hd.FRAME[body], None)
    packed.c.gravity[0].rot.kind = 0   # identity rotation: the harmonic sum is evaluated at the given body-fixed position
    return packed


def _points(body, seed):
    """12 body-fixed positions: 4 with |sin phi| > 0.999 (both poles), 4 at 1.01 r_eq, 4 between 1.01 and 1.2 r_eq."""
    r_eq = hd.FIXTURE[body][2].mean_equatorial_radius_km()
    rng = np.random.default_rng(seed)
    out = []
    for k in range(12):
        if k < 4:
            sphi = (1 if k % 2 else -1) * rng.uniform(0.999, 0.99995)
        else:
            sphi = rng.uniform(-0.95, 0.95)
        lam = rng.uniform(-np.pi, np.pi)
        cphi = np.sqrt(1.0 - sphi * sphi)
        radius = r_eq * (1.01 if k < 8 else rng.uniform(1.01, 1.2))
        out.append(radius * np.array([cphi * np.cos(lam), cphi * np.sin(lam), sphi]))
    return out


def _arbiter_job(job):
    from scripts.arbiter_harmonics import oracle_field_accel
    from tests.arbiters import mp_harmonic_accel_recursion

    body, rb = job
    gd = hd.field_data(body)
    gf = _packed(gd, body).c.gravity[0]
    got = oracle_field_accel(_packed(gd, body).c, rb)
    want = np.array(mp_harmonic_accel_recursion(gd.c_nm, gd.s_nm, 96, 96, gf.mu_km3_s2, gf.r_eq_km, rb))
    return float(np.abs(got - want).max() / np.abs(want).max())


def test_recursion_arbiter_against_the_closed_form_arbiter():
    """The two arbiters share only the spherical gradient: on the degree-21 (Earth) and degree-12 (Moon) points of
    test_oracle_arbiters, unrounded, they agree to 1e-25 relative.  At degree 96 the comparison is scripts/arbiter_harmonics.py
    --points96 (profiles/r02_arbiter_harmonics.json): the closed form takes minutes per point there."""
    from tests.arbiters import mp_harmonic_accel, mp_harmonic_accel_recursion

    for fixture, deg, seeds in (("jgm3_70x70", 21, range(100, 104)), ("luna_jggrx_80x80", 12, range(200, 204))):
        moon = fixture.startswith("luna")
        gd = nb.GravityFieldData.from_fixture(fixture, deg, deg, nb.IAU_MOON_FRAME if moon else nb.IAU_EARTH_FRAME)
        gf = _packed(gd, "moon" if moon else "earth").c.gravity[0]
        for seed in seeds:
            rng = np.random.default_rng(seed)
            d = rng.normal(size=3)
            rb = d / np.linalg.norm(d) * gf.r_eq_km * rng.uniform(1.02, 1.5)
            args = (gd.c_nm, gd.s_nm, deg, deg, gf.mu_km3_s2, gf.r_eq_km, rb)
            a = mp_harmonic_accel(*args, dps=40, as_mpf=True)
            b = mp_harmonic_accel_recursion(*args, dps=50, as_mpf=True)
            rel = max(abs(x - y) for x, y in zip(a, b)) / max(abs(x) for x in a)
            assert rel < 1e-25, (fixture, seed, float(rel))


def test_oracle_harmonics_at_degree_96_against_the_arbiter(oracle):
    """GravityField::eom as restated by the oracle, degree 96, Earth and Moon, 12 points each (near both poles, at 1.01 r_eq where
    rho^96 ~ 0.4), relative to the largest component of the non-central acceleration: <= 1e-13 (measured at most 1.8e-15), except
    near the lunar poles.  There the f64 sum of the reference algorithm itself loses about two digits on the rough lunar field:
    1.4e-13 at sin(phi) = -0.99928 (the arbiter at 50 and 90 digits agrees to 1e-48), 5e-15 to 1e-14 at the other three; the
    JGM-3 polar points stay below 1e-15.  Bound there: 3e-13."""
    jobs = [(body, rb) for body, seed in (("earth", 961), ("moon", 962)) for rb in _points(body, seed)]
    with mp.get_context("fork").Pool(min(8, mp.cpu_count())) as pool:
        errs = pool.map(_arbiter_job, jobs, chunksize=1)
    polar = np.array([abs(rb[2]) / np.linalg.norm(rb) > 0.999 for _, rb in jobs])
    errs = np.array(errs)
    print(f"arbiter 96x96 max rel err: polar {errs[polar].max():.2e}, others {errs[~polar].max():.2e}")
    assert polar.sum() == 8 and (errs[~polar] < 1e-13).all() and (errs[polar] < 3e-13).all(), errs


def _grad_job(job):
    import mpmath
    from tests.arbiters import mp_harmonic_accel_recursion

    body, rb = job
    gd = hd.field_data(body)
    gf = _packed(gd, body).c.gravity[0]
    # central differences of the unrounded 50-digit acceleration: step 1e-4 km, truncation error h^2 a''' / 6 ~ 1e-8 h^2 |a| (n / r)^3
    # with n / r ~ 0.05 / km on the Moon, far below the f64 gradient's own rounding
    h = 1e-4
    G = np.zeros((3, 3))
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        ap = mp_harmonic_accel_recursion(gd.c_nm, gd.s_nm, 96, 96, gf.mu_km3_s2, gf.r_eq_km, rb + e, as_mpf=True)
        am = mp_harmonic_accel_recursion(gd.c_nm, gd.s_nm, 96, 96, gf.mu_km3_s2, gf.r_eq_km, rb - e, as_mpf=True)
        step = mpmath.mpf((rb + e)[k]) - mpmath.mpf((rb - e)[k])   # the f64 positions, not 2h: rb + e rounds at 1e-12 km
        G[:, k] = [float((ap[i] - am[i]) / step) for i in range(3)]
    return G


def test_dual_number_gradient_at_degree_96_against_differences_of_the_arbiter(oracle):
    """dual_eom's da/dr at degree 96 (one Earth and one Moon point, both at 1.02 r_eq) against central differences of the arbiter,
    after the analytic two-body part is removed: 1e-10 relative (measured 2.4e-13 Earth, 1.9e-12 Moon)."""
    jobs = [("earth", _points("earth", 963)[9] * 1.02 / 1.01), ("moon", _points("moon", 964)[5] * 1.02 / 1.01)]
    with mp.get_context("fork").Pool(2) as pool:
        grads = pool.map(_grad_job, jobs)
    for (body, rb), G_h in zip(jobs, grads):
        packed = _packed(hd.field_data(body), body)
        mu = packed.c.mu_central_km3_s2
        y = np.concatenate([rb, [1.0, 2.0, 3.0], [1.8, 2.2, 0.0]])
        _, A = oracle.dual_eom(packed.c, 0, y, np.array([100.0, 0.0, 1.0, 1.0]))
        r = np.linalg.norm(rb)
        G_tb = -mu / r ** 3 * (np.eye(3) - 3.0 * np.outer(rb, rb) / r ** 2)
        got_h = A[3:6, 0:3] - G_tb
        err = np.abs(got_h - G_h).max() / np.abs(G_h).max()
        print(f"dual gradient 96x96 {body}: rel err {err:.2e}")
        assert err < 1e-10, (body, got_h, G_h)


@pytest.mark.parametrize("body", ("moon", "earth"))
@pytest.mark.parametrize("drop", hd.DROPS)
def test_every_high_degree_change_moves_the_fixed_step_answer(oracle, body, drop):
    """Each change of the field above degree 80 moves the oracle's fixed-step final position by >= 1e3 x the GPU bound
    (hd.fixed_bounds): on every trajectory, except the sectoral (96, 96) term alone, which scales as cos(phi)^96 and so is felt only
    within a few degrees of the equator; the near-polar orbits whose periapsis lies at high latitude hardly feel it, and half of the
    ensemble must."""
    full = hd.oracle_fixed(body)[0]
    changed = hd.oracle_fixed(body, drop=drop)[0]
    dr = np.sqrt(((full[:3] - changed[:3]) ** 2).sum(0))
    need = 1e3 * hd.fixed_bounds(body)[0]
    print(f"{body} {drop}: moved min {dr.min():.2e} median {np.median(dr):.2e} km, need {need:.1e}")
    if drop == "sectoral_96":
        assert (dr > need).mean() >= 0.5, np.sort(dr)
    else:
        assert dr.min() > need, np.sort(dr)


def test_ensembles_reach_the_pole_and_low_altitude(oracle):
    """The lunar periapses lie at 30..60 km and the LEO orbits at 250..300 km; exactly polar and near-polar orbits are flown."""
    for body, lo, hi in (("moon", 30.0, 62.0), ("earth", 248.0, 302.0)):
        st = hd.ensemble(body)[0]
        r_eq = hd.FIXTURE[body][2].mean_equatorial_radius_km()
        alt0 = np.linalg.norm(st[:3], axis=0) - r_eq
        assert alt0.min() > lo - 1.0
        h = np.cross(st[:3].T, st[3:6].T)
        inc = np.degrees(np.arccos(h[:, 2] / np.linalg.norm(h, axis=1)))
        assert np.isclose(inc, 90.0, atol=1e-9).any() and ((np.abs(inc - 90.0) < 3.0).sum() >= 4), inc
    assert hd.ensemble("moon")[0].shape[1] == 40 and hd.ensemble("earth")[0].shape[1] == 24


def test_degree_96_field_continues_the_fixture_spectrum():
    """The drawn rows follow the power law fitted over the fixture's top ten degrees: the degree RMS of rows above the fixture stays
    within a factor 1.6 of the law, and the first drawn row is within a factor 1.6 of the fixture's last row."""
    for body in ("earth", "moon"):
        c, s, (a, b) = hd._full(body)
        top = hd.FIXTURE[body][1]
        assert b < 0
        for n in range(top + 1, hd.TOP + 1):
            law = np.exp(a + b * np.log(n))
            assert 1 / 1.6 < hd.degree_rms(c, s, n) / law < 1.6, (body, n)
        assert 1 / 1.6 < hd.degree_rms(c, s, top + 1) / hd.degree_rms(c, s, top) < 1.6
        assert (s[:, 0] == 0).all() and np.count_nonzero(c[hd.TOP]) == hd.TOP + 1


def test_four_columns_per_lane_at_degree_96():
    assert om.coop_columns_per_lane(96, 96) == 4
    assert om.coop_columns_per_lane(96, 95) == om.coop_columns_per_lane(95, 95) == om.coop_columns_per_lane(81, 81) == 3


def _dump_field(gd, lanes):
    from tests.test_coop_table import _dump

    return _dump(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd))).pack(nb.MOON_J2000, None), lanes)


TABLE_SHAPES = [(71, 71), (80, 80), (95, 95), (96, 96), (96, 0), (96, 1), (96, 95)]


@pytest.mark.parametrize("lanes", (8, 16, 32))
@pytest.mark.parametrize("degree,order", TABLE_SHAPES, ids=[f"{d}x{o}" for d, o in TABLE_SHAPES])
def test_cooperative_table_at_high_degree(oracle, degree, order, lanes):
    """K2's schedule and packed records (tests/test_coop_table.py) for the lunar degree-96 field's shapes, walked at 4 points at 1.03..1.6 r_eq
    and 16 at 1.005..1.05 r_eq.  Close to the surface, a recursion left running through a lane's idle gap after its last column
    overflows (95x95 on 32 lanes idles for 62 entries): the schedule stops it there with a stop column."""
    from tests.test_coop_table import check_table

    gd = hd.field_data("moon", degree, order)
    L, kmax, _, col_start, col_m, _ = _dump_field(gd, lanes)
    if (degree, order, lanes) == (95, 95, 32):
        assert (col_m[col_start <= L] == degree + 2).any()
    check_table(oracle, gd, nb.MOON_J2000, lanes)
    check_table(oracle, gd, nb.MOON_J2000, lanes, radii=(1.005, 1.05), points=16)
