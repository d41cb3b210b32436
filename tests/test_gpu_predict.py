"""GPU covariance mapping (`KalmanODProcess::predict_until`, od/process/mod.rs:440-486) through `nyxb_od_predict_batch`: parity
with the oracle restatement (tests/predict_oracle.py) on every kernel family, and an oracle-free check against a Monte Carlo.

Tolerances (floating point; the reference pins none of these values, see DESIGN.md §3):
  Same step sequence as the oracle (fixed steps, and STRICT adaptive): STRICT |dr| < 1e-9 km, |dv| < 1e-12 km/s, every record's
  covariance within 1e-9 of the largest entry of its 3x3 block (rr, rv, vr, vv); FAST (FMA, and the warp kernel's regrouped
  harmonic sum) 1e-7 km, 1e-10 km/s, 1e-7.  FAST adaptive may flip one accept/grow decision of the controller; the as-coded STM is
  first order in the step, so it then moves at the 1e-3 level (tests/test_gpu_stm_od.py): 1e-6 km and 1e-2 of the block, plus
  1e-2 of the deviation for the recorded states (nominal + Phi x).
  Record counts, record epochs and final epochs are exact; run i alone gives the same bits as run i inside the batch.
Monte Carlo check: variances within 5 % (sampling error sqrt(2/n) = 1 % at n = 20 000), correlations within 0.05."""
import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi

from .od_util import S

pytestmark = pytest.mark.gpu

MS = 60 * S
FAMILIES = ["thread_strict", "thread_fast", "coop"]


@pytest.fixture(scope="module")
def po(oracle):
    from . import predict_oracle

    return predict_oracle


def _setup(family, stepping):
    frame = nb.EARTH_J2000
    gd = nb.GravityFieldData.from_fixture("jgm3_70x70", 12, 12, nb.IAU_EARTH_FRAME)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    mode = nb.MODE_STRICT if family == "thread_strict" else nb.MODE_FAST
    if stepping == "fixed":
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.RungeKutta4, nb.IntegratorOptions.with_fixed_step_s(10.0), mode=mode)
    else:
        prop = nb.Propagator.new(dyn, nb.IntegratorMethod.DormandPrince78, nb.IntegratorOptions(init_step=5 * S), mode=mode)
    eng = prop.engine(frame, None)
    eng.set_kernel(nb.KERNEL_THREAD if family == "thread_fast" else nb.KERNEL_AUTO)
    rng = np.random.default_rng(7)
    ests = []
    for i, t0 in enumerate([0, 30 * S, 0, 7 * S + 3]):
        orbit = nb.Orbit.keplerian(7000.0 + 50 * i, 0.01, 51.6, 30.0 + 10 * i, 40.0, 10.0 * i, t0, frame)
        sc = nb.Spacecraft(orbit=orbit, mass=nb.Mass(500.0, 50.0, 0.0))
        A = rng.normal(size=(6, 6)) * np.array([1.0, 1.0, 1.0, 1e-3, 1e-3, 1e-3])
        cov = np.zeros((9, 9))
        cov[:6, :6] = A @ A.T
        ests.append(nb.KfEstimate(sc, cov, np.concatenate([rng.normal(0, 0.1, 3), rng.normal(0, 1e-4, 3), [0.0, 0.0, 0.0]])))
    # per-run ends: exact multiple, overshoot by 43 s, end before the start, a few chunks
    end = np.array([10 * MS, 30 * S + 10 * MS - 17 * S, -S, 7 * S + 3 + 3 * MS - 1], dtype=np.int64)
    return dict(frame=frame, dyn=dyn, prop=prop, eng=eng, ests=ests, end=end, mode=mode,
                dyn_c=dyn.pack(frame, None).c, opts_c=prop.opts.to_c(prop.method))


def _odp(s, variant, snc):
    odp = nb.KalmanODProcess(s["prop"], variant, None, {}, None)
    if snc == "inertial":
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-10, 2e-10, 3e-10], 3600 * S))
    elif snc == "ric":
        odp.with_process_noise(nb.ProcessNoise3D.from_diagonal([1e-10, 2e-10, 3e-10], 3600 * S, nb.LocalFrame.RIC))
    return odp


def _oracle(po, s, odp, i):
    e = s["ests"][i]
    sc = e.nominal_state
    cs = np.array([sc.mass.dry_mass_kg, sc.mass.extra_mass_kg, sc.srp.area_m2, sc.drag.area_m2])
    return po.predict_until(s["dyn_c"], s["opts_c"], odp.config_c(), sc.to_vector(), cs, sc.epoch(), e.covar, int(s["end"][i]),
                            e.state_deviation)


def _blocks_close(a, b, rtol):
    """a, b: [..][9][9]; each 3x3 block of the 6x6 within rtol of the largest entry of that block of b."""
    for rs in (slice(0, 3), slice(3, 6)):
        for cs_ in (slice(0, 3), slice(3, 6)):
            scale = np.abs(b[..., rs, cs_]).max()
            assert np.abs(a[..., rs, cs_] - b[..., rs, cs_]).max() <= rtol * scale, (rs, cs_, np.abs(a[..., rs, cs_] - b[..., rs, cs_]).max(), scale)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stepping", ["fixed", "adaptive"])
@pytest.mark.parametrize("variant,snc", [(nb.KalmanVariant.ReferenceUpdate, "off"), (nb.KalmanVariant.DeviationTracking, "inertial"),
                                         (nb.KalmanVariant.DeviationTracking, "ric"), (nb.KalmanVariant.ReferenceUpdate, "ric")])
def test_predict_matches_oracle(po, family, stepping, variant, snc):
    s = _setup(family, stepping)
    odp = _odp(s, variant, snc)
    sol = odp.predict_ensemble_until(s["ests"], s["end"])
    assert s["eng"].last_kernel() == (abi.KERNEL_COOP if family == "coop" else abi.KERNEL_THREAD)
    strict = s["mode"] == nb.MODE_STRICT
    for i in range(4):
        ref = _oracle(po, s, odp, i)
        assert sol.status[i] == ref["status"] == 0
        assert sol.rec_count[i] == ref["count"] and sol.final_epoch_ns[i] == ref["epoch"]
        assert np.array_equal(sol.record_epochs(i), ref["rec_epoch"])
        K = ref["count"]
        rs = sol.rec_state[:K, :, i]
        rc = sol.rec_covar[:K, :, i].reshape(K, 9, 9).transpose(0, 2, 1)
        tr, tv, tc = (1e-9, 1e-12, 1e-9) if strict else (1e-7, 1e-10, 1e-7)
        if stepping == "fixed" or strict:
            assert sol.details["n_steps"][i] == ref["n_steps"]
        else:   # FAST adaptive: the step sequence may differ even where the step count does not (measured: 4e-4 of the block);
            # a record's state carries the deviation Phi x, which moves with Phi (measured: 1.5e-5 km for 1 km deviations)
            tc = 1e-2
            tr, tv = 1e-6 + tc * np.abs(ref["state_dev"][:3]).max(), 1e-9 + tc * np.abs(ref["state_dev"][3:6]).max()
        assert np.abs(rs[:, :3] - ref["rec_state"][:, :3]).max() < tr
        assert np.abs(rs[:, 3:6] - ref["rec_state"][:, 3:6]).max() < tv
        assert np.array_equal(rs[:, 6:], ref["rec_state"][:, 6:])
        _blocks_close(rc, ref["rec_covar"], tc)
        _blocks_close(sol.covar[i][None], ref["covar"][None], tc)
        assert np.abs(sol.final_state_soa[:3, i] - ref["state"][:3]).max() < (tr if strict or stepping == "fixed" else 1e-6)
        if variant == nb.KalmanVariant.ReferenceUpdate:
            assert np.array_equal(sol.state_deviation[:, i], np.zeros(9))
        else:
            assert np.abs(sol.state_deviation[:3, i] - ref["state_dev"][:3]).max() < max(tr, tc * 0.1)
    # records past a run's count read back as NaN
    assert np.isnan(sol.rec_state[sol.rec_count[2]:, 0, 2]).all()


@pytest.mark.parametrize("family", FAMILIES)
def test_capacity_null_records_and_batch_invariance(family):
    s = _setup(family, "adaptive")
    odp = _odp(s, nb.KalmanVariant.DeviationTracking, "ric")
    full = odp.predict_ensemble_until(s["ests"], s["end"])
    few = odp.predict_ensemble_until(s["ests"], s["end"], capacity=3)
    bare = odp.predict_ensemble_until(s["ests"], s["end"], capacity=0)
    cov_only = odp.predict_ensemble_until(s["ests"], s["end"], record_states=False)
    assert few.rec_state.shape[0] == 3 and np.array_equal(few.rec_count, full.rec_count)
    assert np.array_equal(few.rec_state, full.rec_state[:3], equal_nan=True)   # run 2 has two records: NaN past them in both
    assert np.array_equal(few.rec_covar, full.rec_covar[:3], equal_nan=True)
    assert bare.rec_state is None and bare.rec_covar is None and cov_only.rec_state is None
    assert np.array_equal(cov_only.rec_covar, full.rec_covar, equal_nan=True)
    for other in (few, bare, cov_only):
        assert np.array_equal(other.final_state_soa, full.final_state_soa) and np.array_equal(other.covar, full.covar)
        assert np.array_equal(other.state_deviation, full.state_deviation) and np.array_equal(other.final_epoch_ns, full.final_epoch_ns)
    for i in range(4):   # run i alone: the same bits as inside the batch
        one = odp.predict_ensemble_until([s["ests"][i]], s["end"][i])
        k = one.rec_count[0]
        assert k == full.rec_count[i]
        assert np.array_equal(one.rec_state[:k, :, 0], full.rec_state[:k, :, i])
        assert np.array_equal(one.rec_covar[:k, :, 0], full.rec_covar[:k, :, i])
        assert np.array_equal(one.covar[0], full.covar[i]) and np.array_equal(one.final_state_soa[:, 0], full.final_state_soa[:, i])


def test_unsupported_setups():
    frame = nb.EARTH_J2000
    sc = nb.Spacecraft(orbit=nb.Orbit.keplerian(7000.0, 0.01, 51.6, 30.0, 40.0, 10.0, 0, frame))
    est = nb.KfEstimate.from_diag(sc, [1.0, 1.0, 1.0, 1e-6, 1e-6, 1e-6, 0.0, 0.0, 0.0])
    drag = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.two_body(), nb.Drag(nb.AtmDensity.Constant(1e-12), nb.IAU_EARTH_FRAME))
    odp = nb.KalmanODProcess(nb.Propagator.default(drag), nb.KalmanVariant.DeviationTracking, None, {}, None)
    with pytest.raises(nb.PropagationError, match="rc=-4.*PartialsUndefined"):
        odp.predict_for(est, MS)
    # states relative to another centre than the integration frame's (integration_frame)
    alm = nb.Almanac.synthetic(frame, 0, 2.0)
    prop = nb.Propagator.default(nb.SpacecraftDynamics.new(nb.OrbitalDynamics.point_masses([nb.MOON, nb.SUN])))
    prop.opts.integration_frame = nb.EARTH_J2000
    moon_sc = nb.Spacecraft(orbit=nb.Orbit.keplerian(1837.4, 0.001, 90.0, 10.0, 0.0, 0.0, 0, nb.MOON_J2000))
    odp2 = nb.KalmanODProcess(prop, nb.KalmanVariant.DeviationTracking, None, {}, alm)
    with pytest.raises(nb.PropagationError, match="rc=-4"):
        odp2.predict_for(nb.KfEstimate.from_diag(moon_sc, [1.0] * 6 + [0.0] * 3), MS)
    # max_step <= 0
    odp.max_step = 0
    with pytest.raises(nb.ODError, match="StepSize"):
        odp.predict_for(est, MS)


def test_linear_covariance_matches_monte_carlo():
    """No oracle: the predicted 6x6 covariance at 6.5 days on the C3 geometry (JWST-like orbit and SRP of
    examples/02_jwst_covar_monte_carlo) against the sample covariance of 20 000 runs drawn by `to_random_variable()` on the device
    (nyxb_mvn_sample) and propagated by nyxb_propagate_batch.  The RIC uncertainty of the example is scaled down 10x.
    The dynamics are Earth gravity + SRP, without the example's Sun and Moon point masses: with them the as-coded third-body partials
    (PointMasses::gradient, DESIGN.md §7) make the reference's own covariance depart from the linearisation of its dynamics by up to
    10 % in variance here (measured: the same departure against a finite-difference STM, at 1/10 and 1/100 of the uncertainty, with
    1-minute and 1-hour chunks), so that geometry checks the reference's partials rather than this prediction."""
    frame = nb.EARTH_J2000
    span = int(6.5 * 86400) * S
    alm = nb.Almanac.synthetic(frame, 0, 8.5)
    srp = nb.SolarPressure.new([nb.EARTH_J2000, nb.MOON_J2000], alm)
    dyn = nb.SpacecraftDynamics.from_model(nb.OrbitalDynamics.two_body(), srp)
    orbit = nb.Orbit.cartesian(119901.070276, -1389299.665421, -1041369.150539, 0.045956, -0.013168, 0.034535, 0, frame)
    jwst = nb.Spacecraft(orbit=orbit, mass=nb.Mass(6200.0, 0.0, 0.0), srp=nb.SRPData(21.197 * 14.162, 1.56))
    unc = nb.SpacecraftUncertainty(jwst, nb.LocalFrame.RIC, x_km=0.05, y_km=0.03, z_km=0.15, vx_km_s=1e-5, vy_km_s=0.6e-4, vz_km_s=3e-4)
    est = unc.to_estimate()
    prop = nb.Propagator.default(dyn, mode=nb.MODE_FAST)
    odp = nb.KalmanODProcess(prop, nb.KalmanVariant.DeviationTracking, None, {}, alm)
    sol = odp.predict_for(est, span, capacity=0)
    assert sol.status[0] == 0 and sol.rec_count[0] == 9361 and sol.final_epoch_ns[0] == span
    P = sol.covar[0][:6, :6]
    n = 20_000
    mvn = est.to_random_variable()
    st, _ = mvn.sample_on_device(2024, n)
    cs = np.zeros((4, n))
    cs[0] = jwst.mass.dry_mass_kg
    cs[2] = jwst.srp.area_m2
    out, oep, _, status = prop.engine(frame, alm).propagate_batch(st, cs, np.zeros(n, dtype=np.int64), span)
    assert (status == 0).all() and (oep == span).all()
    Ps = np.cov(out[:6])
    var_ratio = np.diag(Ps) / np.diag(P)
    assert np.abs(var_ratio - 1.0).max() < 0.05, var_ratio
    d, ds = np.sqrt(np.diag(P)), np.sqrt(np.diag(Ps))
    corr, corr_s = P / np.outer(d, d), Ps / np.outer(ds, ds)
    assert np.abs(corr - corr_s).max() < 0.05, np.abs(corr - corr_s).max()
    print(f"C3 6.5 d: variance ratios MC/predicted {np.round(var_ratio, 4).tolist()}, max |d corr| {np.abs(corr - corr_s).max():.4f}")
