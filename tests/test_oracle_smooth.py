"""CPU checks of the smoother's ground truth: the estimate stream of the restated filter (tests/smooth_oracle.py) on the parity
matrix's inputs (tests/od_matrix.py: blunders, an absent measurement, a NOT_VISIBLE block), the restated ODSolution::smooth against an
independent numpy computation, the host build of the kernel's 9x9 part (nyx_b200/csrc/nyxb_smooth.h), and the C ABI's argument
checks."""
import copy
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from nyx_b200 import abi
from tests import od_matrix as om
from tests import smooth_oracle as so

ROOT = Path(__file__).resolve().parent.parent
S = 10**9


def run_oracle(config, variant, arc_kind="regular", filters=(1, 3), cfg_edit=None):
    """(stream per filter, filter outputs per filter, cfg, stations, tracker, obs) for the chosen filters of the matrix."""
    import nyx_b200 as nb

    prop = om.propagator(config, nb.MODE_STRICT)
    odp, cfg, _, st_c, epochs, tracker, obs, st, cs, ep, cov = om.od_inputs(config, variant, arc_kind, prop)
    if cfg_edit:
        cfg = copy.copy(cfg)
        cfg_edit(cfg)
    packed = prop.dynamics.pack(om.frame(config), om.almanac(config))
    oc = prop.opts.to_c(prop.method)
    streams, outs = [], []
    for i in filters:
        sink = []
        outs.append(so.process_arc(packed.c, oc, cfg, st_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]), st[:, i].copy(),
                                   cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy(), sink=sink))
        streams.append(sink)
    return streams, outs, cfg, st_c, tracker, obs, packed, epochs


@pytest.fixture(scope="module")
def ekf():
    return run_oracle("field", "ekf")


@pytest.mark.parametrize("config,variant,arc_kind", [(c, v, "regular") for c in ("field", "srp") for v in om.VARIANTS] +
                         [("field", "ekf", "edge"), ("field", "ckf_scalar", "edge")])
def test_sink_leaves_the_oracle_filter_unchanged(config, variant, arc_kind):
    """The restated loop with its sink gives the oracle's results bit for bit, on every filter variant, the SRP configuration and the
    edge-case arc (unknown tracker, two measurements at one epoch, a hidden station, a missing Doppler)."""
    from oracle import pyoracle_od
    import nyx_b200 as nb

    filters = (1, 3)
    _, outs, cfg, st_c, tracker, obs, packed, epochs = run_oracle(config, variant, arc_kind, filters=filters)
    prop = om.propagator(config, nb.MODE_STRICT)
    st, cs, ep, cov = om.od_inputs(config, variant, arc_kind, prop)[7:]
    for out, i in zip(outs, filters):
        ref = pyoracle_od.process_arc(packed.c, prop.opts.to_c(prop.method), cfg, st_c, epochs, tracker, np.ascontiguousarray(obs[:, :, i]),
                                      st[:, i].copy(), cs[:, i].copy(), int(ep[i]), cov[:, i].reshape(9, 9).T.copy())
        for key, v in ref.items():
            assert np.array_equal(np.asarray(out[key]), np.asarray(v), equal_nan=True), (key, i)


def test_estimate_stream_follows_the_push_points(ekf):
    streams, outs, *_ , epochs = ekf
    for stream, out, i in zip(streams, outs, (1, 3)):
        meas = [e for e in stream if e["tag"] >= 0]
        # one record per processed window, in order; rejected ones included with their bit
        processed = [k for k in range(om.N_MSR) if out["msr_flags"][k] & so.MSRF_PROCESSED]
        assert [abi.od_tag_fields(e["tag"])[0] for e in meas] == processed
        for e in meas:
            k, w, rej, M = abi.od_tag_fields(e["tag"])
            assert w == 0 and M == 2 and bool(rej) == bool(out["msr_flags"][k] & so.MSRF_REJECTED) and e["epoch"] == epochs[k]
        # nothing for the absent measurement or the NOT_VISIBLE block
        recorded = {abi.od_tag_fields(e["tag"])[0] for e in meas}
        hidden = [k for k in range(om.N_MSR) if out["msr_flags"][k] & (so.MSRF_ABSENT | so.MSRF_NOT_VISIBLE)]
        assert hidden and not recorded & set(hidden)
        if i == 3:
            assert out["msr_flags"][om.ABSENT[0]] == so.MSRF_ABSENT
        if i == 1:
            assert out["msr_flags"][om.BLUNDERS[0][0]] & so.MSRF_REJECTED
        # time updates: one per 45.5 s step chunk that does not land on a measurement epoch
        tu = [e for e in stream if e["tag"] == abi.OD_TAG_TIME_UPDATE]
        assert tu and all(e["epoch"] not in set(epochs.tolist()) for e in tu)
        assert len(stream) == len(meas) + len(tu)


def test_stm_spans_an_invisible_measurement(ekf):
    streams, outs, *_ , epochs = ekf
    stream, out = streams[0], outs[0]
    gaps = np.diff([e["epoch"] for e in stream])
    after = [j for j in range(1, len(stream)) if any(stream[j - 1]["epoch"] < epochs[k] < stream[j]["epoch"]
                                                    for k in range(om.N_MSR) if out["msr_flags"][k] & so.MSRF_NOT_VISIBLE)]
    assert after
    for j in after:                                  # the STM was not reset at the invisible measurement: 60 s, not 45.5 s or 14.5 s
        assert gaps[j - 1] == 60 * S and not np.allclose(stream[j]["stm"], np.eye(9))
    assert gaps.max() == 60 * S and set(np.unique(gaps[[j - 1 for j in range(1, len(stream)) if j not in after]])) <= {45_500_000_000, 14_500_000_000}


def test_ekf_measurement_estimates_carry_the_pre_update_nominal_and_xhat(ekf):
    streams, outs, *_ = ekf
    for stream, out in zip(streams, outs):
        for j, e in enumerate(stream):
            if e["tag"] < 0:
                assert not e["deviation"].any()          # EKF time update: zero deviation
                continue
            k, _, rej, _ = abi.od_tag_fields(e["tag"])
            if rej:
                assert not e["deviation"].any()
                continue
            assert np.abs(e["deviation"][:3]).max() > 0.0
            assert np.array_equal(so.state_of(e), out["est_state"][k])      # state() = the replaced nominal
            # the next estimate starts from the replaced nominal
            assert np.abs(stream[j]["nominal"][:3] - out["est_state"][k][:3]).max() > 0.0


def test_second_scalar_window_has_an_identity_stm():
    streams, outs, *_ = run_oracle("field", "ekf_scalar_noreject", filters=(0,))
    stream = streams[0]
    pairs = 0
    for a, b in zip(stream, stream[1:]):
        if a["tag"] >= 0 and b["tag"] >= 0 and abi.od_tag_fields(a["tag"])[0] == abi.od_tag_fields(b["tag"])[0]:
            assert abi.od_tag_fields(a["tag"])[1:] == (0, 0, 1) and abi.od_tag_fields(b["tag"])[1] == 1
            assert np.array_equal(b["stm"], np.eye(9)) and b["epoch"] == a["epoch"]
            pairs += 1
    assert pairs > 10


def _synthetic(n_est=6, seed=5):
    rng = np.random.default_rng(seed)
    ests = []
    for k in range(n_est):
        A = rng.normal(size=(9, 9))
        ests.append(dict(epoch=k * 60 * S, tag=-1, nominal=np.r_[rng.normal(7000, 1, 3), rng.normal(0, 7, 3), 1.0, 0.0, 50.0],
                         deviation=rng.normal(0, 1e-3, 9), covar=A @ A.T + 9 * np.eye(9), stm=np.eye(9) + 0.1 * rng.normal(size=(9, 9))))
    return ests


def _smooth(ests):
    filt = dict(prefit=np.zeros((0, 2)), postfit=np.zeros((0, 2)), resid_ratio=np.zeros((0, 2)))
    return so.smooth(ests, filt, 2, [], None, np.zeros(0, dtype=np.int32), np.zeros((0, 2)))


def test_smoother_uses_the_filter_estimate_k_plus_1():
    ests = _synthetic()
    sm, res, rat = _smooth(ests)
    for k in range(len(ests) - 1):
        Pi = np.linalg.inv(ests[k + 1]["stm"])
        np.testing.assert_allclose(sm[k]["covar"], Pi @ ests[k + 1]["covar"] @ Pi.T, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sm[k]["deviation"], Pi @ ests[k + 1]["deviation"], rtol=1e-12, atol=1e-15)
        assert np.array_equal(sm[k]["nominal"], ests[k]["nominal"]) and sm[k]["epoch"] == ests[k]["epoch"]
    assert sm[-1] == ests[-1] and rat[-1] is None and all(r is None for r in res)
    # a backward sweep through the SMOOTHED k+1 (the textbook shape) gives another answer at k = l - 2
    Pi1, Pi2 = np.linalg.inv(ests[-1]["stm"]), np.linalg.inv(ests[-2]["stm"])
    chained = Pi2 @ (Pi1 @ ests[-1]["covar"] @ Pi1.T) @ Pi2.T
    assert np.abs(chained - sm[-3]["covar"]).max() > 1e-3 * np.abs(chained).max()


def test_ratios_nan_on_negative_variance_difference_and_errors():
    ests = _synthetic(3)
    ests[1]["covar"] = 1e-9 * np.eye(9)                 # P_f,1 far below P_s,1 = Phi^-1 P_f,2 Phi^-T
    with np.errstate(divide="ignore", invalid="ignore"):
        _, _, rat = _smooth(ests)
    assert np.isnan(rat[1]).all() and np.isfinite(rat[0]).all()
    bad = _synthetic(3)
    bad[2]["stm"][4] = 0.0
    with pytest.raises(so.SingularSTM):
        _smooth(bad)
    with pytest.raises(ValueError):
        _smooth(_synthetic(1))
    with pytest.raises(IndexError):
        _smooth([])


def test_time_update_successor_without_snc_is_an_identity():
    def no_snc(cfg):
        cfg.snc_enabled = 0
    streams, outs, cfg, st_c, tracker, obs, packed, _ = run_oracle("field", "ckf_scalar", filters=(0,), cfg_edit=no_snc)
    stream = streams[0]
    filt = outs[0]
    sm, res, rat = so.smooth(stream, filt, 1, st_c, packed.c, tracker, obs[:, :, 0])
    n = 0
    for k in range(len(stream) - 1):
        if stream[k + 1]["tag"] != abi.OD_TAG_TIME_UPDATE:
            continue
        P = stream[k]["covar"]
        d = np.sqrt(np.outer(np.diag(P), np.diag(P)))
        live = d > 0
        assert (np.abs(sm[k]["covar"] - P)[live] / d[live]).max() < 1e-9
        assert np.abs(sm[k]["deviation"] - stream[k]["deviation"]).max() < 1e-9 * max(1.0, np.abs(stream[k]["deviation"]).max())
        n += 1
    assert n > 20


def test_residuals_are_off_by_one_with_the_bias_at_epoch_k():
    streams, outs, cfg, st_c, tracker, obs, packed, epochs = run_oracle("field", "ekf", filters=(1,))
    stream, filt = streams[0], outs[0]
    sm, res, rat = so.smooth(stream, filt, 2, st_c, packed.c, tracker, obs[:, :, 1])
    raw = [so.residual_of(e, filt, 2) for e in stream]
    assert (res[-1] is None) == (raw[-1] is None)
    if raw[-1] is not None:
        assert res[-1]["k"] == raw[-1]["k"] and np.array_equal(res[-1]["postfit"], raw[-1]["postfit"], equal_nan=True)
    checked = 0
    for k in range(len(stream) - 1):
        if raw[k + 1] is None:
            assert res[k] is None
            continue
        mk = raw[k + 1]["k"]
        gs = st_c[int(tracker[mk])]
        computed, _ = so.measure(gs, packed.c, stream[k]["epoch"], so.state_of(sm[k]))   # epoch k, smoothed state k
        if computed is None:
            assert res[k] is None
            continue
        want = obs[mk, [gs.types[q] for q in range(2)], 1] - (np.array([computed[gs.types[q]] for q in range(2)]) - np.array(list(gs.bias)))
        np.testing.assert_array_equal(res[k]["postfit"], want)
        np.testing.assert_array_equal(res[k]["prefit"], raw[k + 1]["prefit"])
        assert res[k]["ratio"] == raw[k + 1]["ratio"]
        checked += 1
    assert checked > 20
    # the statistics divide by every estimate, time updates included
    r_pre = so.rms(res, "prefit")
    some = [r for r in res if r is not None]
    assert r_pre == pytest.approx(np.sqrt(sum(float(r["prefit"] @ r["prefit"]) for r in some) / len(res)), rel=1e-15)
    assert len(some) < len(res)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so_path = tmp_path_factory.mktemp("shim") / "smooth_core_shim.so"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                    str(ROOT / "tests" / "cpp" / "smooth_core_shim.cpp"), "-o", str(so_path)], check=True, capture_output=True)
    lib = C.CDLL(str(so_path))
    lib.shim_smooth_core.restype = C.c_int
    lib.shim_smooth_core.argtypes = [C.c_void_p] * 6
    return lib


def core(shim, phi, P, x):
    Ps, xs, Pi = np.empty((9, 9)), np.empty(9), np.empty((9, 9))
    phi, P, x = (np.ascontiguousarray(a, dtype=np.float64) for a in (phi, P, x))
    rc = shim.shim_smooth_core(phi.ctypes.data, P.ctypes.data, x.ctypes.data, Ps.ctypes.data, xs.ctypes.data, Pi.ctypes.data)
    return rc, Ps, xs, Pi


def test_host_build_of_the_9x9_core_matches_the_restatement(shim, ekf):
    streams = ekf[0]
    n = 0
    for e in streams[0][1:] + _synthetic(20):
        rc, Ps, xs, Pi = core(shim, e["stm"], e["covar"], e["deviation"])
        assert rc == 0
        inv = np.linalg.inv(e["stm"])
        np.testing.assert_allclose(Pi, inv, rtol=0, atol=1e-12 * np.abs(inv).max())
        ref = inv @ e["covar"] @ inv.T
        np.testing.assert_allclose(Ps, ref, rtol=0, atol=1e-12 * np.abs(ref).max())
        np.testing.assert_allclose(xs, inv @ e["deviation"], rtol=0, atol=1e-12 * max(np.abs(e["deviation"]).max(), 1e-30) * np.abs(inv).max())
        n += 1
    assert n > 100
    # pivoting: a leading zero is no obstacle; an exactly zero pivot is singular
    perm = np.eye(9)[[1, 0, 2, 3, 4, 5, 6, 7, 8]]
    rc, _, _, Pi = core(shim, perm, np.eye(9), np.zeros(9))
    assert rc == 0 and np.array_equal(Pi, perm)
    sing = np.eye(9)
    sing[8, 8] = 0.0
    assert core(shim, sing, np.eye(9), np.zeros(9))[0] == 1


def test_abi_rejects_bad_arguments():
    lib = abi.load_library()
    assert lib.nyxb_od_smooth_batch(None, None, 0, None, None, 1, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
    cfg = abi.OdConfigC()
    assert lib.nyxb_od_ekf_record_batch(None, C.byref(cfg), 0, None, None, 1, None, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
