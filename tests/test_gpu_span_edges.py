"""The step bookkeeping of every kernel family at the edges of a span, against the oracle and the exact integer model
(tests/span_edges.py; the CPU side is tests/test_span_edges_inputs.py).

Families, each forced and checked with `last_kernel()`:
  K1-S / K1-F         per-thread kernel, STRICT / FAST
  K2-G8 / G16 / G32   lane-cooperative FAST kernel, 8 / 16 / 32 lanes per trajectory
  K3-G8 / G16 / G32   lane-cooperative STRICT kernel
  K5-P8 / P10 / P16   transposed kernel, 8 / 10 / 16 walker positions; K5-sliced: 5 attempts per time slice on one CTA
  OD-S / OD-F         the OD arc's propagation, through nyxb_propagate_batch_stm with the step array carried between calls, and
                      through the covariance prediction (predict_ensemble_until) at chunk ends that miss the end epoch
Two-body cases run on K1 and the OD path; JGM-3 21x21 + Moon / Sun cases on every family.

Exact, per call of a chained case, against the oracle and the integer model: the status word (WARN_MAX_ATTEMPTS included), the
final epochs, the step array handed back, details n_steps / n_rejected / attempts / step_ns (and n_rhs against the oracle), the
recorded epochs and their count, with a sink just large enough and with one exactly one record too small.
States: STRICT bit-equal to the oracle (on these cases the controller's pow only feeds clamped proposals, so its last-ulp difference
with glibc cannot reach a state); FAST within fast_matrix.bounds of the method (scaled by |r| / 7 000 km where
a state leaves low orbit: only huge_saturating, whose final cut step lasts up to two days); two-body on K1 and OD within the case's Kepler bound
(twice the oracle's own distance from the 40-digit solution, and at least that distance plus the FAST bound).  FAST STMs within
1e-7 of their largest entry, FAST prediction records within the tolerances of tests/test_gpu_predict.py."""
import numpy as np
import pytest

import nyx_b200 as nb
from tests import span_edges as se
from tests.fast_matrix import bounds
from tests.test_gpu_fast_matrix import force_family
from tests.util import max_dr_dv

pytestmark = pytest.mark.gpu

FAMILIES = ("K1-S", "K1-F", "K2-G8", "K2-G16", "K2-G32", "K3-G8", "K3-G16", "K3-G32", "K5-P8", "K5-P10", "K5-P16", "K5-sliced")
KERNEL = {"K1": nb.KERNEL_THREAD, "K2": nb.KERNEL_COOP, "K3": nb.KERNEL_COOP, "K5": nb.KERNEL_TRANSPOSED}
PARAMS = [(f, c.name) for f in FAMILIES for c in se.CASES if c.dyn == "jgm3" or f.startswith("K1")]
MAXIMA = {}


def strict(family):
    return family in ("K1-S", "OD-S") or family.startswith("K3")


def engine(case, family):
    mode = nb.MODE_STRICT if strict(family) else nb.MODE_FAST
    eng = se.propagator(case, mode).engine(nb.EARTH_J2000, se.almanac(case.dyn, case.t0))
    kind, _, arg = family.partition("-")
    if kind == "K3":
        eng.set_kernel(nb.KERNEL_COOP)
        eng.set_lanes(int(arg[1:]))
    elif kind == "OD":
        eng.set_kernel(nb.KERNEL_THREAD)
    else:
        force_family(eng, family.replace("K1-S", "K1").replace("K1-F", "K1"))
    return eng


def check_states(tag, family, case, got, ref):
    if strict(family):
        same = (got == ref).all(axis=0)
        assert same.all(), (tag, np.flatnonzero(~same)[:8], max_dr_dv(got, ref))
        dr = dv = 0.0
    else:
        dr, dv = max_dr_dv(got, ref)
        # the bounds hold at LEO radius; round-off scales with the state (huge_saturating's cut step of two days leaves the orbit)
        scale = max(1.0, float(np.sqrt((ref[:3] ** 2).sum(0)).max()) / 7000.0)
        bdr, bdv = (b * scale for b in bounds(case.method))
        assert dr < bdr and dv < bdv, (tag, dr, dv)
    m = MAXIMA.setdefault(family, [0.0, 0.0])
    m[0], m[1] = max(m[0], dr), max(m[1], dv)
    return dr, dv


def check_call(tag, case, model_call, g, r, exact_records=True):
    """bookkeeping of one call: GPU g against oracle r and the integer model; g, r = (state, epoch, details, status, step, rec)"""
    st, ep, det, status, step, rec = g
    assert np.array_equal(status, r[3]), (tag, "status", status, r[3])
    assert np.array_equal(ep, r[1]), (tag, "epoch")
    assert np.array_equal(step, r[4]), (tag, "step array", np.flatnonzero(step != r[4])[:8], step[step != r[4]][:4], r[4][step != r[4]][:4])
    for f in ("n_steps", "n_rejected", "attempts", "step_ns", "n_rhs"):
        assert np.array_equal(det[f], r[2][f]), (tag, f, np.flatnonzero(det[f] != r[2][f])[:8])
    want = {f: np.array([m[f] for m in model_call]) for f in ("epoch", "step", "det_step", "attempts", "n_steps", "n_rejected", "warn")}
    assert np.array_equal(ep, want["epoch"]) and np.array_equal(step, want["step"]), tag
    assert np.array_equal(det["step_ns"], want["det_step"]) and np.array_equal(det["attempts"], want["attempts"]), tag
    assert np.array_equal(det["n_steps"], want["n_steps"]) and np.array_equal(det["n_rejected"], want["n_rejected"]), tag
    assert np.array_equal((status & nb.abi.WARN_MAX_ATTEMPTS) != 0, want["warn"]) and ((status & 0xFF) == 0).all(), tag
    if rec is not None:
        assert np.array_equal(rec[2], r[5][2]), (tag, "record count")
        assert np.array_equal(rec[0], r[5][0]), (tag, "record epochs")
        for i, m in enumerate(model_call):
            assert rec[0][: rec[2][i], i].tolist() == m["records"], (tag, "record epochs vs model", i)


@pytest.mark.parametrize("family,name", PARAMS, ids=[f"{f}-{n}" for f, n in PARAMS])
def test_propagate_span_edges(oracle, family, name):
    case = se.CASE[name]
    ref = se.oracle_chain(name)
    cap = se.capacity(case)
    eng = engine(case, family)

    def run(st, cs, ep, end, step, cap_):
        out = eng.propagate_batch(st, cs, ep, end, step, traj_capacity=cap_)
        assert eng.last_kernel() == KERNEL[family[:2]], (family, eng.last_kernel())
        return out

    got = se.chain(run, case, cap=cap)
    for k, (g, r, mc) in enumerate(zip(got, ref, se.model(case))):
        tag = f"{family} {name} call{k}"
        check_call(tag, case, mc, g, r)
        dr, dv = check_states(tag, family, case, g[0], r[0])
        cnt = g[5][2]
        for i in range(case.size):   # every recorded state
            c = int(cnt[i])
            check_states(tag + " records", family, case, g[5][1][:, :c, i], r[5][1][:, :c, i])
        print(f"SPANEDGES {tag} dr={dr:.3e} dv={dv:.3e}")
    if case.dyn == "twobody" and name in se.KEPLER_CASES:
        d = se.kepler_distance(name, got[-1][0])
        assert d < se.kepler_bound(name), (family, name, d, se.kepler_bound(name))
        print(f"SPANEDGES {family} {name} kepler |dr|={d:.3e} bound={se.kepler_bound(name):.3e}")
    # a sink exactly one record too small: the head of the stream is kept, the count is the capacity, nothing else changes
    st, cs = se.ensemble(case.size)
    small = eng.propagate_batch(st, cs, case.epoch0(), case.ends()[0], np.full(case.size, case.first_step(), dtype=np.int64),
                                traj_capacity=cap - 1)
    full = got[0]
    assert np.array_equal(small[4][2], np.minimum(full[5][2], cap - 1))
    assert np.array_equal(small[4][0], full[5][0][: cap - 1]) and np.array_equal(small[4][1], full[5][1][:, : cap - 1])
    assert np.array_equal(small[0], full[0]) and np.array_equal(small[1], full[1]) and np.array_equal(small[3], full[3])


@pytest.mark.parametrize("family", ("OD-S", "OD-F"))
@pytest.mark.parametrize("name", list(se.CASE))
def test_stm_span_edges(oracle, family, name):
    case = se.CASE[name]
    ref = se.oracle_stm_chain(name)
    eng = engine(case, family)

    def run(st, cs, ep, end, step, cap_):
        s, e, stm, det, status = eng.propagate_batch_stm(st, cs, ep, end, step_ns=step)
        return s, e, det, status, stm

    got = se.chain(run, case, cap=1)
    for k, (g, r, mc) in enumerate(zip(got, ref, se.model(case))):
        tag = f"{family} {name} call{k}"
        check_call(tag, case, mc, g[:5] + (None,), r[:5] + (None,))
        dr, dv = check_states(tag, family, case, g[0], r[0])
        if strict(family):
            assert np.array_equal(g[5], r[5]), (tag, "stm")
        else:
            assert np.abs(g[5] - r[5]).max() <= 1e-7 * np.abs(r[5]).max(), (tag, "stm", np.abs(g[5] - r[5]).max())
        print(f"SPANEDGES {tag} dr={dr:.3e} dv={dv:.3e}")
    if case.dyn == "twobody" and name in se.KEPLER_CASES:
        d = se.kepler_distance(name, got[-1][0])
        assert d < se.kepler_bound(name), (family, name, d, se.kepler_bound(name))


@pytest.mark.parametrize("family", ("OD-S", "OD-F"))
@pytest.mark.parametrize("pname", list(se.PREDICT))
def test_predict_span_edges(oracle, family, pname):
    from tests import predict_oracle

    _, case, chunk, _ = se.PREDICT[pname]
    odp = se.predict_process(pname, nb.MODE_STRICT if strict(family) else nb.MODE_FAST)
    engine_ = odp.prop.engine(nb.EARTH_J2000, se.almanac(case.dyn, case.t0))
    engine_.set_kernel(nb.KERNEL_THREAD)
    inputs = se.predict_inputs(pname)
    ests = [x[1] for x in inputs]
    sol = odp.predict_ensemble_until(ests, np.array([x[3] for x in inputs], dtype=np.int64))
    assert engine_.last_kernel() == nb.KERNEL_THREAD
    tr, tv = (1e-9, 1e-12) if strict(family) else (1e-7, 1e-10)
    for i, (sc, est, cs, end) in enumerate(inputs):
        ref = predict_oracle.predict_until(*se.predict_oracle_args(pname), sc.to_vector(), cs, sc.epoch(), est.covar, end)
        rec, run = se.model_predict(case, chunk, sc.epoch(), end)
        tag = f"{family} {pname} run{i}"
        assert sol.status[i] == ref["status"] == 0, tag
        assert sol.rec_count[i] == ref["count"] == len(rec), (tag, sol.rec_count[i], ref["count"], len(rec))
        assert sol.record_epochs(i).tolist() == ref["rec_epoch"].tolist() == rec, tag
        assert sol.final_epoch_ns[i] == ref["epoch"] == run.epoch, tag
        assert sol.details["n_steps"][i] == ref["n_steps"] == run.n_steps, (tag, sol.details["n_steps"][i], ref["n_steps"], run.n_steps)
        K = ref["count"]
        rs = sol.rec_state[:K, :, i]
        dr, dv = np.abs(rs[:, :3] - ref["rec_state"][:, :3]).max(), np.abs(rs[:, 3:6] - ref["rec_state"][:, 3:6]).max()
        assert dr < tr and dv < tv, (tag, dr, dv)
        if strict(family):   # ReferenceUpdate: the recorded state is the integrated one, bit for bit
            assert np.array_equal(rs[:, :6], ref["rec_state"][:, :6]), (tag, "STRICT record states")
        print(f"SPANEDGES {tag} records={K} dr={dr:.3e} dv={dv:.3e}")


def test_zz_report_maxima():
    """per-family maxima of the comparisons above (printed; the bounds are asserted where they are measured)"""
    for fam, (dr, dv) in sorted(MAXIMA.items()):
        print(f"SPANEDGES maxima {fam}: |dr| {dr:.2e} km, |dv| {dv:.2e} km/s")
