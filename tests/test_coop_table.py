"""Host logic of the lane-cooperative FAST kernel, checked on the CPU: the column -> lane schedule and the packed
coefficient records (`nyxb_coop_build_host`, csrc/nyxb_coop.cu) are walked here exactly as `coop_rhs`
(csrc/nyxb_coop_kernel.cuh) walks them, and the resulting acceleration is compared with the oracle's
`GravityField::eom` restatement (gravity_field.rs:148-268).  No device is needed: `nyxb_coop_table_dump` is host-only."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi


def _dump(packed, lanes):
    lib = abi.load_library()
    gf = packed.c.gravity.contents
    L, kmax = C.c_int32(), C.c_int32()
    assert lib.nyxb_coop_table_dump(C.byref(gf), lanes, C.byref(L), C.byref(kmax), None, None, None, None) == 0
    L, kmax, N = L.value, kmax.value, gf.degree
    recs = np.zeros((L + 2) * lanes * 5)
    cs = np.zeros(lanes * kmax, dtype=np.int32)
    cm = np.zeros(lanes * kmax, dtype=np.int32)
    seed = np.zeros((N + 2) * 4)
    assert lib.nyxb_coop_table_dump(C.byref(gf), lanes, C.byref(C.c_int32()), C.byref(C.c_int32()), recs.ctypes.data,
                                    cs.ctypes.data, cm.ctypes.data, seed.ctypes.data) == 0
    return L, kmax, recs.reshape((L + 2) // 2, 5, lanes, 2), cs.reshape(lanes, kmax), cm.reshape(lanes, kmax), seed.reshape(N + 2, 4)


def _walk(gf, lanes, tables, rb):
    """One harmonic evaluation for the body-fixed position rb, lane by lane (same algebra as coop_rhs)."""
    L, kmax, recs, col_start, col_m, seed = tables
    N = gf.degree
    r = float(np.linalg.norm(rb))
    inv_r = 1.0 / r
    rho = gf.r_eq_km * inv_r
    s_, t_, u_ = rb * inv_r
    ub, r2 = u_ * rho, rho * rho
    z = complex(s_, t_)
    rm = np.array([(z**k).real for k in range(N + 2)])
    im = np.array([(z**k).imag for k in range(N + 2)])
    seed = np.vstack([seed, np.zeros(4)])   # row N + 2: the zero seed of the stop column
    rp = np.array([rho**k * seed[k, 0] for k in range(N + 3)])
    X = Y = Z = W = 0.0
    for lane in range(lanes):
        starts = {int(col_start[lane, k]): int(col_m[lane, k]) for k in range(kmax) if col_start[lane, k] <= L}
        Q1 = Q2 = rr = ii = al = be = 0.0
        S = [0.0] * 6

        def fold():
            nonlocal X, Y, Z, W
            X += rr * S[0] + ii * S[1]
            Y += rr * S[1] - ii * S[0]
            Z += rr * S[2] + ii * S[3]
            W += rr * S[4] + ii * S[5]

        for e in range(0, L, 2):
            if e in starts:
                fold()
                m = starts[e]
                Q1, Q2, rr, ii = rp[m], 0.0, rm[m - 1], im[m - 1]
                al, be = seed[m, 3], 0.0
                S = [0.0, 0.0, 0.0, 0.0, Q1 * seed[m, 1], Q1 * seed[m, 2]]
            pair = recs[e // 2, :, lane, :]
            for h in range(2):
                p1, p2 = pair[2 * h]
                p3, p4 = pair[2 * h + 1]
                kap = pair[4, h]
                S[0] += Q1 * p1; S[1] += Q1 * p2; S[2] += Q1 * p3; S[3] += Q1 * p4
                Qn = al * ub * Q1 - be * r2 * Q2
                S[4] += kap * Qn * p3; S[5] += kap * Qn * p4
                Q2, Q1 = Q1, Qn
                be += al; al += 2.0
        fold()
    K0 = gf.mu_km3_s2 / gf.r_eq_km * inv_r
    K1 = K0 * rho
    aw = -K0 * W
    return np.array([aw * s_ + K1 * X, aw * t_ + K1 * Y, aw * u_ + K1 * Z])


@pytest.mark.parametrize("fixture,degree,order,lanes", [("jgm3_70x70", 21, 21, 8), ("jgm3_70x70", 21, 21, 16), ("jgm3_70x70", 8, 5, 8),
                                                          ("jgm3_70x70", 70, 70, 32), ("jgm3_70x70", 30, 30, 32), ("luna_jggrx_80x80", 48, 48, 16),
                                                          ("jgm3_70x70", 8, 0, 8), ("jgm3_70x70", 8, 1, 8), ("jgm3_70x70", 8, 0, 32),
                                                          ("jgm3_70x70", 29, 29, 8), ("jgm3_70x70", 30, 30, 16), ("jgm3_70x70", 40, 40, 16),
                                                          ("jgm3_70x70", 41, 41, 16), ("jgm3_70x70", 47, 47, 16), ("jgm3_70x70", 48, 48, 32)])
def test_cooperative_table_reproduces_oracle_gravity(oracle, fixture, degree, order, lanes):
    """The schedule is the bin packing with aligned column starts (columns reordered / idle gaps inserted so that lane positions
    start columns on common entries)."""
    moon = fixture.startswith("luna")
    body_frame = nb.IAU_MOON_FRAME if moon else nb.IAU_EARTH_FRAME
    gd = nb.GravityFieldData.from_fixture(fixture, degree, order, body_frame.with_rotation(None) if hasattr(body_frame, "with_rotation") else body_frame)
    check_table(oracle, gd, nb.MOON_J2000 if moon else nb.EARTH_J2000, lanes)


def check_table(oracle, gd, frame, lanes, radii=(1.03, 1.6), points=4):
    """Schedule invariants of the field `gd` at `lanes`, and the walk against the oracle's harmonic acceleration at `points`
    points between radii[0] and radii[1] x r_eq."""
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    packed = dyn.pack(frame, None)
    gf = packed.c.gravity.contents
    gf.rot.kind = 0   # identity rotation: the harmonic sum is exercised directly in the integration frame
    tables = _dump(packed, lanes)
    L, kmax, recs, col_start, col_m, seed = tables
    # schedule invariants: even column boundaries, every column m = 1..min(order, degree)+1 present exactly once, and stop columns
    # (m = N + 2, zero seed) only where a column is followed by an idle gap
    real = col_start <= L
    assert L % 2 == 0 and (col_start[real] % 2 == 0).all()
    cols = col_m[real & (col_m != gf.degree + 2)]
    assert sorted(cols.tolist()) == list(range(1, min(gf.order + 1, gf.degree + 1) + 1))
    for lane in range(lanes):   # columns of a lane do not overlap and end inside the walk
        ends = 0
        for k in range(kmax):
            if col_start[lane, k] > L:
                continue
            m = int(col_m[lane, k])
            ln = max(gf.degree + 1 - m, 1)
            assert col_start[lane, k] >= ends
            ends = int(col_start[lane, k]) + ln + (ln & 1)
        assert ends <= L
    rng = np.random.default_rng(5)
    R = gf.r_eq_km
    for _ in range(points):
        d = rng.normal(size=3)
        rb = d / np.linalg.norm(d) * R * rng.uniform(*radii)
        y = np.concatenate([rb, [0.0, 0.0, 0.0, 1.8, 2.2, 0.0]])
        consts = np.array([100.0, 0.0, 1.0, 1.0])
        dy = np.zeros(9)
        L_ = oracle.lib()
        assert L_.nyx_oracle_eom(C.byref(packed.c), 0, 0.0, abi.as_double_p(y), abi.as_double_p(consts), abi.as_double_p(dy)) == 0
        two_body = -packed.c.mu_central_km3_s2 / np.linalg.norm(rb) ** 3 * rb
        want = dy[3:6] - two_body
        got = _walk(gf, lanes, tables, rb)
        # `want` carries the rounding of the full acceleration it was subtracted from (two-body is ~1e3 x larger)
        assert np.abs(got - want).max() < 1e-13 * np.abs(want).max() + 1e-15 * np.abs(two_body).max(), (got, want)
