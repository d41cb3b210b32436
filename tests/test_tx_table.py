"""Host logic of the transposed kernel (csrc/nyxb_tx.cu), checked on the CPU: the zigzag column -> position schedule and the
records of `nyxb_tx_build_host` are walked here exactly as `nyxb_k_tx` walks them — binary powering with the position's two
interleaved exponent sequences, one complex multiplication per column, recursion coefficients advanced by
additions, columns padded to an even number of entries —
and the resulting acceleration is compared with the oracle's `GravityField::eom` restatement (gravity_field.rs:148-268).
No device is needed: `nyxb_tx_table_dump` is host-only."""
import ctypes as C

import numpy as np
import pytest

import nyx_b200 as nb
from nyx_b200 import abi


def _dump(gf, P):
    lib = abi.load_library()
    n_rec, kmax = C.c_int32(), C.c_int32()
    assert lib.nyxb_tx_table_dump(C.byref(gf), P, C.byref(n_rec), C.byref(kmax), None, None, None, None) == 0
    n_rec, kmax, N = n_rec.value, kmax.value, gf.degree
    recA = np.zeros((n_rec + 1) * 4)
    recK = np.zeros(n_rec + 2)
    seed = np.zeros((N + 2) * 4)
    sched = np.zeros(P * (2 + 2 * kmax), dtype=np.int32)
    assert lib.nyxb_tx_table_dump(C.byref(gf), P, C.byref(C.c_int32()), C.byref(C.c_int32()), recA.ctypes.data, recK.ctypes.data,
                                  seed.ctypes.data, sched.ctypes.data) == 0
    return n_rec, kmax, recA.reshape(n_rec + 1, 4), recK, seed.reshape(N + 2, 4), sched.reshape(P, 2 + 2 * kmax)


def _walk(gf, P, tables, rb):
    """One harmonic evaluation for the body-fixed position rb, position by position (same algebra as nyxb_k_tx)."""
    n_rec, kmax, recA, recK, seed, sched = tables
    r = float(np.linalg.norm(rb))
    inv_r = 1.0 / r
    rho = gf.r_eq_km * inv_r
    ub, r2 = rb[2] * inv_r * rho, rho * rho
    X = Y = Z = W = 0.0
    z1 = complex(rb[0] * inv_r, rb[1] * inv_r)
    zq, rq = z1 ** (2 * P), rho ** (2 * P)   # common ratio of both sequences
    for w in range(P):
        # za = z^w, zb = z^(2P-1-w), pa = rho^(w+1), pb = rho^(2P-w): published by the helpers (P = 8, 10) or assembled from
        # z^(2^k) by the walker (P = 16)
        za, zb = z1 ** w, z1 ** (2 * P - 1 - w)
        pa, pb = rho ** (w + 1), rho ** (2 * P - w)
        e = int(sched[w, 0])
        for k in range(int(sched[w, 1])):
            m, ln = int(sched[w, 2 + 2 * k]), int(sched[w, 3 + 2 * k])
            assert abs(za - z1 ** (m - 1)) < 1e-12 and abs(pa / rho ** m - 1.0) < 1e-12
            Q = pa * seed[m, 0]
            al = seed[m, 3]
            c1, m2, d, g = al * ub, 0.0, 0.0, al * r2
            S = [0.0, 0.0, 0.0, 0.0, Q * seed[m, 1], Q * seed[m, 2]]
            for _ in range(ln):
                p1, p2, p3, p4 = recA[e]
                ck = recK[e]
                e += 1
                Qn = c1 * Q - m2
                c1 += 2 * ub; d += g; g += 2 * r2
                m2 = d * Q
                S[0] += Q * p1; S[1] += Q * p2; S[2] += Q * p3; S[3] += Q * p4
                wv = ck * Qn
                S[4] += wv * p3; S[5] += wv * p4
                Q = Qn
            rr, ii = za.real, za.imag
            X += rr * S[0] + ii * S[1]
            Y += rr * S[1] - ii * S[0]
            Z += rr * S[2] + ii * S[3]
            W += rr * S[4] + ii * S[5]
            za, zb, pa, pb = zb, za * zq, pb, pa * rq
    s_, t_, u_ = rb * inv_r
    K0 = gf.mu_km3_s2 / gf.r_eq_km * inv_r
    K1 = K0 * rho
    aw = -K0 * W
    return np.array([aw * s_ + K1 * X, aw * t_ + K1 * Y, aw * u_ + K1 * Z])


@pytest.mark.parametrize("fixture,degree,order,P", [("jgm3_70x70", 21, 21, 8), ("jgm3_70x70", 21, 21, 10), ("jgm3_70x70", 8, 5, 8), ("jgm3_70x70", 12, 12, 8),
                                                      ("jgm3_70x70", 40, 40, 8), ("jgm3_70x70", 70, 70, 16), ("luna_jggrx_80x80", 48, 48, 16),
                                                      ("jgm3_70x70", 33, 20, 16), ("jgm3_70x70", 8, 0, 8), ("jgm3_70x70", 8, 1, 8),
                                                      ("jgm3_70x70", 8, 0, 16), ("jgm3_70x70", 40, 40, 16), ("jgm3_70x70", 41, 41, 16),
                                                      ("jgm3_70x70", 41, 41, 8), ("jgm3_70x70", 30, 30, 10), ("jgm3_70x70", 48, 48, 16)])
def test_transposed_table_reproduces_oracle_gravity(oracle, fixture, degree, order, P):
    moon = fixture.startswith("luna")
    body_frame = nb.IAU_MOON_FRAME if moon else nb.IAU_EARTH_FRAME
    gd = nb.GravityFieldData.from_fixture(fixture, degree, order, body_frame)
    dyn = nb.SpacecraftDynamics.new(nb.OrbitalDynamics.from_model(nb.GravityField.new(gd)))
    packed = dyn.pack(nb.MOON_J2000 if moon else nb.EARTH_J2000, None)
    gf = packed.c.gravity.contents
    gf.rot.kind = 0   # identity rotation: the harmonic sum is exercised directly in the integration frame
    tables = _dump(gf, P)
    n_rec, kmax, recA, recK, seed, sched = tables
    # schedule invariants: every column m = 1..min(order, degree)+1 exactly once, positions contiguous in the record table,
    # exponents of a position alternate between its two sequences
    ms, e = [], 0
    for w in range(P):
        assert sched[w, 0] == e
        assert sched[w, 2 + 2 * sched[w, 1]] == 0 and sched[w, 3 + 2 * sched[w, 1]] == 0   # null column behind the last one
        for k in range(sched[w, 1]):
            m, ln = int(sched[w, 2 + 2 * k]), int(sched[w, 3 + 2 * k])
            assert ln == (max(degree + 1 - m, 1) + 1) // 2 * 2
            assert (m - 1) == (w if k % 2 == 0 else 2 * P - 1 - w) + 2 * P * (k // 2)
            ms.append(m); e += ln
    assert e == n_rec and sorted(ms) == list(range(1, min(gf.order + 1, gf.degree + 1) + 1))
    assert (recA[n_rec] == 0).all() and recK[n_rec] == 0   # null record behind the last entry (prefetch target)
    rng = np.random.default_rng(7)
    for _ in range(4):
        d = rng.normal(size=3)
        rb = d / np.linalg.norm(d) * gf.r_eq_km * rng.uniform(1.03, 1.6)
        y = np.concatenate([rb, [0.0, 0.0, 0.0, 1.8, 2.2, 0.0]])
        consts = np.array([100.0, 0.0, 1.0, 1.0])
        dy = np.zeros(9)
        assert oracle.lib().nyx_oracle_eom(C.byref(packed.c), 0, 0.0, abi.as_double_p(y), abi.as_double_p(consts), abi.as_double_p(dy)) == 0
        two_body = -packed.c.mu_central_km3_s2 / np.linalg.norm(rb) ** 3 * rb
        want = dy[3:6] - two_body
        got = _walk(gf, P, tables, rb)
        # `want` carries the rounding of the full acceleration it was subtracted from (two-body is ~1e3 x larger)
        assert np.abs(got - want).max() < 1e-13 * np.abs(want).max() + 1e-15 * np.abs(two_body).max(), (got, want)
