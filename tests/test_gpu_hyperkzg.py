"""HyperKZG prover side on the device vs the oracle (mirrors crates/jolt-hyperkzg/src/scheme.rs:382-417,
tests/commit_open_verify.rs:50-188 on the prover side), every proof also checked by the reference verifier
(tests/hyperkzg_ref.py) over a power SRS whose secret the test knows. G1 results are compared as affine (x, y)
integers."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import G1Bases, HyperKZG, Polynomial, g1_jacobian_to_affine
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
import hyperkzg_ref as HK
from gpu_util import rand_challenge, rand_limbs

pytestmark = pytest.mark.gpu

G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.mark.parametrize("ell,precompute", [(1, False), (2, False), (3, True), (5, False), (8, True), (11, False),
                                            (14, False), (14, True), (4, True), (16, True), (17, True)])
def test_open_matches_oracle(sess, ell, precompute):
    n = 1 << ell
    tau = O.random_fr(0x4D534D, 1)[0]
    beta = C.ints_to_mont([tau])[0]
    srs_xy = C.g1_powers(n, G, beta) if ell <= 11 else C.g1_powers_fast(n, G, beta)
    bases = G1Bases.from_affine(sess, srs_xy)
    if precompute:       # fixed-SRS tables: shared buckets for the large MSMs, the 8-bit table for the small ones
        bases.precompute()
    evals = rand_limbs(100 + ell, n)
    point = np.stack([rand_challenge(7 + i) if i % 2 else rand_limbs(9 + i, 1)[0] for i in range(ell)])
    r_int, q_int = O.random_fr(1000 + ell, 2)
    seen = {}

    def ch_r(com):
        seen["com"] = [g1_jacobian_to_affine(c) for c in com]
        return r_int

    def ch_q(v):
        seen["v"] = v
        return q_int

    poly = Polynomial.new(sess, evals)
    commitment = g1_jacobian_to_affine(HyperKZG.commit(bases, poly))
    assert commitment == HK.oracle_affine(*C.g1_msm_pippenger(srs_xy, evals, 0, C.max_threads()))
    proof = HyperKZG.open(bases, poly, point, ch_r, ch_q)
    com, w, v = HK.oracle_open(srs_xy, evals, point, r_int, q_int)
    assert seen["com"] == com and [g1_jacobian_to_affine(c) for c in proof.com] == com
    assert proof.v == v and seen["v"] == v
    assert [g1_jacobian_to_affine(x) for x in proof.w] == w
    # the table is untouched by open (the reference borrows `evals`)
    assert (poly.evals() == evals).all()
    # the proof verifies for y = the multilinear evaluation at the point, and not for any other y
    y = HK.host_eval(evals, point)
    if ell <= 8:
        assert y == O.evaluate(C.mont_to_ints(evals), F.limbs_to_ints(point))
    pt = F.limbs_to_ints(point)
    d0 = O.random_fr(2000 + ell, 1)[0]
    assert HK.verify(tau, commitment, pt, y, com, w, v, r_int, q_int, d0)
    assert not HK.verify(tau, commitment, pt, (y + 1) % O.R_MOD, com, w, v, r_int, q_int, d0)


def test_open_rejects_bad_input(sess):
    bases = G1Bases.generate_multiples(sess, G, 8)
    poly = Polynomial.new(sess, rand_limbs(1, 16))
    with pytest.raises(jolt_b200.JoltB200Error, match="SrsTooSmall"):
        HyperKZG.open(bases, poly, rand_limbs(2, 4), lambda c: 1, lambda v: 1)
    with pytest.raises(jolt_b200.JoltB200Error, match="2\\^ell"):
        HyperKZG.open(G1Bases.generate_multiples(sess, G, 16), poly, rand_limbs(2, 3), lambda c: 1, lambda v: 1)
    with pytest.raises(jolt_b200.JoltB200Error, match="EmptyPoint"):
        HyperKZG.open(bases, Polynomial.new(sess, rand_limbs(1, 1)), np.zeros((0, 4), dtype=np.uint64), lambda c: 1, lambda v: 1)


def test_commit_homomorphism(sess):
    # commit(a P + b Q) == a commit(P) + b commit(Q)  (tests/commit_open_verify.rs:131-188)
    n = 1 << 10
    bases = G1Bases.generate_multiples(sess, G, n)
    P, Q = rand_limbs(1, n), rand_limbs(2, n)
    a, b = O.random_fr(3, 2)
    comb = C.f_vec(0, 0, C.f_vec(0, 2, P, np.tile(C.ints_to_mont([a]), (n, 1))), C.f_vec(0, 2, Q, np.tile(C.ints_to_mont([b]), (n, 1))))
    cp, cq, cc = (g1_jacobian_to_affine(HyperKZG.commit(bases, Polynomial.new(sess, x))) for x in (P, Q, comb))
    assert cc == O.g1_add(O.g1_scalar_mul(cp, a), O.g1_scalar_mul(cq, b))
