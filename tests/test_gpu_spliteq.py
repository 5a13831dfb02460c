"""Split-eq (Gruen) member on the device: sum_x eq(w, x) prod_j f_j(x) without materialising eq
(crates/jolt-poly/src/split_eq.rs). Oracle: the plain (m+1)-table product sumcheck over the materialised eq
table - the round polynomials are the same field values (Gruen's factorisation is a schedule, not a relation)."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (BatchMember, EqPolynomial, EqProductMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, ProductMember,
                       UnivariatePoly)
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
from gpu_util import rand_challenge, rand_limbs
import sumcheck_ref as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("m", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 9, 12])
def test_eq_member_lockstep_vs_oracle(sess, m, n, order):
    tabs = [O.random_fr(300 + 10 * m + j, 1 << n) for j in range(m)]
    w = O.random_fr(77 + n, n)
    eq_tab = O.eq_evals(w)                                    # r[0] <-> MSB (eq.rs:218-219)
    ref = O.ProductMember([eq_tab] + tabs, order)
    gpu = EqProductMember(sess, [Polynomial.from_ints(sess, t) for t in tabs], C.ints_to_mont(w), order=order)
    assert gpu.num_rounds() == n and gpu.degree() == m + 1
    claim = sum(eq_tab[i] * int(np.prod([t[i] for t in tabs], dtype=object)) for i in range(1 << n)) % O.R_MOD
    ch = O.random_fr(5, n)
    bind = None
    for rnd in range(n):
        want = ref.prove_round(bind, rnd, claim)
        got = gpu.prove_round(bind, rnd, claim)
        assert got.coefficients == want, f"round {rnd}"
        bind = ch[rnd]
        claim = got.evaluate(bind)
    ref.finish_rounds(bind)
    gpu.finish_rounds(bind)
    fe = ref.final_evals()
    assert gpu.final_evals() == fe[1:]
    assert gpu.eq_scalar() == fe[0]                          # eq(w, r) with the order's challenge-to-variable map
    assert gpu.eq_scalar() * int(np.prod(gpu.final_evals(), dtype=object)) % O.R_MOD == claim


def test_eq_member_scaled_and_challenge_point(sess):
    n, m = 8, 2
    tabs = [O.random_fr(900 + j, 1 << n) for j in range(m)]
    w_limbs = np.stack([rand_challenge(40 + i) for i in range(n)])       # 125-bit challenge point
    w = F.limbs_to_ints(w_limbs)
    scale = O.random_fr(3, 1)[0]
    eq_tab = O.eq_evals(w, scale)
    ref = O.ProductMember([eq_tab] + tabs, O.LOW_TO_HIGH)
    gpu = EqProductMember(sess, [Polynomial.from_ints(sess, t) for t in tabs], w_limbs, scale)
    claim = sum(e * a * b for e, a, b in zip(eq_tab, *tabs)) % O.R_MOD
    bind = None
    for rnd in range(n):
        want = ref.prove_round(bind, rnd, claim)
        got = gpu.prove_round(bind, rnd, claim)
        assert got.coefficients == want
        bind = F.from_limbs(rand_challenge(60 + rnd))
        claim = got.evaluate(bind)


def test_eq_member_in_the_engine_and_errors(sess):
    n, m = 10, 2
    tabs = [O.random_fr(11 + j, 1 << n) for j in range(m)]
    w = O.random_fr(9, n)
    eq_tab = O.eq_evals(w)
    claim = sum(e * a * b for e, a, b in zip(eq_tab, *tabs)) % O.R_MOD
    mem = EqProductMember(sess, [Polynomial.from_ints(sess, t) for t in tabs], C.ints_to_mont(w))
    res = jolt_b200.prove_batch_native([BatchMember(claim, 1, n, 0)], [mem], n, m + 1, claim, seed=5)
    # same proof from the plain member over the materialised eq table
    plain = ProductMember(sess, [EqPolynomial.evals(sess, C.ints_to_mont(w))] + [Polynomial.from_ints(sess, t) for t in tabs],
                          LOW_TO_HIGH)
    res2 = jolt_b200.prove_batch_native([BatchMember(claim, 1, n, 0)], [plain], n, m + 1, claim, seed=5)
    assert res.challenges == res2.challenges and res.final_claim == res2.final_claim
    assert [p.coefficients for p in res.round_polynomials] == [p.coefficients for p in res2.round_polynomials]
    assert mem.eq_scalar() == plain.final_evals()[0]
    fresh = EqProductMember(sess, [Polynomial.from_ints(sess, tabs[0])], C.ints_to_mont(w))
    with pytest.raises(jolt_b200.JoltB200Error, match="claim is required"):
        fresh.prove_round_evals(None, 0, None)
    with pytest.raises(jolt_b200.JoltB200Error, match="point length"):
        EqProductMember(sess, [Polynomial.from_ints(sess, tabs[0])], C.ints_to_mont(w[:-1]))


def eq_member_vs_c_oracle(sess, tabs, w, order, challenge):
    """Every round, the final evaluations and eq(w, r) of the split-eq member against the threaded C oracle over
    the materialised eq table (the oracle's rounds halve, so a run costs about two first rounds)."""
    n, m = len(w), len(tabs)
    thr = C.max_threads()
    gpu = EqProductMember(sess, [Polynomial.new(sess, t) for t in tabs], w, order=order)
    cur = [C.eq_evals(w, None, thr)] + list(tabs)
    bind, claim = None, None
    for rnd in range(n):
        if bind is not None:
            cur = [C.bind(t, bind, order, thr) for t in cur]
        want = C.mont_to_ints(C.product_round_evals(cur, m + 1, order, thr))
        if claim is None:
            claim = (want[0] + want[1]) % O.R_MOD
        assert (want[0] + want[1]) % O.R_MOD == claim, f"round {rnd}: the oracle's own round check"
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = challenge(rnd)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    cur = [C.bind(t, bind, order, thr) for t in cur]
    gpu.finish_rounds(bind)
    fe = [C.mont_to_ints(t)[0] for t in cur]
    assert gpu.final_evals() == fe[1:]
    assert gpu.eq_scalar() == fe[0]
    assert gpu.eq_scalar() * int(np.prod(gpu.final_evals(), dtype=object)) % O.R_MOD == claim
    gpu.close()


def test_eq_member_2pow18_vs_c_oracle(sess):
    """all 18 rounds at 2^18 against the threaded C oracle"""
    n, m = 18, 2
    tabs = [rand_limbs(0xE9 + j, 1 << n) for j in range(m)]
    eq_member_vs_c_oracle(sess, tabs, rand_limbs(0x77, n), LOW_TO_HIGH, lambda rnd: rand_challenge(3000 + rnd))


@pytest.mark.parametrize("n", [15, 16])
@pytest.mark.parametrize("m", [1, 2, 3])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_eq_member_extreme_point_every_round_vs_c_oracle(sess, n, m, order):
    """eq points with coordinates 1, p - 1 and limb-extreme values, tables over all of [0, p), extreme challenges;
    n odd and even so the inner and outer halves of the split differ in size. A zero eq factor is excluded: s(1) is
    recovered from the claim by dividing by eq(w_cur, 1) times the bound eq prefix (as the reference's
    gruen_poly), so a coordinate 0, or challenge 0 against a coordinate 1, is refused (checked below)."""
    tabs = [S.rand_limbs_full(0xE16 + 10 * m + j, 1 << n) for j in range(m)]
    w = S.extreme_point(0x3E + n, n, zero=False)

    def challenge(rnd):
        ch = S.extreme_challenge(rnd, n)
        return ch if ch.any() else S.EXTREME_CHALLENGES[2]
    eq_member_vs_c_oracle(sess, tabs, w, order, challenge)
    # a zero eq factor at the current variable is an error, never a wrong round
    w0 = w.copy()
    w0[n - 1 if order == LOW_TO_HIGH else 0] = 0
    gpu = EqProductMember(sess, [Polynomial.new(sess, t) for t in tabs], w0, order=order)
    with pytest.raises(jolt_b200.JoltB200Error, match="must be invertible"):
        gpu.prove_round_evals(None, 0, 1)
    gpu.close()
