"""Expression members on the device (jb_member_create_expr): every round polynomial, the final evaluations and
eq(w, r) in lockstep with tests/expr_ref.py; full-size checks by linearity against the built members; the batch
engine and the scheduler with expression members mixed into the batch; routing of built shapes; every error."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (BatchMember, EqPolynomial, EqProductMember, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial,
                       ProductMember, RoundScheduler, SumOfProductsMember, UnivariatePoly, _lib)
from jolt_b200 import field as F
from oracle import bn254 as O
from gpu_util import rand_challenge, rand_limbs
import expr_ref as E
import sumcheck_ref as S

pytestmark = pytest.mark.gpu
P = O.R_MOD
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
R_LIMBS_COEFF = S.int_to_limbs(S.R_MONT)   # Montgomery limbs R: the value 1
PM1_LIMBS_COEFF = S.int_to_limbs(P - 1)    # Montgomery limbs p - 1
# name -> (tables, monomials, eq)
SHAPES = {
    "booleanity": (1, [(1, [0, 0]), (-1, [0])], True),
    "ab_minus_c": (3, [(1, [0, 1]), (-1, [2])], True),
    "rw_shared": (4, [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA % P, [1, 3])], True),
    "square_in_product": (2, [(1, [0, 0, 1])], False),
    "square_in_product_eq": (3, [(GAMMA, [0, 1, 1]), (1, [2])], True),
    "degree6_eq": (4, [(GAMMA, [0, 1, 2, 3, 0, 1])], True),
    "degree1": (1, [(7, [0])], False),
    "zero_coeff": (3, [(0, [0, 1]), (1, [1, 2]), (3, [2])], False),
    "extreme_coeffs": (3, [(P - 1, [0, 1]), (PM1_LIMBS_COEFF, [1, 2]), (R_LIMBS_COEFF, [2, 0]), ((1 << 256) % P, [1])], False),
}


def _coeff_int(c):
    return c % P if isinstance(c, int) else F.from_limbs(c)


def _ref_monomials(monomials):
    return [(_coeff_int(c), t) for c, t in monomials]


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sess_verify():
    s = jolt_b200.Session(0)
    s.set_verify_rounds(True)
    yield s
    s.close()


def _tables(seed, T, n, order):
    if n >= 9:
        return [S.extreme_table(seed + j, n, order, rotate=j) for j in range(T)]
    return [S.rand_limbs_full(seed + j, 1 << n) for j in range(T)]


def _challenge(rnd, seed):
    ch = S.extreme_challenge(rnd, seed)   # 125-bit and full challenges, interleaved with the extreme ones
    return ch if ch.any() else S.EXTREME_CHALLENGES[2]   # (a zero challenge against an eq coordinate 1 zeroes eq)


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 9, 12])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_expr_lockstep_vs_reference(sess, sess_verify, shape, n, order, verify):
    T, monomials, eq = SHAPES[shape]
    s = sess_verify if verify else sess
    tabs = _tables(0xE400 + 16 * n, T, n, order)
    w = S.extreme_point(0x3E + n, n, zero=False) if eq else None
    ref = E.ExpressionMember([F.limbs_to_ints(t) for t in tabs], _ref_monomials(monomials), order,
                             None if w is None else F.limbs_to_ints(w))
    gpu = ExpressionMember(s, [Polynomial.new(s, t) for t in tabs], monomials, w, order=order)
    assert gpu.num_rounds() == n and gpu.degree() == ref.degree
    claim = ref.claim()
    bind = None
    for rnd in range(n):
        want = ref.round_evals(None if bind is None else F.from_limbs(bind))
        assert (want[0] + want[1]) % P == claim
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = _challenge(rnd, n)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    ref.finish_rounds(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == ref.final_evals()
    fin = E.expr_value(ref.final_evals(), _ref_monomials(monomials))
    if eq:
        assert gpu.eq_scalar() == ref.eq_scalar()
        fin = fin * ref.eq_scalar() % P
    assert fin == claim
    gpu.close()


def test_expr_without_claim_computes_every_point(sess):
    """no claim: s(1) is computed on the device, nothing is checked"""
    n = 6
    tabs = [S.rand_limbs_full(0x7100 + j, 1 << n) for j in range(2)]
    mons = [(3, [0, 0, 1]), (-1, [1])]
    ref = E.ExpressionMember([F.limbs_to_ints(t) for t in tabs], mons, HIGH_TO_LOW)
    gpu = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], mons, order=HIGH_TO_LOW)
    bind = None
    for rnd in range(n):
        assert gpu.prove_round_evals(bind, rnd, None) == ref.round_evals(None if bind is None else F.from_limbs(bind))
        bind = rand_challenge(0x7200 + rnd)


# ---- full size, by linearity ------------------------------------------------------------------------------------
N_FULL = 22


def _run_pair(a, b, n, claim_a, claim_b, relate, challenge):
    """drive two members through every round; relate(evals_a, evals_b) must hold each round"""
    bind = None
    for rnd in range(n):
        ea = a.prove_round_evals(bind, rnd, claim_a)
        eb = b.prove_round_evals(bind, rnd, claim_b)
        relate(ea, eb, rnd)
        bind = challenge(rnd)
        r = F.from_limbs(bind)
        claim_a = UnivariatePoly.from_evals(ea).evaluate(r)
        claim_b = UnivariatePoly.from_evals(eb).evaluate(r)
    a.finish_rounds(bind)
    b.finish_rounds(bind)
    return claim_a, claim_b


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_scaled_product_2pow22_is_c_times_product(sess, order):
    c = GAMMA
    tabs = [rand_limbs(0xF100 + j, 1 << N_FULL) for j in range(2)]
    pa = [Polynomial.new(sess, t) for t in tabs]
    pb = [p.clone() for p in pa]
    a = ExpressionMember(sess, pa, [(c, [0, 1])], order=order)
    b = ProductMember(sess, pb, order)

    def rel(ea, eb, rnd):
        assert ea == [c * v % P for v in eb], f"round {rnd}"
    # round 0 without a claim (every point computed), then the hint
    _run_pair(a, b, N_FULL, None, None, rel, lambda r: rand_challenge(0xF200 + r) if r % 2 else rand_limbs(0xF300 + r, 1)[0])
    assert a.final_evals() == b.final_evals()


def test_square_2pow22_equals_product_with_clone(sess):
    order = LOW_TO_HIGH
    t0 = rand_limbs(0xF400, 1 << N_FULL)
    p0 = Polynomial.new(sess, t0)
    a = ExpressionMember(sess, [p0.clone()], [(1, [0, 0])], order=order)
    b = ProductMember(sess, [p0, p0.clone()], order)

    def rel(ea, eb, rnd):
        assert ea == eb, f"round {rnd}"
    _run_pair(a, b, N_FULL, None, None, rel, lambda r: rand_challenge(0xF500 + r))
    assert a.final_evals() * 2 == b.final_evals()


def test_eq_scaled_triple_2pow22_is_3_times_eq_member(sess):
    order = HIGH_TO_LOW
    tabs = [rand_limbs(0xF600 + j, 1 << N_FULL) for j in range(3)]
    w = np.stack([rand_challenge(0xF700 + i) for i in range(N_FULL)])
    a = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], [(3, [0, 1, 2])], w, order=order)
    b = EqProductMember(sess, [Polynomial.new(sess, t) for t in tabs], w, order=order)
    # the input claim: s(0) + s(1) of the plain product member over the materialised eq table
    eqp = EqPolynomial.evals(sess, w)
    ref4 = ProductMember(sess, [eqp] + [Polynomial.new(sess, t) for t in tabs], order)
    ev = ref4.prove_round_evals(None, 0, None)
    ref4.close()
    claim_b = (ev[0] + ev[1]) % P

    def rel(ea, eb, rnd):
        assert ea == [3 * v % P for v in eb], f"round {rnd}"
    fa, fb = _run_pair(a, b, N_FULL, 3 * claim_b % P, claim_b, rel, lambda r: rand_challenge(0xF800 + r))
    assert a.final_evals() == b.final_evals() and a.eq_scalar() == b.eq_scalar()
    assert fa == 3 * fb % P


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_booleanity_2pow22_closes(sess, order):
    """eq * (f^2 - f) over a 0/1 table sums to 0; the final claim is eq(w, r) * (f(r)^2 - f(r))"""
    rng = np.random.Generator(np.random.PCG64(0xB00))
    bits = rng.integers(0, 2, size=1 << N_FULL, dtype=np.uint8)
    w = np.stack([rand_challenge(0xB100 + i) for i in range(N_FULL)])
    gpu = ExpressionMember(sess, [Polynomial.from_small(sess, bits)], [(1, [0, 0]), (-1, [0])], w, order=order)
    assert gpu.degree() == 3
    claim = 0
    bind = None
    for rnd in range(N_FULL):
        ev = gpu.prove_round_evals(bind, rnd, claim)
        assert (ev[0] + ev[1]) % P == claim
        bind = rand_challenge(0xB200 + rnd)
        claim = UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    f = gpu.final_evals()[0]
    assert gpu.eq_scalar() * (f * f - f) % P == claim
    assert claim != 0


# ---- the batch engine and the scheduler -------------------------------------------------------------------------
def _mixed_batch(sess, count, seed):
    """count members of ragged sizes: expression (with and without eq), product, sum-of-products and eq members;
    returns (device members, oracle members, descs)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    dev, ref, desc = [], [], []
    for i in range(count):
        n = int(rng.integers(3, 8))
        kind = i % 5
        if kind == 0:
            T, mons, eq = 3, [(1, [0, 1]), (-1, [2]), (GAMMA, [0, 0, 2])], True
        elif kind == 1:
            T, mons, eq = 2, [(5, [0, 0, 1]), (1, [1])], False
        elif kind == 2:
            T, mons, eq = 2, [(1, [0, 1])], False          # a product member
        elif kind == 3:
            T, mons, eq = 4, [(1, [0, 1]), (1, [2, 3])], False   # a sum-of-products member
        else:
            T, mons, eq = 2, [(1, [0, 1])], True           # an eq member
        tabs = [O.random_fr(seed * 100 + 10 * i + j, 1 << n) for j in range(T)]
        w = O.random_fr(seed * 100 + 10 * i + 9, n) if eq else None
        r = E.ExpressionMember(tabs, mons, LOW_TO_HIGH, w)
        polys = [Polynomial.from_ints(sess, t) for t in tabs]
        wl = None if w is None else np.stack([F.to_limbs(v) for v in w])
        if kind == 2:
            d = ProductMember(sess, polys, LOW_TO_HIGH)
        elif kind == 3:
            d = SumOfProductsMember(sess, polys, 2, 2, LOW_TO_HIGH)
        elif kind == 4:
            d = EqProductMember(sess, polys, wl, order=LOW_TO_HIGH)
        else:
            d = ExpressionMember(sess, polys, mons, wl, order=LOW_TO_HIGH)
        dev.append(d)
        ref.append(r)
        desc.append((r.claim(), (i * 7 + 3) % P, n))
    return dev, ref, desc


def _challenge_fn(rnd, coeffs):
    return (sum(int(c) for c in coeffs) * 7 + 31 * rnd + 5) % P


@pytest.mark.parametrize("count", [5, 17])
def test_prove_batch_mixed_matches_oracle_engine(sess, count):
    dev, ref, desc = _mixed_batch(sess, count, 0x60 + count)
    max_n = max(d[2] for d in desc)
    max_deg = max(r.degree for r in ref)
    claimed = sum(c * k * pow(2, max_n - n, P) for c, k, n in desc) % P
    # a member of n < max_n rounds takes the last n rounds (its claim halves over the first max_n - n)
    want = O.prove_batch([dict(input_claim=c, coefficient=k, rounds=n, offset=max_n - n) for c, k, n in desc], ref, max_n,
                         max_deg, claimed, _challenge_fn)
    got = jolt_b200.prove_batch_native([BatchMember(c, k, n, max_n - n) for c, k, n in desc], dev, max_n, max_deg, claimed,
                                       absorb_round=lambda r, poly: _challenge_fn(r, poly.coefficients))
    assert got.challenges == want["challenges"]
    assert got.final_claim == want["final_claim"]
    assert got.member_claims == want["member_claims"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for d, r in zip(dev, ref):
        assert d.final_evals() == r.final_evals()


def test_scheduler_mixed_17_members_matches_oracle(sess):
    dev, ref, desc = _mixed_batch(sess, 17, 0x90)
    sched = RoundScheduler(sess, dev)
    n_max = max(d[2] for d in desc)
    claims = [d[0] for d in desc]
    binds = [None] * len(dev)
    for rnd in range(n_max):
        work = [(i, rnd, binds[i], claims[i]) for i in range(len(dev)) if rnd < desc[i][2]]
        polys = sched.batch_prove_round(work)
        c = (rnd * 1234567 + 89) % P
        for (i, *_), poly in zip(work, polys):
            want = ref[i].prove_round(binds[i], rnd, claims[i])
            assert poly.coefficients == want + [0] * (len(poly.coefficients) - len(want)), (i, rnd)
            claims[i] = poly.evaluate(c)
            binds[i] = c
    sched.batch_finish_rounds([(i, binds[i]) for i in range(len(dev))])
    for i, (d, r) in enumerate(zip(dev, ref)):
        r.finish_rounds(binds[i])
        assert d.final_evals() == r.final_evals()
    sched.close()


# ---- routing ------------------------------------------------------------------------------------------------------
def test_built_shape_gets_the_resident_member(sess):
    """an expression that is exactly a product is the product member: the whole sumcheck is one launch"""
    n = 12
    tabs = [rand_limbs(0xA100 + j, 1 << n) for j in range(2)]
    ref = E.ExpressionMember([F.limbs_to_ints(t) for t in tabs], [(1, [0, 1])], LOW_TO_HIGH)
    gpu = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], [(1, [0, 1])], order=LOW_TO_HIGH)
    claim = ref.claim()
    l0 = sess.launch_count
    bind = None
    for rnd in range(n):
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == ref.round_evals(None if bind is None else F.from_limbs(bind))
        bind = rand_challenge(0xA200 + rnd)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    assert sess.launch_count - l0 == 1
    ref.finish_rounds(F.from_limbs(bind))
    assert gpu.final_evals() == ref.final_evals()


def test_expression_never_joins_a_resident_run(sess):
    """f0 * f0 has the (m, terms) of a degree-2 product; in a batch with a product member it still runs its own pass
    every round (a resident run would prove it as f0 * <its missing second table>)"""
    n = 10
    t0, t1, t2 = (rand_limbs(0xA300 + j, 1 << n) for j in range(3))
    r_expr = E.ExpressionMember([F.limbs_to_ints(t0)], [(1, [0, 0])], LOW_TO_HIGH)
    r_prod = E.ExpressionMember([F.limbs_to_ints(t1), F.limbs_to_ints(t2)], [(1, [0, 1])], LOW_TO_HIGH)
    d_expr = ExpressionMember(sess, [Polynomial.new(sess, t0)], [(1, [0, 0])], order=LOW_TO_HIGH)
    d_prod = ProductMember(sess, [Polynomial.new(sess, t1), Polynomial.new(sess, t2)], LOW_TO_HIGH)
    sched = RoundScheduler(sess, [d_expr, d_prod])
    claims = [r_expr.claim(), r_prod.claim()]
    l0 = sess.launch_count
    bind = None
    for rnd in range(n):
        polys = sched.batch_prove_round([(0, rnd, bind, claims[0]), (1, rnd, bind, claims[1])])
        assert polys[0].coefficients == r_expr.prove_round(bind, rnd, claims[0])
        assert polys[1].coefficients == r_prod.prove_round(bind, rnd, claims[1])
        bind = (rnd * 99991 + 7) % P
        claims = [p.evaluate(bind) for p in polys]
    assert sess.launch_count - l0 >= n    # the expression member launched its pass every round
    sched.batch_finish_rounds([(0, bind), (1, bind)])
    r_expr.finish_rounds(bind)
    r_prod.finish_rounds(bind)
    assert d_expr.final_evals() == r_expr.final_evals() and d_prod.final_evals() == r_prod.final_evals()
    sched.close()


# ---- errors -------------------------------------------------------------------------------------------------------
def _create(sess, T, monomials, n=4, w=None, scale=None, order=LOW_TO_HIGH, polys=None, nvars=None):
    polys = polys if polys is not None else [Polynomial.new(sess, rand_limbs(0xEE0 + j, 1 << n)) for j in range(T)]
    handles = np.array([p.handle for p in polys], dtype=np.uint64)
    mons = (_lib.MonomialC * max(len(monomials), 1))()
    for k, (coeff, tabs, *deg) in enumerate(monomials):
        mons[k].coeff[:] = [int(x) for x in (F.to_limbs(coeff) if isinstance(coeff, int) else coeff)]
        mons[k].degree = deg[0] if deg else len(tabs)
        for i, t in enumerate(tabs[:6]):
            mons[k].table[i] = t
    h = ctypes.c_void_p()
    wp = None if w is None else np.ascontiguousarray(w, dtype=np.uint64).reshape(-1, 4)
    st = sess.lib.jb_member_create_expr(sess.h, handles.ctypes.data_as(_lib.c_u64p), len(handles),
                                        ctypes.cast(mons, ctypes.c_void_p), len(monomials),
                                        None if wp is None else wp.ctypes.data_as(_lib.c_u64p),
                                        nvars if nvars is not None else (0 if wp is None else wp.shape[0]),
                                        None if scale is None else scale.ctypes.data_as(_lib.c_u64p), order, ctypes.byref(h))
    if st == _lib.JB_OK:
        sess.lib.jb_member_destroy(h)
    return st


def test_errors_and_context_stays_usable(sess):
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    bad = S.int_to_limbs(P)   # not canonical
    w4 = np.stack([F.to_limbs(v) for v in O.random_fr(5, 4)])
    assert _create(sess, 1, [(1, [0], 0)]) == INV                              # a zero-degree monomial
    assert _create(sess, 2, [(1, [0, 2])]) == INV                              # a table index >= ntables
    assert _create(sess, 3, [(1, [0, 1])]) == INV                              # a table no monomial uses
    p = Polynomial.new(sess, rand_limbs(1, 16))
    assert _create(sess, 2, [(1, [0, 1])], polys=[p, p]) == INV                # duplicate handles
    assert _create(sess, 2, [(1, [0, 1])], polys=[Polynomial.new(sess, rand_limbs(2, 16)),
                                                  Polynomial.new(sess, rand_limbs(3, 32))]) == INV   # lengths differ
    assert _create(sess, 1, [(bad, [0, 0])]) == INV                            # a non-canonical coefficient
    w_bad = w4.copy()
    w_bad[2] = bad
    assert _create(sess, 1, [(2, [0, 0])], w=w_bad) == INV                     # a non-canonical point
    assert _create(sess, 1, [(2, [0, 0])], w=w4, scale=bad) == INV             # a non-canonical scale
    assert _create(sess, 1, [(2, [0, 0])], w=w4[:3]) == INV                    # nvars != log2(length)
    assert _create(sess, 1, [(2, [0, 0])], order=7) == INV                     # an unknown order
    assert _create(sess, 1, [(1, [0] * 6, 7)]) == UNS                          # degree above JB_EXPR_MAX_DEGREE
    assert _create(sess, 9, [(1, list(range(6))), (1, [6, 7, 8])]) == UNS     # more than JB_EXPR_MAX_TABLES tables
    assert _create(sess, 1, [(k + 1, [0]) for k in range(17)]) == UNS          # more than JB_EXPR_MAX_MONOMIALS
    assert _create(sess, 1, [(2, [0, 0])]) == _lib.JB_OK
    # the context still proves
    test_expr_without_claim_computes_every_point(sess)
    # a zero eq factor at the current variable is refused, as for the split-eq member
    w0 = w4.copy()
    w0[3] = 0
    gpu = ExpressionMember(sess, [Polynomial.new(sess, rand_limbs(9, 16))], [(1, [0, 0]), (-1, [0])], w0, order=LOW_TO_HIGH)
    with pytest.raises(jolt_b200.JoltB200Error, match="must be invertible"):
        gpu.prove_round_evals(None, 0, 1)
    with pytest.raises(jolt_b200.JoltB200Error, match="claim is required"):
        gpu.prove_round_evals(None, 0, None)
    gpu.close()
