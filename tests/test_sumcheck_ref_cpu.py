"""CPU pins of the sumcheck edge-test references (tests/sumcheck_ref.py): the C oracle on limb-extreme tables and
challenges against Python big ints, the sign-tensor closed form against brute force, and the input generators."""
import math

import numpy as np
import pytest

from oracle import bn254 as O
from oracle import coracle as C
import sumcheck_ref as S

P = O.R_MOD


def test_rand_limbs_full_covers_the_whole_field():
    a = S.rand_limbs_full(7, 1 << 14)
    raw = S.raw_ints(a)
    assert max(raw) < P
    top = sum(v >= 1 << 253 for v in raw) / len(raw)
    assert 0.3 < top < 0.4                      # (p - 2^253) / p ~ 0.34 of a uniform draw
    assert (S.rand_limbs_full(7, 1 << 14) == a).all()
    assert S.below_p(np.stack([S.int_to_limbs(v) for v in (0, P - 1, P, P + 1, (1 << 256) - 1)])).tolist() == \
        [True, True, False, False, False]


def test_extreme_values_and_challenges():
    assert len(set(S.EXTREME_RAW)) == len(S.EXTREME_RAW) and max(S.EXTREME_RAW) < P
    w = S.EXTREME_RAW[9]
    assert [(w >> (32 * k)) & 0xFFFFFFFF for k in range(7)] == [0xFFFFFFFF] * 7 and w < P and w + (1 << 224) > P
    assert C.mont_to_ints(S.int_to_limbs(S.R_MONT))[0] == 1
    for ch in S.EXTREME_CHALLENGES:
        assert O.mont_raw(ch) < P
    assert C.mont_to_ints(S.EXTREME_CHALLENGES[0])[0] == 0 and C.mont_to_ints(S.EXTREME_CHALLENGES[3])[0] == 1
    assert all(O.mont_raw(S.extreme_challenge(r, 3)) < P for r in range(14))


@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
def test_extreme_table_places_every_ordered_pair(order):
    n = 11
    t = S.extreme_table(5, n, order, rotate=3)
    half = 1 << (n - 1)
    got = set()
    for y in range(half):
        lo, hi = (t[2 * y], t[2 * y + 1]) if order == O.LOW_TO_HIGH else (t[y], t[y + half])
        got.add((O.mont_raw(lo), O.mont_raw(hi)))
    assert {(a, b) for a in S.EXTREME_RAW for b in S.EXTREME_RAW} <= got
    assert max(S.raw_ints(t)) < P


@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
def test_c_oracle_on_extreme_limbs_vs_big_ints(order):
    """bind, product_round_evals and eq_evals of the C oracle on limb-extreme tables and challenges, against the
    Python big-int restatement: the C oracle is the reference of the device edge tests."""
    n = 9
    tabs = [S.extreme_table(40 + j, n, order, rotate=j) for j in range(4)]
    ints = [C.mont_to_ints(t) for t in tabs]
    for m in (1, 2, 3, 4):
        assert C.mont_to_ints(C.product_round_evals(tabs[:m], m, order)) == O.product_round_evals(ints[:m], m, order)
    cur, cur_i = tabs, ints
    for rnd in range(n - 1):
        ch = S.extreme_challenge(rnd, 2)
        c_int = C.mont_to_ints(ch)[0]
        cur = [C.bind(t, ch, order) for t in cur]
        cur_i = [O.bind(t, c_int, order) for t in cur_i]
        assert [C.mont_to_ints(t) for t in cur] == cur_i, f"bind round {rnd}"
        assert C.mont_to_ints(C.product_round_evals(cur, 4, order)) == O.product_round_evals(cur_i, 4, order)
    # eq tables over extreme coordinates, as full elements and as 125-bit challenges
    pts = np.concatenate([S.extreme_limbs, S.EXTREME_CHALLENGES])
    assert C.mont_to_ints(C.eq_evals(pts)) == O.eq_evals(C.mont_to_ints(pts))
    scale = S.int_to_limbs(P - 1)
    assert C.mont_to_ints(C.eq_evals(pts[::-1].copy(), scale)) == O.eq_evals(C.mont_to_ints(pts[::-1]),
                                                                              C.mont_to_ints(scale)[0])


def test_sop_round_evals_is_the_sum_of_term_products():
    n = 8
    tabs = [S.rand_limbs_full(60 + j, 1 << n) for j in range(4)]
    ints = [C.mont_to_ints(t) for t in tabs]
    for order in (O.HIGH_TO_LOW, O.LOW_TO_HIGH):
        want = [(a + b) % P for a, b in zip(O.product_round_evals(ints[:2], 2, order),
                                             O.product_round_evals(ints[2:], 2, order))]
        assert S.sop_round_evals(tabs, 2, order) == want


def test_sign_table_entries():
    pat = S.sign_patterns(3, 5, 2)[0][0]
    t = S.sign_table(pat)
    vals = C.mont_to_ints(t)
    assert set(S.raw_ints(t)) <= {1, P - 1}
    for x in range(1 << 5):
        sign = math.prod(pat[i][(x >> (4 - i)) & 1] for i in range(5))
        assert vals[x] == S.C_SIGN * sign % P


@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
@pytest.mark.parametrize("shape", [(1, 1), (2, 1), (3, 1), (4, 1), (2, 2)])
@pytest.mark.parametrize("n", [1, 6, 10])
def test_sign_closed_form_vs_brute_force(order, shape, n):
    """closed-form round evaluations, final evaluations and final claim against O.ProductMember driven round by
    round over the materialised tables (a sum of products as the sum over its terms)."""
    D, T = shape
    terms = S.sign_patterns(100 * n + 10 * D, n, D, T)
    challenges = [C.mont_to_ints(S.extreme_challenge(r, n))[0] for r in range(n)]
    got = S.sign_sumcheck(terms, order, challenges)
    refs = [O.ProductMember([C.mont_to_ints(S.sign_table(pat)) for pat in tm], order) for tm in terms]
    bind = None
    for rnd in range(n):
        evals = [0] * (D + 1)
        for ref in refs:
            if bind is not None:
                ref.tables = [O.bind(t, bind, order) for t in ref.tables]
            ev = O.product_round_evals(ref.tables, D, order)
            evals = [(a + b) % P for a, b in zip(evals, ev)]
        assert got["rounds"][rnd] == evals, f"round {rnd}"
        assert any(got["rounds"][rnd]), "a vanishing round polynomial tests nothing"
        bind = challenges[rnd]
    for ref in refs:
        ref.finish_rounds(bind)
    finals = [f for ref in refs for f in ref.final_evals()]
    assert got["finals"] == finals
    assert got["final_claim"] == sum(math.prod(finals[k * D:(k + 1) * D]) for k in range(T)) % P


def test_constant_table_closed_form():
    """all-plus patterns: the constant table with limbs p - 1, s_k(t) = 2^(n-1-k) c^m"""
    n, m = 7, 3
    terms = [[[(1, 1)] * n for _ in range(m)]]
    assert set(S.raw_ints(S.sign_table(terms[0][0]))) == {P - 1}
    got = S.sign_sumcheck(terms, O.LOW_TO_HIGH, [5] * n)
    for k in range(n):
        assert got["rounds"][k] == [pow(2, n - 1 - k, P) * pow(S.C_SIGN, m, P) % P] * (m + 1)
    assert got["finals"] == [S.C_SIGN] * m
