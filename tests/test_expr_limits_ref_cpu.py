"""CPU checks for the references that tests/test_gpu_expr_limits.py runs the device against, at the expression limits
(8 tables or sources, 16 monomials, degree 6, degree 7 with eq): tests/expr_ref.py and tests/source_ref.py against brute
force over the hypercube (each round polynomial from the multilinear extensions at (bound challenges, t, free
variables); one-hot and compact entries from their definitions) for every limit shape and source case, without eq, with
eq and with eq and a scale, in both orders."""
import math

import numpy as np
import pytest

from jolt_b200 import field as F
from oracle import bn254 as O
import expr_ref as E
import mle_eval_ref as M
import source_ref as SR
import sumcheck_ref as S
from test_expr_ref_cpu import _eq, brute_round
from test_gpu_expr_limits import SCALE, SHAPES, SOURCE_CASES, ref_monomials, source_inputs, source_monomials

P = O.R_MOD
EQ_VARIANTS = {"plain": (False, None), "eq": (True, None), "eq_scaled": (True, SCALE)}


def check_against_brute_force(ref, tables, monomials, order, n, w, scale):
    """every round of `ref` (an ExpressionMember over `tables`), its final evaluations and eq scalar, by brute force"""
    deg = E.expr_degree(monomials, w is not None)
    assert ref.degree == deg
    bound, bind = [], None
    for rnd in range(n):
        ev = ref.round_evals(bind)
        want = [brute_round(tables, monomials, order, bound, t, w, 1 if scale is None else scale) for t in range(deg + 1)]
        assert ev == want, f"round {rnd}"
        bind = O.random_fr(0x910 + rnd, 1)[0] if rnd % 2 else F.from_limbs(S.extreme_challenge(rnd + 1))
        bound.append(bind)
    ref.finish_rounds(bind)
    pt = bound if order == O.HIGH_TO_LOW else list(reversed(bound))
    fin = ref.final_evals()
    assert fin == [O.evaluate(t, pt) for t in tables]
    if w is not None:
        assert ref.eq_scalar() == (1 if scale is None else scale) * _eq(w, pt) % P
    return pt, fin


@pytest.mark.parametrize("variant", sorted(EQ_VARIANTS))
@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_expr_reference_at_limits_matches_brute_force(shape, order, variant):
    T, mons, _, _ = SHAPES[shape]
    eq, scale = EQ_VARIANTS[variant]
    n = 4 if shape == "max" else 3
    tables = [F.limbs_to_ints(S.rand_limbs_full(0x61 + j, 1 << n)) for j in range(T)]
    tables[0][:len(S.EXTREME_RAW)] = [F.from_limbs(S.extreme_limbs[i]) for i in range(min(1 << n, len(S.EXTREME_RAW)))]
    w = O.random_fr(0xE5 + n, n) if eq else None
    rm = ref_monomials(mons)
    ref = E.ExpressionMember(tables, rm, order, w, scale)
    assert E.expr_round_evals(tables, rm, order, w, scale) == ref.round_evals(None)
    check_against_brute_force(E.ExpressionMember(tables, rm, order, w, scale), tables, rm, order, n, w, scale)


def test_limit_shapes_are_at_the_limits():
    """the shapes the device tests run reach every declared limit and use every table"""
    T, mons, _, _ = SHAPES["max"]
    assert T == 8 and len(mons) == 16 and max(len(t) for _, t in mons) == 6
    assert {len(t) for _, t in mons} == set(range(1, 7))
    assert [3] * 6 in [t for _, t in mons] and [7, 0, 7, 1, 7, 2] in [t for _, t in mons]
    for T, mons, _, _ in SHAPES.values():
        assert sorted({t for _, tabs in mons for t in tabs}) == list(range(T))
    assert {T for T, mons, _, _ in SHAPES.values() if max(len(t) for _, t in mons) == 6} >= {5, 6, 7, 8}
    for case, (specs, *_rest) in SOURCE_CASES.items():
        assert sorted({t for _, tabs in source_monomials(len(specs)) for t in tabs}) == list(range(len(specs)))
    assert SOURCE_CASES["one_hot8_u8_K256"][0] == ["oh_u8_256"] * 8


def entry(src, j):
    """entry j of a reference source from its definition"""
    if src[0] == "table":
        return src[1][j] % P
    if src[0] == "compact":
        return M.promote(src[1][j])
    _, addr, K, r = src
    a = addr[j]
    if a is None:
        return 0
    lk = K.bit_length() - 1
    return math.prod((r[i] if (a >> (lk - 1 - i)) & 1 else 1 - r[i]) for i in range(lk)) % P


@pytest.mark.parametrize("variant", sorted(EQ_VARIANTS))
@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
@pytest.mark.parametrize("case", sorted(SOURCE_CASES))
def test_source_reference_at_limits_matches_brute_force(case, order, variant):
    specs = SOURCE_CASES[case][0]
    eq, scale = EQ_VARIANTS[variant]
    n = 3
    _, refsrc, _ = source_inputs(None, case, n)
    tables = [[entry(src, j) for j in range(1 << n)] for src in refsrc]
    assert [SR.source_table(src) for src in refsrc] == tables
    w = O.random_fr(0xE9 + n, n) if eq else None
    rm = ref_monomials(source_monomials(len(specs)))
    ref = SR.SourcesMember(refsrc, rm, order, w, scale)
    pt, fin = check_against_brute_force(ref, tables, rm, order, n, w, scale)
    for j, src in enumerate(refsrc):   # a one-hot source's final value is the one-hot polynomial at (cycle, address)
        if src[0] == "one_hot":
            assert fin[j] == M.one_hot_evaluate_direct(src[1], src[2], 1 << n, list(pt) + list(src[3]), "cycle_major")
        elif src[0] == "compact":
            assert fin[j] == M.evaluate_small(src[1], pt)
