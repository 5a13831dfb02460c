"""Read-write checking member at the sizes it exists for, bit-exact:
  - against the dense device expression member over the materialised tables (ra_a, Val, inc and a replicated eq table,
    degree-3 monomials c_a E ra_a Val and c_a E ra_a inc) at K T = 2^20 .. 2^24, register- and RAM-shaped, with
    compact u64 value columns from host memory and from device tensors;
  - at T = 2^22 for registers (K = 128, A = 3) and RAM (K = 2^16, u16): the claimed sum from the columns, every round's
    s(0) + s(1) check, and the final values against independent evaluations - ra_a by one_hot_evaluate, inc by
    evaluate_small, Val(r) = init~(r_addr) + sum_j inc(j) eq(r_addr, addr_w(j)) LT(j, r_cycle) with the LT table;
  - in jb_prove_batch next to a member of fewer variables."""
import numpy as np
import pytest
import torch

import jolt_b200
from jolt_b200 import (LOW_TO_HIGH, BatchMember, ExpressionMember, LtPolynomial, Polynomial, ProductMember,
                       ReadWriteCheckingMember, Source, evaluate_small, one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
import rw_ref as R

P = O.R_MOD
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def rw_member(sess, wl, w, device=False):
    def col(x):
        return torch.from_numpy(x.view(np.int16) if x.dtype == np.uint16 else x).cuda() if device else x
    addr_cols = {id(a): col(a) for a in wl["addrs"]}
    acc = [(addr_cols[id(a)], Source.compact(col(v.view(np.int64)) if device else v, "u64"), c, d)
           for a, v, c, d in zip(wl["addrs"], wl["values"], wl["coeffs"], wl["ds"])]
    return ReadWriteCheckingMember(sess, acc, wl["write"], Source.compact(wl["inc"], "u64"),
                                   Source.compact(wl["init"], "u64"), wl["K"], w)


def claimed_sum(sess, wl, w):
    """sum_j eq(w, j) sum_a c_a (v_a(j) + d_a inc(j)): the columns' evaluations at w (v_a and inc vanish where no access)."""
    ev = evaluate_small(sess, wl["values"] + [wl["inc"]], w, "u64")
    return sum(c * (v + d * ev[-1]) for c, v, d in zip(wl["coeffs"], ev, wl["ds"])) % P


@pytest.mark.parametrize("K,T,shape,device", [(128, 1 << 13, "registers", False), (128, 1 << 15, "registers", True),
                                              (128, 1 << 17, "registers", False), (1 << 16, 1 << 4, "ram", True),
                                              (1 << 16, 1 << 6, "ram", False), (1 << 16, 1 << 8, "ram", False)])
def test_matches_dense_expression_member(sess, K, T, shape, device):
    wl = R.columns_workload(K + T, K, T, shape)
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    w = O.random_fr(K * 3 + T, t)
    ch = O.random_fr(K * 5 + T, t + kappa)
    rw = rw_member(sess, wl, w, device)
    dense = R.dense_member(sess, wl, w)
    claim = claimed_sum(sess, wl, w)
    bind = None
    for rnd in range(t + kappa):
        got = rw.prove_round_evals(bind, rnd, claim)
        assert got == dense.prove_round_evals(bind, rnd, claim), rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    rw.finish_rounds(bind)
    dense.finish_rounds(bind)
    want = dense.final_evals()
    assert rw.final_evals() == want[:-1]
    assert rw.eq_scalar() == want[-1]
    rw.close()
    dense.close()


def val_at(sess, wl, r_addr, r_cycle):
    """init~(r_addr) + sum_j inc(j) eq(r_addr, addr_w(j)) LT(j, r_cycle), the sum taken as s(0) + s(1) of the first
    round of the value-evaluation expression member over the write's one-hot column, inc and the LT table."""
    K = wl["K"]
    lt = LtPolynomial.evals(sess, F.ints_to_limbs(r_cycle))
    m = ExpressionMember.from_sources(
        sess, [Source.one_hot(wl["addrs"][wl["write"]], K, r_addr), Source.compact(wl["inc"], "u64"), Source.table(lt)],
        [(1, [0, 1, 2])], order=LOW_TO_HIGH)
    s = m.prove_round_evals(None, 0, None)
    m.close()
    init_r = evaluate_small(sess, [wl["init"]], r_addr, "u64")[0]
    return (init_r + s[0] + s[1]) % P


@pytest.mark.parametrize("K,shape", [(128, "registers"), (1 << 16, "ram")])
def test_t_2_22_against_independent_evaluations(sess, K, shape):
    T = 1 << 22
    wl = R.columns_workload(7 + K, K, T, shape)
    t, kappa = 22, K.bit_length() - 1
    w = O.random_fr(8 + K, t)
    ch = O.random_fr(9 + K, t + kappa)
    m = rw_member(sess, wl, w)
    claim = claimed_sum(sess, wl, w)
    bind = None
    for rnd in range(t + kappa):
        got = m.prove_round_evals(bind, rnd, claim)
        assert (got[0] + got[1]) % P == claim, rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    fin = m.final_evals()
    e = m.eq_scalar()
    A = len(wl["addrs"])
    assert claim == e * sum(c * fin[a] * (fin[A] + d * fin[A + 1])
                            for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"]))) % P
    r_cycle, r_addr = ch[:t][::-1], ch[t:][::-1]
    for a in range(A):
        assert fin[a] == one_hot_evaluate(sess, wl["addrs"][a], K, r_addr + r_cycle, layout="address_major")[0], a
    assert fin[A + 1] == evaluate_small(sess, [wl["inc"]], r_cycle, "u64")[0]
    assert fin[A] == val_at(sess, wl, r_addr, r_cycle)
    m.close()


def test_prove_batch_with_a_member_of_fewer_variables(sess):
    wl = R.workload(61, 8, 64, 3, "registers")
    K, T, accesses, write, inc, init = wl
    w = O.random_fr(62, 6)
    cols = {}
    acc = []
    for ad, values, c, d in accesses:
        cols.setdefault(id(ad), np.array([0xFF if x is None else x for x in ad], dtype=np.uint8))
        acc.append((cols[id(ad)], Source.table(Polynomial.from_ints(sess, values)), c, d))
    rw = ReadWriteCheckingMember(sess, acc, write, Source.table(Polynomial.from_ints(sess, inc)),
                                 Source.compact(np.array(init, dtype=np.uint64)), K, w)
    tabs = [O.random_fr(63 + j, 16) for j in range(2)]
    pm = ProductMember(sess, [Polynomial.from_ints(sess, x) for x in tabs], LOW_TO_HIGH)
    c_rw = R.claimed_sum(T, accesses, inc, w)
    c_pm = sum(a * b for a, b in zip(*tabs)) % P
    k_rw, k_pm = 3, 5
    n = 9
    claimed = (k_rw * c_rw + k_pm * c_pm * pow(2, n - 4, P)) % P
    got = jolt_b200.prove_batch_native([BatchMember(c_rw, k_rw, n, 0), BatchMember(c_pm, k_pm, 4, n - 4)], [rw, pm], n, 3,
                                       claimed, absorb_round=lambda r, poly: (sum(poly.coefficients) * 7 + r + 3) % P)
    # the read-write member ran every round at the batch's challenges: its rounds and values are the reference's
    want_rounds, want_final = R.sparse_prove(*wl, w, None, got.challenges)
    assert rw.final_evals() == want_final
    fin = want_final
    e = rw.eq_scalar()
    member = e * sum(c * fin[a] * (fin[-2] + d * fin[-1]) for a, (_x, _v, c, d) in enumerate(accesses)) % P
    assert got.member_claims[0] == member
    pf = pm.final_evals()
    assert got.member_claims[1] == pf[0] * pf[1] % P
    assert got.final_claim == (k_rw * member + k_pm * got.member_claims[1]) % P
    for rnd, poly in enumerate(got.round_polynomials[:n - 4]):  # the product member halves its claim meanwhile
        half = c_pm * pow(2, n - 4 - rnd - 1, P) % P
        assert [poly.evaluate(x) for x in range(4)] == [(k_rw * s + k_pm * half) % P for s in want_rounds[rnd]]
    rw.close()
    pm.close()
