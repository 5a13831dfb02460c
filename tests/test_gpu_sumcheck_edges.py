"""Sumcheck kernels at the edges of their arithmetic and in every pass shape, limb for limb against independent
references: the C oracle on limb-extreme tables with extreme challenges (single-block, thin / lookahead and
multi-block passes; resident and one-launch-per-round), the sum-of-products member every round up to 2^22, closed
forms of sign-tensor tables at 2^24 and 2^26, and batches of 9 to 24 members against the oracle engine."""
import os

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, Polynomial, ProductMember, RoundScheduler,
                       SumOfProductsMember, UnivariatePoly)
from oracle import bn254 as O
from oracle import coracle as C
import sumcheck_ref as S

pytestmark = pytest.mark.gpu
P = O.R_MOD


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sess_launch():
    """the resident service off: one kernel launch per round all the way down"""
    os.environ["JB_NO_TAIL"] = "1"
    try:
        s = jolt_b200.Session(0)
    finally:
        del os.environ["JB_NO_TAIL"]
    yield s
    s.close()


def make_member(sess, tabs, factors, terms, order):
    polys = [Polynomial.new(sess, t) for t in tabs]
    if terms == 1:
        return ProductMember(sess, polys, order)
    return SumOfProductsMember(sess, polys, factors, terms, order)


def lockstep_vs_c(sess, tabs, factors, terms, order, challenge, verify=False):
    """Every round's evaluations, the final evaluations and the final claim of the device member against the
    C oracle over the same tables, challenge(rnd) binding after round rnd."""
    n = tabs[0].shape[0].bit_length() - 1
    thr = C.max_threads()
    sess.set_verify_rounds(verify)
    try:
        gpu = make_member(sess, tabs, factors, terms, order)
        cur, bind, claim = tabs, None, None
        for rnd in range(n):
            if bind is not None:
                cur = [C.bind(t, bind, order, thr) for t in cur]
            want = S.sop_round_evals(cur, factors, order, thr)
            if claim is None:
                claim = (want[0] + want[1]) % P
            assert (want[0] + want[1]) % P == claim, f"round {rnd}: the oracle's own round check"
            got = gpu.prove_round_evals(bind, rnd, claim)
            assert got == want, f"round {rnd}"
            bind = challenge(rnd)
            claim = UnivariatePoly.from_evals(got).evaluate(C.mont_to_ints(bind)[0])
        cur = [C.bind(t, bind, order, thr) for t in cur]
        gpu.finish_rounds(bind)
        fe = gpu.final_evals()
        assert fe == [C.mont_to_ints(t)[0] for t in cur]
        prods = [int(np.prod(fe[k * factors:(k + 1) * factors], dtype=object)) for k in range(terms)]
        assert sum(prods) % P == claim
        gpu.close()
    finally:
        sess.set_verify_rounds(False)


SHAPES = [(1, 1), (2, 1), (3, 1), (4, 1), (2, 2)]      # (factors, terms): products m = 1..4 and IncClaimReduction's 2 x 2


@pytest.mark.parametrize("path", ["resident", "launch"])
@pytest.mark.parametrize("n", [9, 12, 14, 18])
@pytest.mark.parametrize("mode", ["hint", "verify"])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_extreme_limbs_lockstep_vs_c_oracle(sess, sess_launch, shape, order, mode, n, path):
    """Every ordered pair of limb-extreme values (0, 1, 2, p-1, p-2, p-2^32, 2^253-1, 2^253, 2^64-1, the all-ones
    word pattern below p, Montgomery one, R^2 mod p) as a first-round (lo, hi) pair of every table, the rest drawn
    over all of [0, p); challenges cycle through 0, the largest 125-bit one, [0,0,1,0], one, p-1 and random 125-bit
    and 254-bit ones. n = 9 is a single-block pass, 12 and 14 thin / lookahead rounds, 18 multi-block passes."""
    D, T = shape
    tabs = [S.extreme_table(0x5EED + 100 * n + 10 * D + j, n, order, rotate=j) for j in range(D * T)]
    s = sess if path == "resident" else sess_launch
    lockstep_vs_c(s, tabs, D, T, order, lambda rnd: S.extreme_challenge(rnd, n), verify=(mode == "verify"))


def mixed_challenge(rnd):
    return C.rand_challenge(5000 + rnd) if rnd % 3 else S.rand_limbs_full(5000 + rnd, 1)[0]


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_sum_of_products_2pow16_every_round_vs_c_oracle(sess, order):
    n = 16
    tabs = [S.rand_limbs_full(0x50B + j, 1 << n) for j in range(4)]
    lockstep_vs_c(sess, tabs, 2, 2, order, mixed_challenge)


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_sum_of_products_2pow22_every_round_vs_c_oracle(sess, order):
    """all 22 rounds of the 2 x 2 sum of products at 2^22 against the threaded C oracle (its rounds halve, so the
    run costs about two first rounds)"""
    n = 22
    tabs = [S.rand_limbs_full(0x522 + j, 1 << n) for j in range(4)]
    lockstep_vs_c(sess, tabs, 2, 2, order, mixed_challenge)


# ---- full size through closed forms ---------------------------------------------------------------------
def sign_tensor_run(s, tables, factors, terms, order, challenges, want):
    """one member through the native batch engine (prove_batch_native) with the given challenges; the proof must
    be the closed form's"""
    n = len(challenges)
    mem = make_member(s, tables, factors, terms, order)
    claim = (want["rounds"][0][0] + want["rounds"][0][1]) % P
    res = jolt_b200.prove_batch_native([BatchMember(claim, 1, n, 0)], [mem], n, factors, claim,
                                       lambda rnd, poly: challenges[rnd])
    assert res.challenges == challenges
    for rnd in range(n):
        assert res.round_polynomials[rnd].coefficients == S.trimmed_coeffs(want["rounds"][rnd]), f"round {rnd}"
    assert mem.final_evals() == want["finals"]
    assert res.final_claim == want["final_claim"]
    mem.close()


@pytest.mark.parametrize("factors,terms,n,order", [
    (2, 1, 24, HIGH_TO_LOW), (2, 1, 24, LOW_TO_HIGH), (3, 1, 24, HIGH_TO_LOW), (4, 1, 24, LOW_TO_HIGH),
    (2, 2, 24, LOW_TO_HIGH), (2, 1, 26, LOW_TO_HIGH),
], ids=["m2-24-H2L", "m2-24-L2H", "m3-24-H2L", "m4-24-L2H", "sop2x2-24-L2H", "m2-26-L2H"])
def test_sign_tensor_full_size_closed_form(sess, sess_launch, factors, terms, n, order):
    """f_j(x) = c * prod_i g_{j,i}(x_i), entries +-c with limbs p - 1 and 1 (adjacent pairs reach the 2p - 2 and
    2 lazy differences), through the resident kernel and through one launch per round. At 2^26 (BASELINE config
    4's global size on one device) the two factors are one host table uploaded twice."""
    pats = S.sign_patterns(0x516 + n + 10 * factors + 100 * terms, n, factors, terms)
    if n == 26:
        pats = [[pats[0][0], pats[0][0]]]     # f * f: one 2 GiB host table
    host = {}
    for tm in pats:
        for p in tm:
            if tuple(p) not in host:
                host[tuple(p)] = S.sign_table(p)
    tables = [host[tuple(p)] for tm in pats for p in tm]
    challenges = [C.mont_to_ints(S.extreme_challenge(r, n))[0] for r in range(n)]
    want = S.sign_sumcheck(pats, order, challenges)
    for s in (sess, sess_launch):
        sign_tensor_run(s, tables, factors, terms, order, challenges, want)


def test_constant_table_2pow24_closed_form(sess, sess_launch):
    """the degenerate sign tensor: every entry has limbs p - 1, s_k(t) = 2^(n-1-k) c^2"""
    n = 24
    pats = [[[(1, 1)] * n] * 2]
    t = S.sign_table(pats[0][0])
    challenges = [C.mont_to_ints(S.extreme_challenge(r, 7))[0] for r in range(n)]
    want = S.sign_sumcheck(pats, HIGH_TO_LOW, challenges)
    c2 = S.C_SIGN * S.C_SIGN % P
    assert want["rounds"] == [[pow(2, n - 1 - k, P) * c2 % P] * 3 for k in range(n)]
    for s in (sess, sess_launch):
        sign_tensor_run(s, [t, t], 2, 1, HIGH_TO_LOW, challenges, want)


# ---- batches of many members ----------------------------------------------------------------------------
def batch_shapes(form, count):
    """[(m, log_len, offset)] for `count` members; a shorter member's window is front-padded (offset + log_len is
    the batch's round count, prover.rs:246-343)"""
    if form == "homogeneous":
        return [(2, 8, 0)] * count
    if form == "ragged":
        return [(2, 3 + (5 * i) % 7, 6 - (5 * i) % 7) for i in range(count)]
    return [(1 + i % 3, 6 + i % 3, 2 - i % 3) for i in range(count)]


def batch_fixture(shapes, seed):
    tabs = [[O.random_fr(seed + 10 * i + j, 1 << ln) for j in range(m)] for i, (m, ln, off) in enumerate(shapes)]
    max_vars = max(ln + off for _, ln, off in shapes)
    desc, total = [], 0
    for i, (m, ln, off) in enumerate(shapes):
        claim = sum(int(np.prod([t[x] for t in tabs[i]], dtype=object)) for x in range(1 << ln)) % P
        coeff = O.random_fr(seed + 1000 + i, 1)[0]
        desc.append(dict(input_claim=claim, coefficient=coeff, rounds=ln, offset=off))
        total = (total + coeff * claim * pow(2, max_vars - ln, P)) % P
    return tabs, desc, total, max_vars


@pytest.mark.parametrize("form", ["homogeneous", "ragged", "heterogeneous"])
@pytest.mark.parametrize("count", [9, 15, 16, 17, 24])
def test_batch_sizes_match_oracle_engine(sess, monkeypatch, form, count):
    """prove_batch_native over 9..24 members (Jolt stages batch 5-20) against the oracle engine: challenges, every
    batched round polynomial, member claims and final evaluations; the sequential traversal
    (JB_SEQUENTIAL_ROUNDS=1) must give the identical proof."""
    shapes = batch_shapes(form, count)
    order = LOW_TO_HIGH if count % 2 else HIGH_TO_LOW
    tabs, desc, total, max_vars = batch_fixture(shapes, 7000 + count)
    max_deg = max(m for m, _, _ in shapes)
    pts = O.synthetic_point(max_vars, 401)
    want = O.prove_batch(desc, [O.ProductMember(t, order) for t in tabs], max_vars, max_deg, total, lambda r, c: pts[r])

    def prove():
        mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], order) for tb in tabs]
        got = jolt_b200.prove_batch_native([BatchMember(**d) for d in desc], mems, max_vars, max_deg, total,
                                           lambda r, poly: pts[r])
        fe = [m.final_evals() for m in mems]
        for m in mems:
            m.close()
        return got, fe

    got, fe = prove()
    assert got.challenges == want["challenges"] and got.final_claim == want["final_claim"]
    assert got.member_claims == want["member_claims"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for f, tb, d in zip(fe, tabs, desc):
        window = pts[d["offset"]:d["offset"] + d["rounds"]]
        point = window if order == HIGH_TO_LOW else list(reversed(window))
        assert f == [O.evaluate(t, point) for t in tb]
    monkeypatch.setenv("JB_SEQUENTIAL_ROUNDS", "1")
    seq, seq_fe = prove()
    assert seq.challenges == got.challenges and seq.final_claim == got.final_claim
    assert seq.member_claims == got.member_claims and seq_fe == fe
    assert [p.coefficients for p in seq.round_polynomials] == [p.coefficients for p in got.round_polynomials]


def test_scheduler_direct_17_members(sess):
    """RoundScheduler::batch_prove_round with 17 active members (more than the result slots) == member by member"""
    n, count = 9, 17
    tabs = [[O.random_fr(9100 + 10 * i + j, 1 << n) for j in range(2)] for i in range(count)]
    ch = O.synthetic_point(n, 23)
    claims0 = [sum(a * b for a, b in zip(*tb)) % P for tb in tabs]

    mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], HIGH_TO_LOW) for tb in tabs]
    claims, seq = list(claims0), []
    for rnd in range(n):
        polys = [m.prove_round(None if rnd == 0 else ch[rnd - 1], rnd, c) for m, c in zip(mems, claims)]
        seq.append([p.coefficients for p in polys])
        claims = [p.evaluate(ch[rnd]) for p in polys]
    for m in mems:
        m.finish_rounds(ch[-1])
    seq_final = [m.final_evals() for m in mems]

    mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], HIGH_TO_LOW) for tb in tabs]
    sched = RoundScheduler(sess, mems)
    claims, got = list(claims0), []
    for rnd in range(n):
        polys = sched.batch_prove_round([(i, rnd, None if rnd == 0 else ch[rnd - 1], claims[i]) for i in range(count)])
        got.append([p.coefficients for p in polys])
        claims = [p.evaluate(ch[rnd]) for p in polys]
    sched.batch_finish_rounds([(i, ch[-1]) for i in range(count)])
    assert got == seq and [m.final_evals() for m in mems] == seq_final
    assert seq_final == [[O.evaluate(t, ch) for t in tb] for tb in tabs]
    sched.close()
