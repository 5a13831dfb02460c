"""The LT and eq+1 tables on the device (jb_lt_evals, jb_eq_plus_one_evals): bit-exact against the C build for every n
from 0 to 14 (single-block and streaming paths, scaled and unscaled, 125-bit, full and extreme coordinates) and in full
at 2^22 and 2^24; evaluations and sums against the closed forms; value evaluation and shift sumchecks over them in
lockstep with the expression reference, and their final claims against the closed forms at 2^20; every error."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (EqPlusOnePolynomial, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, LtPolynomial, Polynomial,
                       ProductSourcesMember, Source, UnivariatePoly, _lib)
from jolt_b200 import field as F
from oracle import bn254 as O
from gpu_util import rand_challenge
import source_ref as SR
import structured_ref as R
import sumcheck_ref as S
from test_gpu_expr_sources import _challenge, address_column, compact_column

pytestmark = pytest.mark.gpu
P = O.R_MOD
P_MINUS_1 = F.to_limbs(P - 1)
ONE = F.to_limbs(1)


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def point(kind: str, n: int, seed: int) -> np.ndarray:
    """(n, 4) Montgomery limbs: 'full' uniform over [0, p), 'short' 125-bit challenges, 'extreme' the extreme
    challenges, 1 and p - 1 interleaved with full coordinates."""
    if n == 0:
        return np.zeros((0, 4), dtype=np.uint64)
    if kind == "full":
        return S.rand_limbs_full(seed, n)
    if kind == "short":
        return np.stack([rand_challenge(seed + i) for i in range(n)])
    pool = list(S.EXTREME_CHALLENGES) + [P_MINUS_1, ONE]
    full = S.rand_limbs_full(seed, n)
    return np.stack([pool[i % len(pool)] if i % 3 != 2 else full[i] for i in range(n)])


def _scale(scaled: bool, seed: int):
    return S.rand_limbs_full(seed, 1)[0] if scaled else None


BUILDS = {"lt": (LtPolynomial, R.lt_evals_c), "eq_plus_one": (EqPlusOnePolynomial, R.eq_plus_one_evals_c)}


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("kind", ["full", "short", "extreme"])
@pytest.mark.parametrize("n", range(15))
@pytest.mark.parametrize("table", list(BUILDS))
def test_table_bit_exact(sess, table, n, kind, scaled):
    cls, cref = BUILDS[table]
    r, sc = point(kind, n, 0x5100 + n), _scale(scaled, 0x5200 + n)
    got = cls.evals(sess, r, sc)
    assert len(got) == 1 << n
    assert np.array_equal(got.evals(), cref(r, sc)), (table, n, kind, scaled)


def test_scale_p_minus_one_matches_python(sess):
    n = 9
    r = point("extreme", n, 0x5300)
    ri = F.limbs_to_ints(r)
    assert LtPolynomial.evals(sess, r, P - 1).to_ints() == R.lt_table(ri, P - 1)
    assert EqPlusOnePolynomial.evals(sess, r, P - 1).to_ints() == R.eq_plus_one_table(ri, P - 1)


@pytest.mark.parametrize("n,kind,scaled", [(22, "short", True), (22, "full", False), (24, "short", False),
                                           (24, "full", True)])
@pytest.mark.parametrize("table", list(BUILDS))
def test_large_tables_in_full(sess, table, n, kind, scaled):
    cls, cref = BUILDS[table]
    r, sc = point(kind, n, 0x5400 + n), _scale(scaled, 0x5500 + n)
    got = cls.evals(sess, r, sc)
    assert np.array_equal(got.evals(), cref(r, sc))
    got.free()


@pytest.mark.parametrize("kind", ["short", "full"])
def test_evaluations_are_the_closed_forms_at_2_24(sess, kind):
    n = 24
    r, sc = point(kind, n, 0x5600), S.rand_limbs_full(0x5601, 1)[0]
    ri, s = F.limbs_to_ints(r), F.from_limbs(sc)
    lt, e1 = LtPolynomial.evals(sess, r, sc), EqPlusOnePolynomial.evals(sess, r, sc)
    for k in range(3):
        rho = O.random_fr(0x5610 + k, n)
        got = Polynomial.batch_evaluate([lt, e1], F.ints_to_limbs(rho))
        assert got[0] == s * LtPolynomial.evaluate(rho, ri) % P
        assert got[1] == s * EqPlusOnePolynomial.evaluate(ri, rho) % P
    lt.free()
    e1.free()


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("n", [1, 11, 12, 16])
def test_sums_are_the_closed_forms(sess, n, scaled):
    r, sc = point("full", n, 0x5700 + n), _scale(scaled, 0x5701)
    ri, s = F.limbs_to_ints(r), 1 if sc is None else F.from_limbs(sc)
    prod = 1
    for v in ri:
        prod = prod * v % P
    assert sum(LtPolynomial.evals(sess, r, sc).to_ints()) % P == s * sum(v << (n - 1 - i) for i, v in enumerate(ri)) % P
    assert sum(EqPlusOnePolynomial.evals(sess, r, sc).to_ints()) % P == s * (1 - prod) % P


# ---- the relations -------------------------------------------------------------------------------------------------
def _rho(chs, order):
    """the bound point MSB first: HighToLow binds the most significant variable first"""
    pts = [F.from_limbs(c) for c in chs]
    return pts if order == HIGH_TO_LOW else pts[::-1]


def _lockstep(gpu, ref, n, seed):
    claim = ref.claim()
    bind, chs = None, []
    for rnd in range(n):
        want = ref.round_evals(None if bind is None else F.from_limbs(bind))
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = _challenge(rnd, seed)
        chs.append(bind)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    ref.finish_rounds(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    fin = gpu.final_evals()
    assert fin == ref.final_evals()
    return fin, claim, chs


def _value_eval_inputs(n, seed):
    wa = address_column(n, 64, seed, dtype=np.uint8)
    inc, inc_ref = compact_column("i64", n, seed + 1)
    r_addr, r_cycle = O.random_fr(seed + 2, 6), point("short", n, seed + 3)
    return wa, inc, inc_ref, r_addr, r_cycle


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 5, 12])
def test_value_evaluation_expression(sess, n, order):
    """Val(r_addr, r_cycle) = sum_j inc(j) wa(r_addr, j) LT(j, r_cycle): registers (K = 64, u8), inc as i64"""
    seed = 0x5800 + n
    wa, inc, inc_ref, r_addr, r_cycle = _value_eval_inputs(n, seed)
    lt = LtPolynomial.evals(sess, r_cycle)
    mons = [(1, [0, 1, 2])]
    ref = SR.SourcesMember([("one_hot", SR.addresses(wa), 64, r_addr), ("compact", inc_ref), ("table", lt.to_ints())],
                           mons, order)
    gpu = ExpressionMember.from_sources(sess, [Source.one_hot(wa, 64, r_addr), Source.compact(inc, "i64"),
                                               Source.table(lt)], mons, order=order)
    fin, claim, chs = _lockstep(gpu, ref, n, seed)
    assert fin[2] == LtPolynomial.evaluate(_rho(chs, order), F.limbs_to_ints(r_cycle))
    assert claim == fin[0] * fin[1] * fin[2] % P
    gpu.close()


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 3, 12])
def test_value_evaluation_product_of_address_chunks(sess, n, order):
    """RAM: the address split into two u8 chunks, sum_j ra_0(r_0, j) ra_1(r_1, j) inc(j) LT(j, r_cycle)"""
    seed = 0x5900 + n
    a0, a1 = address_column(n, 256, seed, dtype=np.uint8), address_column(n, 256, seed + 1, dtype=np.uint8)
    inc, inc_ref = compact_column("i128", n, seed + 2)
    r0, r1, r_cycle = O.random_fr(seed + 3, 8), O.random_fr(seed + 4, 8), point("full", n, seed + 5)
    sc = S.rand_limbs_full(seed + 6, 1)[0]
    lt = LtPolynomial.evals(sess, r_cycle, sc)
    ref = SR.SourcesMember([("one_hot", SR.addresses(a0), 256, r0), ("one_hot", SR.addresses(a1), 256, r1),
                            ("compact", inc_ref), ("table", lt.to_ints())], [(1, [0, 1, 2, 3])], order)
    gpu = ProductSourcesMember.from_sources(sess, [Source.one_hot(a0, 256, r0), Source.one_hot(a1, 256, r1),
                                                   Source.compact(inc, "i128"), Source.table(lt)], order=order)
    fin, claim, chs = _lockstep(gpu, ref, n, seed)
    assert fin[3] == F.from_limbs(sc) * LtPolynomial.evaluate(_rho(chs, order), F.limbs_to_ints(r_cycle)) % P
    assert claim == fin[0] * fin[1] * fin[2] * fin[3] % P
    gpu.close()


def _pc_columns(n, seed):
    rng = np.random.default_rng(seed)
    pc = rng.integers(0, 1 << 63, 1 << n, dtype=np.uint64) * np.uint64(2) + np.uint64(rng.integers(0, 2))
    upc = rng.integers(0, 1 << 64, 1 << n, dtype=np.uint64)
    upc[::7] = np.uint64((1 << 64) - 1)
    return pc, upc


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 6, 12])
def test_shift_expression(sess, n, order):
    """NextPC(r) + gamma NextUnexpandedPC(r) = sum_j EqPlusOne(r, j) (PC(j) + gamma UnexpandedPC(j)), u64 columns"""
    seed = 0x5A00 + n
    pc, upc = _pc_columns(n, seed)
    r, gamma = point("extreme", n, seed + 1), O.random_fr(seed + 2, 1)[0]
    e1 = EqPlusOnePolynomial.evals(sess, r)
    mons = [(1, [0, 1]), (gamma, [0, 2])]
    ref = SR.SourcesMember([("table", e1.to_ints()), ("compact", [int(v) for v in pc]),
                            ("compact", [int(v) for v in upc])], mons, order)
    gpu = ExpressionMember.from_sources(sess, [Source.table(e1), Source.compact(pc, "u64"), Source.compact(upc, "u64")],
                                        mons, order=order)
    fin, claim, chs = _lockstep(gpu, ref, n, seed)
    assert fin[0] == EqPlusOnePolynomial.evaluate(F.limbs_to_ints(r), _rho(chs, order))
    assert claim == fin[0] * (fin[1] + gamma * fin[2]) % P
    gpu.close()


def _drive(gpu, n, claim, seed):
    chs = []
    bind = None
    for rnd in range(n):
        got = gpu.prove_round_evals(bind, rnd, claim)
        bind = _challenge(rnd, seed)
        chs.append(bind)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    return gpu.final_evals(), claim, chs


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_final_claims_are_the_closed_forms_at_2_20(sess, order):
    n, seed = 20, 0x5B00
    wa, inc, inc_ref, r_addr, r_cycle = _value_eval_inputs(n, seed)
    lt = LtPolynomial.evals(sess, r_cycle)
    eq_addr = O.eq_evals(r_addr)
    wa_vals = [0 if a is None else eq_addr[a] for a in SR.addresses(wa)]
    inc_vals = SR.promote_column(inc_ref)
    claim = sum(a * b * c for a, b, c in zip(wa_vals, inc_vals, lt.to_ints())) % P
    gpu = ExpressionMember.from_sources(sess, [Source.one_hot(wa, 64, r_addr), Source.compact(inc, "i64"),
                                               Source.table(lt)], [(1, [0, 1, 2])], order=order)
    fin, final_claim, chs = _drive(gpu, n, claim, seed)
    rho = _rho(chs, order)
    assert fin[2] == LtPolynomial.evaluate(rho, F.limbs_to_ints(r_cycle))
    assert final_claim == fin[0] * fin[1] * fin[2] % P
    gpu.close()

    pc, upc = _pc_columns(n, seed + 1)
    r, gamma = point("full", n, seed + 2), O.random_fr(seed + 3, 1)[0]
    e1 = EqPlusOnePolynomial.evals(sess, r)
    claim = sum(e * (int(a) + gamma * int(b)) for e, a, b in zip(e1.to_ints(), pc, upc)) % P
    gpu = ExpressionMember.from_sources(sess, [Source.table(e1), Source.compact(pc, "u64"), Source.compact(upc, "u64")],
                                        [(1, [0, 1]), (gamma, [0, 2])], order=order)
    fin, final_claim, chs = _drive(gpu, n, claim, seed + 4)
    assert fin[0] == EqPlusOnePolynomial.evaluate(F.limbs_to_ints(r), _rho(chs, order))
    assert final_claim == fin[0] * (fin[1] + gamma * fin[2]) % P
    gpu.close()


# ---- errors --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["jb_lt_evals", "jb_eq_plus_one_evals"])
def test_errors_leave_the_context_usable(sess, fn):
    f = getattr(sess.lib, fn)
    h = ctypes.c_uint64()
    r = point("full", 41, 0x5C00)
    rp = r.ctypes.data_as(_lib.c_u64p)
    bad = np.array([(P >> (64 * w)) & (2**64 - 1) for w in range(4)], dtype=np.uint64)  # p itself: not canonical
    r_bad = r[:4].copy()
    r_bad[2] = bad
    cases = [
        (lambda: f(sess.h, rp, 3, None, None), _lib.JB_ERR_INVALID),                 # null out
        (lambda: f(sess.h, None, 3, None, ctypes.byref(h)), _lib.JB_ERR_INVALID),    # null point
        (lambda: f(sess.h, rp, 41, None, ctypes.byref(h)), _lib.JB_ERR_INVALID),     # nvars > 40
        (lambda: f(sess.h, r_bad.ctypes.data_as(_lib.c_u64p), 4, None, ctypes.byref(h)), _lib.JB_ERR_INVALID),
        (lambda: f(sess.h, rp, 4, bad.ctypes.data_as(_lib.c_u64p), ctypes.byref(h)), _lib.JB_ERR_INVALID),
        (lambda: f(sess.h, rp, 40, None, ctypes.byref(h)), _lib.JB_ERR_OOM),         # 32 TiB
    ]
    cls, cref = BUILDS["lt" if fn == "jb_lt_evals" else "eq_plus_one"]
    for i, (call, want) in enumerate(cases):
        h.value = 0
        assert call() == want, i
        assert h.value == 0, i
        t = cls.evals(sess, r[:13])
        assert np.array_equal(t.evals(), cref(r[:13])), i
        t.free()
