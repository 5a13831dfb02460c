"""Expression members and members over sources at their declared limits (JB_EXPR_MAX_TABLES = 8 tables or sources,
JB_EXPR_MAX_MONOMIALS = 16 monomials, JB_EXPR_MAX_DEGREE = 6): every round, the final evaluations and eq(w, r) in
lockstep with tests/expr_ref.py and tests/source_ref.py (pinned against brute force by tests/test_expr_limits_ref_cpu.py);
the largest shapes at 2^18 .. 2^24 against an initial claim and final evaluations computed on the host with the C
oracle; the batch engine and the scheduler with limit members in the batch (a degree-6 eq member fills the scheduler's
8-evaluation row); and the refusals one past each limit.

Where these shapes reach paths that smaller ones do not: from 6 tables the expression pass needs more than the 48 KiB
default of dynamic shared memory, at 7-8 tables its occupancy drops to 3 blocks per SM, 8 staged one-hot sources fill the
source pass's largest shared-memory layout, and staged and L2-read one-hot sources interleave in it."""
import ctypes
import functools

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (BatchMember, EqProductMember, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, ProductMember,
                       RoundScheduler, Source, UnivariatePoly, _lib, one_hot_evaluate, small_scalars)
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
import expr_ref as E
import mle_eval_ref as M
import source_ref as SR
import sumcheck_ref as S

pytestmark = pytest.mark.gpu
P = O.R_MOD
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
R_LIMBS_COEFF = S.int_to_limbs(S.R_MONT)   # Montgomery limbs R: the value 1
PM1_LIMBS_COEFF = S.int_to_limbs(P - 1)    # Montgomery limbs p - 1
SCALE = (P - 1) * GAMMA % P

# 8 tables, 16 monomials of degrees 1..6; coefficients 1, -1, 0, general values and Montgomery-limb extremes
MAX_MONOMIALS = [
    (GAMMA, [3] * 6),
    (-1, [7, 0, 7, 1, 7, 2]),
    (1, [4, 5, 6]),
    (0, [0, 1, 2, 3, 4]),
    (PM1_LIMBS_COEFF, [5, 6]),
    (R_LIMBS_COEFF, [6, 7, 0, 1]),
    ((1 << 256) % P, [1]),
    (GAMMA * GAMMA % P, [2, 4, 6, 0, 2, 4]),
    (P - 1, [5]),
    (3, [7, 7]),
    (GAMMA + 1, [0, 1, 2, 3, 4, 5]),
    (1, [6, 6, 6, 1, 1]),
    (S.C_SIGN, [2, 5, 7]),
    (-GAMMA, [3, 4]),
    (7, [1, 2, 3, 5, 6, 7]),
    (1, [0]),
]


def table_count_monomials(T):
    """D = 6 over T tables, every table used"""
    return [(GAMMA, [i % T for i in range(6)]), (-1, [T - 1, T - 1]), (5, list(range(5, T)) + [1])]


def fold_monomials(monomials, T):
    """the monomials with table t read as t mod T (every one of T <= 8 tables stays used)"""
    return [(c, [t % T for t in tabs]) for c, tabs in monomials]


# name -> (tables, monomials, eq, scale). None of them is a unit-coefficient product / sum of products, so each gets
# the expression pass (asserted).
SHAPES = {
    "max": (8, MAX_MONOMIALS, False, None),
    "max_eq": (8, MAX_MONOMIALS, True, None),
    "max_eq_scaled": (8, MAX_MONOMIALS, True, SCALE),
    "tables5_d6": (5, table_count_monomials(5), False, None),
    "tables6_d6_eq": (6, table_count_monomials(6), True, None),
    "tables7_d6": (7, table_count_monomials(7), False, None),
    "tables8_d6_eq_scaled": (8, table_count_monomials(8), True, SCALE),
    "d4": (4, [(GAMMA, [0, 1, 2, 3]), (-1, [1, 2]), (3, [0])], False, None),
    "d5": (5, [(PM1_LIMBS_COEFF, [0, 1, 2, 3, 4]), (GAMMA, [4, 4, 0])], False, None),
    "d6": (3, [(7, [0, 0, 1, 1, 2, 2]), (1, [2])], False, None),
    "d5_eq": (4, [(GAMMA, [0, 1, 2, 3, 0]), (1, [1, 3])], True, None),
}


def coeff_int(c):
    return c % P if isinstance(c, int) else F.from_limbs(c)


def ref_monomials(monomials):
    return [(coeff_int(c), list(t)) for c, t in monomials]


def expr_inputs(shape, n, order):
    """the tables (limbs) and the eq point (limbs or None) of a lockstep case"""
    T, _, eq, _ = SHAPES[shape]
    seed = 0xE800 + 16 * n
    if n >= 9:
        tabs = [S.extreme_table(seed + j, n, order, rotate=j) for j in range(T)]
    else:
        tabs = [S.rand_limbs_full(seed + j, 1 << n) for j in range(T)]
    return tabs, (S.extreme_point(0x4E + n, n, zero=False) if eq else None)


def challenge(rnd, seed):
    ch = S.extreme_challenge(rnd, seed)   # 125-bit and full challenges, interleaved with the extreme ones
    return ch if ch.any() else S.EXTREME_CHALLENGES[2]   # (a zero challenge against an eq coordinate 1 zeroes eq)


def run_reference(ref, n, seed):
    """(initial claim, every round's evaluations, final evaluations, eq scalar or None) of a reference member under
    the challenges challenge(rnd, seed)"""
    claim = ref.claim()
    rounds, bind = [], None
    for rnd in range(n):
        rounds.append(ref.round_evals(None if bind is None else F.from_limbs(bind)))
        bind = challenge(rnd, seed)
    ref.finish_rounds(F.from_limbs(bind))
    return claim, rounds, ref.final_evals(), (ref.eq_scalar() if ref.eq is not None else None)


@functools.lru_cache(maxsize=None)
def expr_transcript(shape, n, order):
    T, mons, eq, scale = SHAPES[shape]
    tabs, w = expr_inputs(shape, n, order)
    ref = E.ExpressionMember([F.limbs_to_ints(t) for t in tabs], ref_monomials(mons), order,
                             None if w is None else F.limbs_to_ints(w), scale)
    return run_reference(ref, n, n)


def assert_expression_pass(sess, member):
    """the member is served by the expression pass, not by a built product / eq member (those are sharded)"""
    torch = pytest.importorskip("torch")
    lanes = torch.zeros(64, dtype=torch.int64, device="cuda")
    assert sess.lib.jb_member_prove_round_partials(member.h, None, 0, 0, ctypes.c_void_p(lanes.data_ptr())) == \
        _lib.JB_ERR_UNSUPPORTED


def drive_lockstep(gpu, transcript, monomials, n, seed):
    claim, rounds, fin_want, eq_want = transcript
    bind = None
    for rnd in range(n):
        want = rounds[rnd]
        assert (want[0] + want[1]) % P == claim
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = challenge(rnd, seed)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    fin = gpu.final_evals()
    assert fin == fin_want
    value = E.expr_value(fin, ref_monomials(monomials))
    if eq_want is not None:
        assert gpu.eq_scalar() == eq_want
        value = value * eq_want % P
    assert value == claim


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


# ---- expression members in lockstep with the reference ----------------------------------------------------------
@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 9, 12])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_expr_limits_lockstep_vs_reference(sess, sess_verify, shape, n, order, verify):
    s = sess_verify if verify else sess
    T, mons, eq, scale = SHAPES[shape]
    tabs, w = expr_inputs(shape, n, order)
    gpu = ExpressionMember(s, [Polynomial.new(s, t) for t in tabs], mons, w, scale, order=order)
    assert_expression_pass(s, gpu)
    assert gpu.num_rounds() == n and gpu.degree() == E.expr_degree(mons, eq)
    drive_lockstep(gpu, expr_transcript(shape, n, order), mons, n, n)
    gpu.close()


# ---- sources at the limits ----------------------------------------------------------------------------------------
NAMED = {"u128", "i128", "s64", "s128"}   # kinds that Source.compact takes as Python values with the kind named
MIXED8 = ["oh_u8_256", "i128", "oh_u16_65536", "s128", "oh_u8_1", "u8", "table", "i64"]   # staged, L2, staged one-hot


def one_hot_params(spec):
    _, width, K = spec.split("_")
    return (np.uint8 if width == "u8" else np.uint16), int(K)


def make_source(sess, spec, n, seed, on_device=False):
    """(device source, reference source) of one source of a case: "oh_<u8|u16>_<K>", "table" or a compact kind"""
    if spec.startswith("oh_"):
        dt, K = one_hot_params(spec)
        a = SR.address_column(n, K, seed, dtype=dt)
        r = O.random_fr(seed + 1, K.bit_length() - 1)
        col = a
        if on_device:   # (a 16-bit column travels as int16: its raw words)
            import torch
            col = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()
        return Source.one_hot(col, K, r), ("one_hot", SR.addresses(a), K, r)
    if spec == "table":
        t = S.rand_limbs_full(seed, 1 << n)
        return (Source.table(Polynomial.new(sess, t)) if sess is not None else None), ("table", F.limbs_to_ints(t))
    col, vals = SR.compact_column(spec, n, seed)
    if on_device and spec not in NAMED:
        import torch
        col = torch.from_numpy(col).cuda()
    return Source.compact(col, spec if spec in NAMED else None), ("compact", vals)


# name -> (source specs, eq, scale, columns as CUDA tensors)
SOURCE_CASES = {
    "one_hot8_u8_K256": (["oh_u8_256"] * 8, True, SCALE, False),
    "mixed8": (MIXED8, True, None, False),
    "mixed8_cuda_columns": (["oh_u16_65536", "u8", "oh_u8_256", "i64", "s128", "oh_u8_1", "table", "i128"], False, None, True),
}
SOURCE_CASES.update({f"mixed{k}": (MIXED8[:k], k % 2 == 1, None, False) for k in (5, 6, 7)})


def source_monomials(k):
    return fold_monomials(MAX_MONOMIALS, k)


def source_seed(case, n):
    return 0x5A00 + 64 * n + 8 * sorted(SOURCE_CASES).index(case)


def source_inputs(sess, case, n):
    specs, eq, _, dev = SOURCE_CASES[case]
    seed = source_seed(case, n)
    pairs = [make_source(sess, spec, n, seed + 4 * j, dev and sess is not None) for j, spec in enumerate(specs)]
    w = S.extreme_point(0x5E + n, n, zero=False) if eq else None
    return [p[0] for p in pairs], [p[1] for p in pairs], w


@functools.lru_cache(maxsize=None)
def source_transcript(case, n, order):
    specs, eq, scale, _ = SOURCE_CASES[case]
    _, refsrc, w = source_inputs(None, case, n)
    ref = SR.SourcesMember(refsrc, ref_monomials(source_monomials(len(specs))), order,
                           None if w is None else F.limbs_to_ints(w), scale)
    return run_reference(ref, n, n)


def source_lockstep_cases():
    for case in sorted(SOURCE_CASES):
        for n in ([1, 2, 3, 5, 9] if len(SOURCE_CASES[case][0]) == 8 else [1, 2]):   # 5-7 sources: the terminal bind
            yield case, n


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("case,n", list(source_lockstep_cases()))
def test_sources_limits_lockstep_vs_reference(sess, sess_verify, case, n, order, verify):
    s = sess_verify if verify else sess
    specs, eq, scale, _ = SOURCE_CASES[case]
    mons = source_monomials(len(specs))
    dev, _, w = source_inputs(s, case, n)
    gpu = ExpressionMember.from_sources(s, dev, mons, w, scale, order=order)
    assert_expression_pass(s, gpu)
    assert gpu.num_rounds() == n and gpu.degree() == E.expr_degree(mons, eq)
    drive_lockstep(gpu, source_transcript(case, n, order), mons, n, n)
    gpu.close()


# ---- at scale: the claim and the final evaluations from the host ------------------------------------------------
THREADS = C.max_threads()
CHUNK_BITS = 20


def eq_point_value(w, r):
    """eq(w, r) of two points in index order (coordinate 0 <-> the index MSB)"""
    v = 1
    for a, b in zip(w, r):
        v = v * (a * b + (1 - a) * (1 - b)) % P
    return v


def host_claim(n, chunk, monomials, w=None, scale=None):
    """sum_x [scale eq(w, x)] sum_k c_k prod_i f_{t_k,i}(x) with the C oracle, 2^CHUNK_BITS indices at a time:
    chunk(lo, hi) -> the tables' limbs over [lo, hi). A monomial (with the chunk of the eq table as one more factor) is
    a product of at most 7 tables, and its first-round s(0) + s(1) is its sum over the chunk."""
    bits = min(n, CHUNK_BITS)
    total = 0
    for c in range(1 << (n - bits)):
        tabs = chunk(c << bits, (c + 1) << bits)
        extra = []
        if w is not None:   # eq(w, x) = eq(w_hi, c) * eq(w_lo, x_lo) on the chunk whose high index bits are c
            hi = [(c >> (n - bits - 1 - i)) & 1 for i in range(n - bits)]
            pre = eq_point_value(w[:n - bits], hi) * (1 if scale is None else scale) % P
            extra = [C.eq_evals(F.ints_to_limbs(w[n - bits:]), F.to_limbs(pre), threads=THREADS)]
        for coeff, idx in ref_monomials(monomials):
            ev = C.product_round_evals(extra + [tabs[t] for t in idx], 1, HIGH_TO_LOW, threads=THREADS)
            total += coeff * sum(F.limbs_to_ints(ev))
    return total % P


def host_final(table, challenges, order):
    """the table's value at the challenges, bound one variable at a time with the C oracle"""
    for ch in challenges:
        table = C.bind(table, ch, order, threads=THREADS)
    return F.from_limbs(table[0])


def prove_from_claim(gpu, n, order, claim, seed):
    """every round from an initial claim computed outside the member; returns (final claim, challenges, the point in
    index order)"""
    bind, chs = None, []
    for rnd in range(n):
        ev = gpu.prove_round_evals(bind, rnd, claim)
        assert (ev[0] + ev[1]) % P == claim
        bind = challenge(rnd, seed)
        chs.append(bind)
        claim = UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    r = [F.from_limbs(c) for c in chs]
    return claim, chs, (r if order == HIGH_TO_LOW else list(reversed(r)))


def check_final_claim(gpu, claim, monomials, w, scale, point):
    fin = gpu.final_evals()
    value = E.expr_value(fin, ref_monomials(monomials))
    if w is not None:
        eq = eq_point_value(w, point) * (1 if scale is None else scale) % P
        assert gpu.eq_scalar() == eq
        value = value * eq % P
    assert claim == value
    return fin


@pytest.mark.parametrize("n,order,eq", [(18, LOW_TO_HIGH, False), (18, HIGH_TO_LOW, True), (22, HIGH_TO_LOW, False),
                                        (22, LOW_TO_HIGH, True)])
def test_max_shape_at_scale(sess, n, order, eq):
    seed = 0xC100 + n + order
    tabs = [S.extreme_table(seed + j, n, order, rotate=j) for j in range(8)]
    w = O.random_fr(seed + 9, n) if eq else None
    scale = SCALE if eq else None
    claim = host_claim(n, lambda lo, hi: [t[lo:hi] for t in tabs], MAX_MONOMIALS, w, scale)
    gpu = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], MAX_MONOMIALS,
                           None if w is None else F.ints_to_limbs(w), scale, order=order)
    assert_expression_pass(sess, gpu)
    fin_claim, chs, point = prove_from_claim(gpu, n, order, claim, seed)
    fin = check_final_claim(gpu, fin_claim, MAX_MONOMIALS, w, scale, point)
    assert fin == [host_final(t, chs, order) for t in tabs]
    gpu.close()


def palette_column(spec, n, seed):
    """2^n compact entries drawn from a palette of the kind's magnitude extremes (both signs; -0 for the sign-magnitude
    kinds) and random values: (the column as Source.compact takes it, its promoted limbs)"""
    rng = np.random.default_rng(seed)
    top = max(SR.MAGS[spec])
    pal = list(SR.MAGS[spec]) + [int(v) for v in rng.integers(0, min(top, 1 << 62), 4)]
    if spec in ("i64", "i128"):
        pal = [min(m, top - 1) for m in pal] + [-m for m in pal]
    if spec in ("s64", "s128"):
        pal = [(m, True) for m in pal] + [(m, False) for m in pal]
    idx = rng.integers(0, len(pal), 1 << n)
    recs, _, _ = small_scalars(pal if spec in NAMED else np.array(pal, dtype={"u8": np.uint8, "i64": np.int64}[spec]),
                               spec if spec in NAMED else None)
    limbs = F.ints_to_limbs([M.promote(v) for v in pal])[idx]
    col = np.ascontiguousarray(recs[idx])
    if spec in NAMED:   # the raw records, on the device
        import torch
        return Source.compact(torch.from_numpy(col.view(np.int64)).cuda(), spec), limbs
    return Source.compact(col), limbs


def gathered_limbs(addr, K, r_addr):
    """eq(r_addr, addr[j]) as limbs, 0 for the none value (the all-ones value of the width, an address below K = 2^8 or
    2^16 too)"""
    eq = C.eq_evals(F.ints_to_limbs(r_addr)) if len(r_addr) else F.ints_to_limbs([1])
    idx = addr.astype(np.int64)
    idx[(addr == np.iinfo(addr.dtype).max) | (idx >= K)] = K
    return np.concatenate([eq, np.zeros((1, 4), np.uint64)])[idx]


@pytest.mark.parametrize("case,n,order,eq", [("mixed8", 22, HIGH_TO_LOW, True), ("mixed8", 22, LOW_TO_HIGH, False),
                                             ("one_hot8_u8_K256", 24, LOW_TO_HIGH, True)])
def test_sources_at_scale(sess, case, n, order, eq):
    specs = SOURCE_CASES[case][0]
    seed = 0xC900 + n + order
    mons = source_monomials(len(specs))
    dev, host, one_hot = [], [], []   # host: per source a function (lo, hi) -> limbs, or the whole table
    for j, spec in enumerate(specs):
        if spec.startswith("oh_"):
            dt, K = one_hot_params(spec)
            a = SR.address_column(n, K, seed + 4 * j, dtype=dt)
            r = O.random_fr(seed + 4 * j + 1, K.bit_length() - 1)
            dev.append(Source.one_hot(a, K, r))
            host.append(functools.partial(lambda a, K, r, lo, hi: gathered_limbs(a[lo:hi], K, r), a, K, r))
            one_hot.append((j, a, K, r))
        elif spec == "table":
            t = S.extreme_table(seed + 4 * j, n, order)
            dev.append(Source.table(Polynomial.new(sess, t)))
            host.append(t)
        else:
            src, limbs = palette_column(spec, n, seed + 4 * j)
            dev.append(src)
            host.append(limbs)
    w = O.random_fr(seed + 99, n) if eq else None
    scale = SCALE if eq else None
    claim = host_claim(n, lambda lo, hi: [h(lo, hi) if callable(h) else h[lo:hi] for h in host], mons, w, scale)
    gpu = ExpressionMember.from_sources(sess, dev, mons, None if w is None else F.ints_to_limbs(w), scale, order=order)
    assert_expression_pass(sess, gpu)
    fin_claim, chs, point = prove_from_claim(gpu, n, order, claim, seed)
    fin = check_final_claim(gpu, fin_claim, mons, w, scale, point)
    for j, h in enumerate(host):
        assert fin[j] == host_final(h(0, 1 << n) if callable(h) else h, chs, order), f"source {j} ({specs[j]})"
    for j, a, K, r in one_hot:
        if K > 1:
            assert fin[j] == one_hot_evaluate(sess, a, K, point + list(r))[0], f"source {j}"
    gpu.close()


# ---- the batch engine and the scheduler ---------------------------------------------------------------------------
def limit_batch(sess, count, seed):
    """ragged members: limit expression members (with eq up to degree 7: 8 evaluations), limit members over sources,
    product and eq members; returns (device members, reference members, descs)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    dev, ref, desc = [], [], []
    kinds = ["max", "tables8_d6_eq_scaled", "mixed8", "product", "max_eq", "one_hot8_u8_K256", "eq"]
    for i in range(count):
        n = int(rng.integers(3, 8))
        kind = kinds[i % len(kinds)]
        if kind in SHAPES:
            T, mons, eq, scale = SHAPES[kind]
            tabs = [S.rand_limbs_full(seed * 100 + 10 * i + j, 1 << n) for j in range(T)]
            w = S.extreme_point(seed * 100 + 10 * i + 9, n, zero=False) if eq else None
            r = E.ExpressionMember([F.limbs_to_ints(t) for t in tabs], ref_monomials(mons), LOW_TO_HIGH,
                                   None if w is None else F.limbs_to_ints(w), scale)
            d = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], mons, w, scale, order=LOW_TO_HIGH)
        elif kind in SOURCE_CASES:
            specs, eq, scale, _ = SOURCE_CASES[kind]
            mons = source_monomials(len(specs))
            pairs = [make_source(sess, spec, n, seed * 100 + 10 * i + j) for j, spec in enumerate(specs)]
            w = S.extreme_point(seed * 100 + 10 * i + 9, n, zero=False) if eq else None
            r = SR.SourcesMember([p[1] for p in pairs], ref_monomials(mons), LOW_TO_HIGH,
                                 None if w is None else F.limbs_to_ints(w), scale)
            d = ExpressionMember.from_sources(sess, [p[0] for p in pairs], mons, w, scale, order=LOW_TO_HIGH)
        else:
            tabs = [O.random_fr(seed * 100 + 10 * i + j, 1 << n) for j in range(2)]
            w = O.random_fr(seed * 100 + 10 * i + 9, n) if kind == "eq" else None
            r = E.ExpressionMember(tabs, [(1, [0, 1])], LOW_TO_HIGH, w)
            polys = [Polynomial.from_ints(sess, t) for t in tabs]
            d = ProductMember(sess, polys, LOW_TO_HIGH) if w is None else \
                EqProductMember(sess, polys, F.ints_to_limbs(w), order=LOW_TO_HIGH)
        dev.append(d)
        ref.append(r)
        desc.append((r.claim(), (i * 7 + 3) % P, n))
    return dev, ref, desc


def challenge_fn(rnd, coeffs):
    return (sum(int(c) for c in coeffs) * 7 + 31 * rnd + 5) % P


@pytest.mark.parametrize("count", [7, 17])
def test_prove_batch_with_limit_members_matches_oracle_engine(sess, count):
    dev, ref, desc = limit_batch(sess, count, 0x70 + count)
    max_n = max(d[2] for d in desc)
    max_deg = max(r.degree for r in ref)
    assert max_deg == 7
    claimed = sum(c * k * pow(2, max_n - n, P) for c, k, n in desc) % P
    want = O.prove_batch([dict(input_claim=c, coefficient=k, rounds=n, offset=max_n - n) for c, k, n in desc], ref, max_n,
                         max_deg, claimed, challenge_fn)
    got = jolt_b200.prove_batch_native([BatchMember(c, k, n, max_n - n) for c, k, n in desc], dev, max_n, max_deg, claimed,
                                       absorb_round=lambda r, poly: challenge_fn(r, poly.coefficients))
    assert got.challenges == want["challenges"]
    assert got.final_claim == want["final_claim"]
    assert got.member_claims == want["member_claims"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for d, r in zip(dev, ref):
        assert d.final_evals() == r.final_evals()


def test_scheduler_with_limit_members_matches_oracle(sess):
    dev, ref, desc = limit_batch(sess, 14, 0xA0)
    assert sum(1 for d in dev if d.degree() == 7) == 8   # degree 7: the 8-evaluation row of out_evals, full
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


# ---- refusals one past each limit ---------------------------------------------------------------------------------
def raw_monomials(monomials):
    """(coeff, tables[, degree]) -> the C array; `degree` may exceed the tables given (one past JB_EXPR_MAX_DEGREE)"""
    mons = (_lib.MonomialC * max(len(monomials), 1))()
    for k, (coeff, tabs, *deg) in enumerate(monomials):
        mons[k].coeff[:] = [int(x) for x in F.to_limbs(coeff % P)]
        mons[k].degree = deg[0] if deg else len(tabs)
        for i, t in enumerate(tabs[:_lib.JB_EXPR_MAX_DEGREE]):
            mons[k].table[i] = t
    return mons


def create_expr(sess, T, monomials, n=3):
    handles = np.array([Polynomial.new(sess, S.rand_limbs_full(0xEF0 + j, 1 << n)).handle for j in range(T)], dtype=np.uint64)
    h = ctypes.c_void_p()
    st = sess.lib.jb_member_create_expr(sess.h, handles.ctypes.data_as(_lib.c_u64p), T,
                                        ctypes.cast(raw_monomials(monomials), ctypes.c_void_p), len(monomials), None, 0,
                                        None, LOW_TO_HIGH, ctypes.byref(h))
    if st == _lib.JB_OK:
        sess.lib.jb_member_destroy(h)
    return st


def create_sources(sess, count, monomials, n=3):
    cols = [SR.address_column(n, 4, 0xEF0 + j) for j in range(count)]
    r = F.ints_to_limbs(O.random_fr(0xEF9, 2))
    arr = (_lib.SourceC * count)()
    for i, a in enumerate(cols):
        arr[i].type, arr[i].kind, arr[i].on_device = _lib.JB_SOURCE_ONE_HOT, 1, 0
        arr[i].values = a.ctypes.data
        arr[i].K = 4
        arr[i].r_addr = r.ctypes.data_as(_lib.c_u64p)
    h = ctypes.c_void_p()
    st = sess.lib.jb_member_create_expr_sources(sess.h, ctypes.cast(arr, ctypes.c_void_p), count, 1 << n,
                                                ctypes.cast(raw_monomials(monomials), ctypes.c_void_p), len(monomials),
                                                None, 0, None, LOW_TO_HIGH, ctypes.byref(h))
    if st == _lib.JB_OK:
        sess.lib.jb_member_destroy(h)
    return st


def test_refusals_one_past_each_limit(sess):
    """(9 expression tables, 17 expression monomials, expression degree 7 and 9 sources are refused in
    tests/test_gpu_expr.py and tests/test_gpu_expr_sources.py)"""
    INV, UNS, OK = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED, _lib.JB_OK
    at_limit = [(k + 2, tabs) for k, (_, tabs) in enumerate(MAX_MONOMIALS)]
    assert create_expr(sess, 8, at_limit) == OK
    assert create_sources(sess, 8, at_limit) == OK
    assert create_expr(sess, 8, at_limit[:-1] + [(2, [8])]) == INV                      # table index 8 of 8 tables
    assert create_expr(sess, 8, at_limit[:-1] + [(2, [0, 1, 2, 3, 4, 8])]) == INV        # index 8 as the 6th factor
    assert create_sources(sess, 8, at_limit[:-1] + [(2, [8])]) == INV                   # source index 8 of 8 sources
    assert create_sources(sess, 8, at_limit + [(2, [1])]) == UNS                        # 17 monomials over sources
    assert create_sources(sess, 8, at_limit[:-1] + [(2, [0] * 6, 7)]) == UNS            # degree 7 over sources
    assert create_expr(sess, 8, at_limit[:-1] + [(2, [0] * 6, 7)]) == UNS               # degree 7 at the table limit
    # the context still proves at the limits
    n, order = 3, HIGH_TO_LOW
    tabs, w = expr_inputs("max_eq_scaled", n, order)
    _, mons, _, scale = SHAPES["max_eq_scaled"]
    gpu = ExpressionMember(sess, [Polynomial.new(sess, t) for t in tabs], mons, w, scale, order=order)
    drive_lockstep(gpu, expr_transcript("max_eq_scaled", n, order), mons, n, n)
    gpu.close()
    dev, _, w = source_inputs(sess, "mixed8", n)
    mons = source_monomials(8)
    gpu = ExpressionMember.from_sources(sess, dev, mons, w, order=order)
    drive_lockstep(gpu, source_transcript("mixed8", n, order), mons, n, n)
    gpu.close()
