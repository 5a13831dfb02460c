"""Product members over sources on the device (jb_member_create_product_sources): every round polynomial and the final
evaluations in lockstep with tests/source_ref.py for 1 .. 16 factors of mixed source types; bit-identity with the
expression member over sources, the product member and the split-eq member where the shapes overlap; d = 16 and d = 9
one-hot products at 2^22 against the evaluation entry points; the batch engine and the scheduler; every error."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (BatchMember, EqPolynomial, EqProductMember, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, ProductMember,
                       RoundScheduler, Source, UnivariatePoly, _lib, one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
from gpu_util import rand_challenge
import expr_ref as E
import source_ref as SR
import sumcheck_ref as S
from test_gpu_expr_sources import address_column, compact_column, _challenge

pytestmark = pytest.mark.gpu
P = O.R_MOD
KINDS = ["u8", "u16", "u32", "u64", "i64", "u128", "i128", "s64", "s128"]
ONE_HOT = [(1, np.uint8), (2, np.uint8), (16, np.uint8), (256, np.uint8), (16, np.uint16), (1 << 16, np.uint16)]


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


def mixed_sources(d, n, seed):
    """d factors cycling through field tables, every compact kind and one-hot u8 / u16 columns (K = 1 .. 2^16, with
    none values); returns (device sources, table limbs to upload per factor or None, reference sources)"""
    dev, ref = [], []
    for i in range(d):
        kind = (i + seed) % 3
        if kind == 0:
            t = S.rand_limbs_full(seed + 7 * i, 1 << n)
            dev.append(("table", t))
            ref.append(("table", F.limbs_to_ints(t)))
        elif kind == 1:
            k = KINDS[(i + seed) % len(KINDS)]
            a, ra = compact_column(k, n, seed + 7 * i)
            dev.append(Source.compact(a, k))
            ref.append(("compact", ra))
        else:
            K, dt = ONE_HOT[(i + seed) % len(ONE_HOT)]
            a = address_column(n, K, seed + 7 * i, dtype=dt)
            r = O.random_fr(seed + 7 * i + 1, K.bit_length() - 1)
            dev.append(Source.one_hot(a, K, r))
            ref.append(("one_hot", SR.addresses(a), K, r))
    return dev, ref


def device_sources(sess, dev):
    return [Source.table(Polynomial.new(sess, s[1])) if isinstance(s, tuple) else s for s in dev]


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("eq", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("d", [1, 2, 3, 5, 7, 8, 9, 12, 16])
def test_product_lockstep_vs_reference(sess, sess_verify, d, n, order, eq, verify):
    _lockstep(sess_verify if verify else sess, d, n, order, eq)


@pytest.mark.parametrize("eq", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("d,n", [(3, 12), (9, 10), (16, 10)])
def test_product_lockstep_multi_block(sess, d, n, order, eq):
    """sizes whose first rounds run many 64-thread blocks and the last block's fold of their partials"""
    _lockstep(sess, d, n, order, eq)


def _lockstep(s, d, n, order, eq):
    seed = 0x9100 + 32 * d + n
    dev, refsrc = mixed_sources(d, n, seed)
    w = S.extreme_point(0x41 + n, n, zero=False) if eq else None
    mons = [(1, list(range(d)))]
    ref = SR.SourcesMember(refsrc, mons, order, None if w is None else F.limbs_to_ints(w))
    gpu = ProductMember.from_sources(s, device_sources(s, dev), w, order=order)
    assert gpu.num_rounds() == n and gpu.degree() == ref.degree == d + (1 if eq else 0)
    claim = ref.claim()
    bind = None
    for rnd in range(n):
        want = ref.round_evals(None if bind is None else F.from_limbs(bind))
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = _challenge(rnd, n + d)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    ref.finish_rounds(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    fin = gpu.final_evals()
    assert fin == ref.final_evals()
    want_claim = 1
    for v in fin:
        want_claim = want_claim * v % P
    if eq:
        assert gpu.eq_scalar() == ref.eq_scalar()
        want_claim = want_claim * ref.eq_scalar() % P
    assert want_claim == claim
    gpu.close()


@pytest.mark.parametrize("d", [2, 9, 16])
def test_product_without_claim_computes_every_point(sess, d):
    n = 4
    dev, refsrc = mixed_sources(d, n, 0x9900 + d)
    ref = SR.SourcesMember(refsrc, [(1, list(range(d)))], HIGH_TO_LOW)
    gpu = ProductMember.from_sources(sess, device_sources(sess, dev))
    bind = None
    for rnd in range(n):
        assert gpu.prove_round_evals(bind, rnd, None) == ref.round_evals(None if bind is None else F.from_limbs(bind))
        bind = rand_challenge(0x9A00 + rnd)


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_product_from_cuda_tensors(sess, order):
    """compact and one-hot columns handed over as CUDA tensors give the member of the same columns from host arrays"""
    import torch
    n, seed = 11, 0x9C00
    u8 = address_column(n, 256, seed, dtype=np.uint8)
    u16 = address_column(n, 1 << 16, seed + 1, dtype=np.uint16)
    c8, _ = compact_column("u8", n, seed + 2)
    i64, _ = compact_column("i64", n, seed + 3)
    r8, r16 = O.random_fr(seed + 4, 8), O.random_fr(seed + 5, 16)
    t = S.rand_limbs_full(seed + 6, 1 << n)
    w = S.extreme_point(0x5A, n, zero=False)

    def srcs(dev):
        col = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if dev else (lambda a: a)
        return [Source.one_hot(col(u8), 256, r8), Source.one_hot(col(u16), 1 << 16, r16), Source.compact(col(c8)),
                Source.compact(col(i64)), Source.table(Polynomial.new(sess, t))]
    a = ProductMember.from_sources(sess, srcs(True), w, order=order)
    b = ProductMember.from_sources(sess, srcs(False), w, order=order)
    _drive_pair(a, b, n, _claim(sess, srcs(False), w), 0x9D00)


# ---- device against device ------------------------------------------------------------------------------------------
def _drive_pair(a, b, n, claim, seed):
    bind = None
    for rnd in range(n):
        ea = a.prove_round_evals(bind, rnd, claim)
        eb = b.prove_round_evals(bind, rnd, claim)
        assert ea == eb, f"round {rnd}"
        bind = rand_challenge(seed + rnd) if rnd % 3 else S.extreme_challenge(rnd, seed)
        claim = UnivariatePoly.from_evals(ea).evaluate(F.from_limbs(bind))
    a.finish_rounds(bind)
    b.finish_rounds(bind)
    assert a.final_evals() == b.final_evals()


@pytest.mark.parametrize("n", [16, 20])
@pytest.mark.parametrize("eq", [False, True])
@pytest.mark.parametrize("d", [1, 2, 3, 4, 5, 6])
def test_product_matches_expression_member(sess, d, eq, n):
    seed = 0xA100 + d + n
    w = S.extreme_point(0x51 + n, n, zero=False) if eq else None
    a = ProductMember.from_sources(sess, device_sources(sess, mixed_sources(d, n, seed)[0]), w, order=LOW_TO_HIGH)
    b = ExpressionMember.from_sources(sess, device_sources(sess, mixed_sources(d, n, seed)[0]), [(1, list(range(d)))], w,
                                      order=LOW_TO_HIGH)
    _drive_pair(a, b, n, _claim(sess, mixed_sources(d, n, seed)[0], w), seed)


def _claim(sess, dev, w):
    """sum_x [eq(w, x) *] prod_i f_i(x) from round 0 of a product member without eq (eq as one more table source)"""
    srcs = device_sources(sess, dev) + ([] if w is None else [Source.table(EqPolynomial.evals(sess, w))])
    c = ProductMember.from_sources(sess, srcs)
    ev = c.prove_round_evals(None, 0, None)
    c.close()
    return (ev[0] + ev[1]) % P


@pytest.mark.parametrize("eq", [False, True])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_product_matches_table_members(sess, d, eq):
    n = 18
    if eq and d > 3:
        pytest.skip("the split-eq member takes 1..3 tables")
    tabs = [S.rand_limbs_full(0xB100 + 5 * j, 1 << n) for j in range(d)]
    w = S.extreme_point(0x61, n, zero=False) if eq else None
    polys = [Polynomial.new(sess, t) for t in tabs]
    b = EqProductMember(sess, polys, w, order=HIGH_TO_LOW) if eq else ProductMember(sess, polys, HIGH_TO_LOW)
    # the initial claim from the plain product member (over the materialised eq table with eq)
    pre = [EqPolynomial.evals(sess, w)] if eq else []
    c = ProductMember(sess, pre + [Polynomial.new(sess, t) for t in tabs], HIGH_TO_LOW)
    ev = c.prove_round_evals(None, 0, None)
    c.close()
    a = ProductMember.from_sources(sess, [Source.table(Polynomial.new(sess, t)) for t in tabs], w, order=HIGH_TO_LOW)
    _drive_pair(a, b, n, (ev[0] + ev[1]) % P, 0xB200 + d)


# ---- at scale -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["d16_u8_K256", "d9_u16_K65536_table"])
def test_product_at_scale(sess_verify, shape):
    """every round in verify mode from the round-0 sums; final claim = eq scalar x prod of the final evaluations, and each
    one-hot final evaluation equals jb_one_hot_evaluate at the challenge point"""
    s = sess_verify
    n = 22
    rng = np.random.default_rng(0xC100)
    if shape.startswith("d16"):
        cols = [rng.integers(0, 256, 1 << n).astype(np.uint8) for _ in range(16)]
        K, tab = 256, None
    else:
        cols = [rng.integers(0, 1 << 16, 1 << n).astype(np.uint16) for _ in range(8)]
        K, tab = 1 << 16, S.rand_limbs_full(0xC200, 1 << n)
    for c in cols:
        c[rng.random(1 << n) < 0.05] = np.iinfo(c.dtype).max
    r_addrs = [O.random_fr(0xC300 + i, K.bit_length() - 1) for i in range(len(cols))]
    srcs = [Source.one_hot(c, K, r) for c, r in zip(cols, r_addrs)]
    if tab is not None:
        srcs.append(Source.table(Polynomial.new(s, tab)))
    # d = 16 without eq (round 0 without a claim gives the initial claim), d = 9 with eq (claim through the eq table)
    w = S.extreme_point(0x71, n, zero=False) if tab is not None else None
    claim = None if w is None else _claim(s, srcs, w)
    srcs = [Source.one_hot(c, K, r) for c, r in zip(cols, r_addrs)]
    if tab is not None:
        srcs.append(Source.table(Polynomial.new(s, tab)))
    m = ProductMember.from_sources(s, srcs, w, order=LOW_TO_HIGH)
    bind, rs = None, []
    for rnd in range(n):
        ev = m.prove_round_evals(bind, rnd, claim)   # verify mode: s(0) + s(1) == claim is checked on the device side
        bind = rand_challenge(0xC400 + rnd)
        rs.append(F.from_limbs(bind))
        claim = UnivariatePoly.from_evals(ev).evaluate(rs[-1])
    m.finish_rounds(bind)
    fin = m.final_evals()
    prod = 1 if w is None else m.eq_scalar()
    for v in fin:
        prod = prod * v % P
    assert prod == claim
    point = list(reversed(rs))  # LowToHigh binds the least significant index bit first
    for i, (c, r) in enumerate(zip(cols, r_addrs)):
        assert fin[i] == one_hot_evaluate(s, c, K, point + list(r))[0], i


# ---- batches ----------------------------------------------------------------------------------------------------------
def _members(sess, degs, seed, eq_every=2, existing=0):
    """product members over mixed sources (every eq_every-th with eq) and their references; then `existing` members of
    the existing kinds (a product of 2 tables, a split-eq product of 2 tables) with theirs"""
    dev, ref, desc = [], [], []
    for k in range(existing):
        n = 4 + k % 2
        tabs = [O.random_fr(seed * 3 + 10 * k + j, 1 << n) for j in range(2)]
        polys = [Polynomial.from_ints(sess, t) for t in tabs]
        if k % 2:
            w = O.random_fr(seed * 3 + 10 * k + 9, n)
            dev.append(EqProductMember(sess, polys, F.ints_to_limbs(w), order=LOW_TO_HIGH))
            ref.append(E.ExpressionMember(tabs, [(1, [0, 1])], LOW_TO_HIGH, w))
        else:
            dev.append(ProductMember(sess, polys, LOW_TO_HIGH))
            ref.append(E.ExpressionMember(tabs, [(1, [0, 1])], LOW_TO_HIGH))
        desc.append((ref[-1].claim(), (k * 5 + 1) % P, n))
    for k, d in enumerate(degs):
        n = 3 + k % 3
        src, refsrc = mixed_sources(d, n, seed + 11 * k)
        w = O.random_fr(seed + 100 * k, n) if k % eq_every == 1 else None
        wl = None if w is None else F.ints_to_limbs(w)
        dev.append(ProductMember.from_sources(sess, device_sources(sess, src), wl, order=LOW_TO_HIGH))
        ref.append(SR.SourcesMember(refsrc, [(1, list(range(d)))], LOW_TO_HIGH, w))
        desc.append((ref[-1].claim(), (k * 7 + 3) % P, n))
    return dev, ref, desc


def _challenge_fn(rnd, coeffs):
    return (sum(int(c) for c in coeffs) * 7 + 31 * rnd + 5) % P


@pytest.mark.parametrize("existing", [0, 2])
@pytest.mark.parametrize("degs", [[16, 2, 9, 3], [7, 3, 5], [12, 16]])
def test_product_prove_batch_matches_oracle_engine(sess, degs, existing):
    """jb_prove_batch with product members up to degree 17, alone and mixed with existing members (the device scheduler
    serves batches it can, member order the rest), and the Python prove_batch twin, against the oracle's sequential
    engine"""
    dev, ref, desc = _members(sess, degs, 0xE100, existing=existing)
    max_n = max(d[2] for d in desc)
    max_deg = max(r.degree for r in ref)
    claimed = sum(c * k * pow(2, max_n - n, P) for c, k, n in desc) % P
    want = O.prove_batch([dict(input_claim=c, coefficient=k, rounds=n, offset=max_n - n) for c, k, n in desc], ref, max_n,
                         max_deg, claimed, _challenge_fn)
    got = jolt_b200.prove_batch_native([BatchMember(c, k, n, max_n - n) for c, k, n in desc], dev, max_n, max_deg, claimed,
                                       absorb_round=lambda r, poly: _challenge_fn(r, poly.coefficients))
    assert got.challenges == want["challenges"]
    assert got.final_claim == want["final_claim"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for d, r in zip(dev, ref):
        assert d.final_evals() == r.final_evals()
    twin, _, _ = _members(sess, degs, 0xE100, existing=existing)
    py = jolt_b200.prove_batch([BatchMember(c, k, n, max_n - n) for c, k, n in desc], twin, max_n, max_deg, claimed,
                               lambda r, poly: _challenge_fn(r, poly.coefficients))
    assert py.challenges == want["challenges"]
    assert py.final_claim == want["final_claim"]


@pytest.mark.parametrize("degs", [[7, 2, 5], [1, 6, 3, 4]])
def test_product_scheduler_matches_oracle(sess, degs):
    dev, ref, desc = _members(sess, degs, 0xD100, existing=2)
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


@pytest.mark.parametrize("degs", [[8], [2, 16], [7, 3]])
def test_product_scheduler_refuses_degree_8(sess, degs):
    dev, _, _ = _members(sess, degs, 0xD300, eq_every=2)
    if max(m.degree() for m in dev) < 8:
        RoundScheduler(sess, dev).close()
        return
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        RoundScheduler(sess, dev)
    assert e.value.status == _lib.JB_ERR_UNSUPPORTED


# ---- errors -----------------------------------------------------------------------------------------------------------
def _call(sess, srcs, length, w=None, nvars=0, scale=None, order=HIGH_TO_LOW):
    import ctypes
    arr = (_lib.SourceC * max(len(srcs), 1))()
    keep = []
    for i, s in enumerate(srcs):
        s._fill(arr[i], keep)
    h = ctypes.c_void_p()
    return sess.lib.jb_member_create_product_sources(sess.h, ctypes.cast(arr, ctypes.c_void_p), len(srcs), length,
                                                     w, nvars, scale, order, ctypes.byref(h)), h


def test_product_errors(sess):
    import ctypes
    n = 4
    a = address_column(n, 16, 1)
    ok = Source.one_hot(a, 16, O.random_fr(2, 4))
    st, _ = _call(sess, [], 1 << n)
    assert st == _lib.JB_ERR_INVALID
    st, _ = _call(sess, [ok] * 17, 1 << n)
    assert st == _lib.JB_ERR_UNSUPPORTED
    st, _ = _call(sess, [ok], 1 << n, order=7)
    assert st == _lib.JB_ERR_INVALID
    st, _ = _call(sess, [ok], 3)
    assert st == _lib.JB_ERR_INVALID
    bad = a.copy()
    bad[3] = 17  # an address >= K that is not the none value: found on the device
    st, _ = _call(sess, [ok, Source.one_hot(bad, 16, O.random_fr(2, 4))], 1 << n)
    assert st == _lib.JB_ERR_INVALID
    big = Source.one_hot(a.astype(np.uint16), 1 << 16, O.random_fr(3, 16))
    big.K = 1 << 17
    st, _ = _call(sess, [big], 1 << n)
    assert st == _lib.JB_ERR_INVALID
    w = np.zeros((n + 1, 4), dtype=np.uint64)
    st, _ = _call(sess, [ok], 1 << n, w=w.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), nvars=n + 1)
    assert st == _lib.JB_ERR_INVALID
    sc = np.full(4, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    st, _ = _call(sess, [ok], 1 << n, scale=sc.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)))
    assert st == _lib.JB_ERR_INVALID
    # the context stays usable, and a table source is still the caller's after a failed creation
    t = Polynomial.new(sess, S.rand_limbs_full(5, 1 << n))
    st, _ = _call(sess, [Source.table(t), Source.one_hot(bad, 16, O.random_fr(2, 4))], 1 << n)
    assert st == _lib.JB_ERR_INVALID
    assert len(t.to_ints()) == 1 << n
    m = ProductMember.from_sources(sess, [Source.table(t), ok])
    assert m.degree() == 2
    m.close()
    gpu = ProductMember.from_sources(sess, [ok])
    import ctypes as C
    lanes = np.zeros(64, dtype=np.uint64)
    assert sess.lib.jb_member_prove_round_partials(gpu.h, None, 0, 0, C.c_void_p(lanes.ctypes.data)) == \
        _lib.JB_ERR_UNSUPPORTED
    gpu.close()
    m = ProductMember.from_sources(sess, [ok], S.extreme_point(1, n, zero=False))
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        m.prove_round_evals(None, 0, None)   # the running claim is mandatory with eq
    assert e.value.status == _lib.JB_ERR_INVALID
    m.close()
