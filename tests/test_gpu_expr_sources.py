"""Expression members over sources on the device (jb_member_create_expr_sources): every round polynomial and the final
evaluations in lockstep with tests/source_ref.py; bit-identity with jb_member_create_expr over promoted and gathered
tables at 2^16 .. 2^22; RA virtualization and read checking against the evaluation entry points at 2^22 and 2^24;
skewed address columns; the batch engine and the scheduler with a sources member in the batch; every error."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (BatchMember, EqPolynomial, EqProductMember, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial,
                       ProductMember, RoundScheduler, Source, UnivariatePoly, _lib, evaluate_small, one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
from gpu_util import rand_challenge, rand_limbs
import expr_ref as E
import source_ref as SR
import sumcheck_ref as S

pytestmark = pytest.mark.gpu
from source_ref import MAGS, address_column, compact_column

P = O.R_MOD
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF


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


# ---- columns (compact_column and address_column are in source_ref) -------------------------------------------------
def r_limbs(vals):
    return F.ints_to_limbs(list(vals)) if len(vals) else np.zeros((0, 4), dtype=np.uint64)


def _challenge(rnd, seed):
    ch = S.extreme_challenge(rnd, seed)   # 125-bit and full challenges, interleaved with the extreme ones
    return ch if ch.any() else S.EXTREME_CHALLENGES[2]


# name -> builder(n, seed) -> (device sources, reference sources, monomials, eq)
def _compact_shape(kind):
    def build(n, seed):
        a, ra = compact_column(kind, n, seed)
        b, rb = compact_column(kind, n, seed + 1)
        t = S.rand_limbs_full(seed + 2, 1 << n)
        return ([Source.compact(a, kind), Source.compact(b, kind), ("table", t)],
                [("compact", ra), ("compact", rb), ("table", F.limbs_to_ints(t))],
                [(1, [0, 1]), (-1, [2]), (GAMMA, [0, 0, 2])], n % 2 == 1)
    return build


def _one_hot_shape(K, dtype):
    def build(n, seed):
        a = address_column(n, K, seed, dtype=dtype)
        r = O.random_fr(seed + 3, K.bit_length() - 1)
        t = S.rand_limbs_full(seed + 4, 1 << n)
        return ([Source.one_hot(a, K, r), ("table", t)],
                [("one_hot", SR.addresses(a), K, r), ("table", F.limbs_to_ints(t))],
                [(1, [0, 1]), (1, [0, 0]), (-1, [0])], True)
    return build


def _read_checking(n, seed):
    """eq * (ra val + g wa val + g^2 wa inc): ra, wa one-hot (u8, K = 16), val a field table, inc an i64 column"""
    ra, wa = address_column(n, 16, seed), address_column(n, 16, seed + 1, none_frac=0.0)
    r1, r2 = O.random_fr(seed + 2, 4), O.random_fr(seed + 3, 4)
    val = S.rand_limbs_full(seed + 4, 1 << n)
    inc, rinc = compact_column("i64", n, seed + 5)
    return ([Source.one_hot(ra, 16, r1), Source.one_hot(wa, 16, r2), ("table", val), Source.compact(inc)],
            [("one_hot", SR.addresses(ra), 16, r1), ("one_hot", SR.addresses(wa), 16, r2), ("table", F.limbs_to_ints(val)),
             ("compact", rinc)],
            [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA % P, [1, 3])], True)


SHAPES = {f"compact_{k}": _compact_shape(k) for k in MAGS}
SHAPES.update({f"one_hot_u8_K{K}": _one_hot_shape(K, np.uint8) for K in (1, 2, 16, 128)})
SHAPES.update({"one_hot_u16_K16": _one_hot_shape(16, np.uint16), "one_hot_u16_K65536": _one_hot_shape(1 << 16, np.uint16)})
SHAPES["read_checking"] = _read_checking


def _device_sources(sess, dev):
    return [Source.table(Polynomial.new(sess, s[1])) if isinstance(s, tuple) else s for s in dev]


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 9])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_sources_lockstep_vs_reference(sess, sess_verify, shape, n, order, verify):
    s = sess_verify if verify else sess
    dev, refsrc, mons, eq = SHAPES[shape](n, 0x5300 + 16 * n)
    w = S.extreme_point(0x3E + n, n, zero=False) if eq else None
    ref = SR.SourcesMember(refsrc, mons, order, None if w is None else F.limbs_to_ints(w))
    gpu = ExpressionMember.from_sources(s, _device_sources(s, dev), mons, w, order=order)
    assert gpu.num_rounds() == n and gpu.degree() == ref.degree
    claim = ref.claim()
    bind = None
    for rnd in range(n):
        want = ref.round_evals(None if bind is None else F.from_limbs(bind))
        got = gpu.prove_round_evals(bind, rnd, claim)
        assert got == want, f"round {rnd}"
        bind = _challenge(rnd, n)
        claim = UnivariatePoly.from_evals(got).evaluate(F.from_limbs(bind))
    ref.finish_rounds(F.from_limbs(bind))
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == ref.final_evals()
    fin = E.expr_value(ref.final_evals(), mons)
    if eq:
        assert gpu.eq_scalar() == ref.eq_scalar()
        fin = fin * ref.eq_scalar() % P
    assert fin == claim
    gpu.close()


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_sources_without_claim_computes_every_point(sess, order):
    n = 6
    dev, refsrc, mons, _ = SHAPES["compact_i128"](n, 0x7100)
    ref = SR.SourcesMember(refsrc, mons, order)
    gpu = ExpressionMember.from_sources(sess, _device_sources(sess, dev), mons, order=order)
    bind = None
    for rnd in range(n):
        assert gpu.prove_round_evals(bind, rnd, None) == ref.round_evals(None if bind is None else F.from_limbs(bind))
        bind = rand_challenge(0x7200 + rnd)


# ---- device against device --------------------------------------------------------------------------------------
def _gathered_limbs(addr: np.ndarray, K: int, r_addr) -> np.ndarray:
    """ra(r_addr, j) as field limbs, gathered on the host: eq(r_addr, .) indexed by the column, 0 for none"""
    eq = np.concatenate([F.ints_to_limbs(O.eq_evals(list(r_addr)) if len(r_addr) else [1]), np.zeros((1, 4), np.uint64)])
    idx = addr.astype(np.int64)
    idx[idx >= K] = K     # the none value
    return np.ascontiguousarray(eq[idx])


def _drive_pair(a, b, n, claim, seed):
    """both members through every round with the same challenges; every round polynomial identical. Returns the final
    claim and the challenges in round order."""
    bind, bound = None, []
    for rnd in range(n):
        ea = a.prove_round_evals(bind, rnd, claim)
        eb = b.prove_round_evals(bind, rnd, claim)
        assert ea == eb, f"round {rnd}"
        bind = rand_challenge(seed + rnd) if rnd % 3 else S.extreme_challenge(rnd, seed)
        bound.append(F.from_limbs(bind))
        claim = UnivariatePoly.from_evals(ea).evaluate(bound[-1])
    a.finish_rounds(bind)
    b.finish_rounds(bind)
    assert a.final_evals() == b.final_evals()
    return claim, bound


def _read_checking_pair(sess, n, order, seed, ra, wa):
    K = 16
    r1, r2 = O.random_fr(seed + 2, 4), O.random_fr(seed + 3, 4)
    val = rand_limbs(seed + 4, 1 << n)
    inc = np.random.default_rng(seed + 5).integers(-(1 << 63), (1 << 63) - 1, 1 << n, dtype=np.int64)
    mons = [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA % P, [1, 3])]
    w = np.stack([F.to_limbs(v) for v in O.random_fr(seed + 6, n)])
    a = ExpressionMember.from_sources(sess, [Source.one_hot(ra, K, r1), Source.one_hot(wa, K, r2),
                                             Source.table(Polynomial.new(sess, val)), Source.compact(inc)], mons, w, order=order)

    def tables():
        return [Polynomial.new(sess, _gathered_limbs(ra, K, r1)), Polynomial.new(sess, _gathered_limbs(wa, K, r2)),
                Polynomial.new(sess, val), Polynomial.from_small(sess, inc)]
    b = ExpressionMember(sess, tables(), mons, w, order=order)
    # the starting claim: s(0) + s(1) of the first round with eq(w, .) as one more table (computed, not derived)
    c = ExpressionMember(sess, [EqPolynomial.evals(sess, w)] + tables(), [(k, [0] + [t + 1 for t in tabs]) for k, tabs in mons],
                         order=order)
    e0 = c.prove_round_evals(None, 0, None)
    c.close()
    return a, b, mons, (r1, r2, inc), (e0[0] + e0[1]) % P


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("n", [16, 20, 22])
def test_sources_bit_identical_to_promoted_and_gathered_tables(sess, n, order):
    seed = 0x8800 + n
    ra, wa = address_column(n, 16, seed), address_column(n, 16, seed + 1, none_frac=0.0)
    a, b, mons, (r1, r2, inc), claim = _read_checking_pair(sess, n, order, seed, ra, wa)
    fin_claim, bound = _drive_pair(a, b, n, claim, seed)
    fin = a.final_evals()
    assert fin_claim == a.eq_scalar() * E.expr_value(fin, mons) % P
    # the final evaluations are the columns' values at the challenge point (cycle order)
    r = bound if order == HIGH_TO_LOW else list(reversed(bound))
    assert fin[0] == one_hot_evaluate(sess, ra, 16, r + list(r1))[0]
    assert fin[1] == one_hot_evaluate(sess, wa, 16, r + list(r2))[0]
    assert fin[3] == evaluate_small(sess, inc, r)[0]
    a.close()
    b.close()


@pytest.mark.parametrize("n", [16])
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("kind", ["u8", "u64", "i128", "s64"])
def test_compact_bit_identical_to_upload_small(sess, kind, order, n):
    """eq * (a b - c) over compact columns against the same member over jb_table_upload_small tables"""
    cols = [compact_column(kind, n, 0x8900 + j)[0] for j in range(3)]
    mons = [(1, [0, 1]), (-1, [2])]
    w = np.stack([F.to_limbs(v) for v in O.random_fr(0x8950, n)])
    named = kind if kind in ("u128", "i128", "s64", "s128") else None
    a = ExpressionMember.from_sources(sess, [Source.compact(c, named) for c in cols], mons, w, order=order)
    b = ExpressionMember(sess, [Polynomial.from_small(sess, c, named) for c in cols], mons, w, order=order)
    tabs = [F.limbs_to_ints(Polynomial.from_small(sess, c, named).evals()) for c in cols]
    claim = E.ExpressionMember(tabs, mons, order, F.limbs_to_ints(w)).claim()
    _drive_pair(a, b, n, claim, 0x8960)


# ---- RA virtualization against the evaluation entry points ----------------------------------------------------------
def _ra_chunks(n, K, d, seed, none_frac=0.1):
    """d address chunks of one virtual address (chunk 0 the most significant); a cycle is none in every chunk or none"""
    rng = np.random.default_rng(seed)
    T = 1 << n
    none = rng.random(T) < none_frac
    chunks = []
    for i in range(d):
        hi = K - 1 if K == 256 else (K - 1 if i else K - 2)   # u8: addresses < 255; K^d <= 2^16: the all-ones address is none
        c = rng.integers(0, hi, T, dtype=np.int64).astype(np.uint8)
        c[none] = 0xFF
        chunks.append(c)
    return chunks


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("d,K", [(1, 16), (2, 16), (4, 16), (1, 256), (2, 256), (4, 256)])
@pytest.mark.parametrize("n", [22, 24])
def test_ra_virtualization_matches_one_hot_evaluate(sess, n, d, K, order):
    """sum_j eq(r_cycle, j) prod_i ra_i(r_addr_i, j) with eq(r_cycle, .) as a table source and d one-hot sources"""
    seed = 0x9100 + 16 * n + d + K
    chunks = _ra_chunks(n, K, d, seed)
    lk = K.bit_length() - 1
    r_cycle = O.random_fr(seed + 1, n)
    r_addr = [O.random_fr(seed + 2 + i, lk) for i in range(d)]
    eq_tab = EqPolynomial.evals(sess, r_limbs(r_cycle))
    gpu = ExpressionMember.from_sources(sess, [Source.table(eq_tab)] + [Source.one_hot(c, K, r) for c, r in zip(chunks, r_addr)],
                                        [(1, list(range(d + 1)))], order=order)
    e0 = gpu.prove_round_evals(None, 0, None)
    claim = (e0[0] + e0[1]) % P
    if K ** d <= 1 << 16:
        virt = np.zeros(1 << n, dtype=np.int64)
        for c in chunks:
            virt = virt * K + c.astype(np.int64)
        virt = virt.astype(np.uint16)
        virt[chunks[0] == 0xFF] = 0xFFFF
        point = list(r_cycle) + [x for r in r_addr for x in r]
        assert claim == one_hot_evaluate(sess, virt, K ** d, point)[0]
    bound = []
    bind = None
    for rnd in range(n):
        ev = e0 if rnd == 0 else gpu.prove_round_evals(bind, rnd, claim)
        bind = rand_challenge(seed + 0x40 + rnd)
        bound.append(F.from_limbs(bind))
        claim = UnivariatePoly.from_evals(ev).evaluate(bound[-1])
    gpu.finish_rounds(bind)
    r = bound if order == HIGH_TO_LOW else list(reversed(bound))
    fin = gpu.final_evals()
    want_eq = 1
    for a_, b_ in zip(r_cycle, r):
        want_eq = want_eq * (a_ * b_ + (1 - a_) * (1 - b_)) % P
    assert fin[0] == want_eq
    for i in range(d):
        assert fin[1 + i] == one_hot_evaluate(sess, chunks[i], K, r + list(r_addr[i]))[0], f"chunk {i}"
    prod = 1
    for v in fin:
        prod = prod * v % P
    assert claim == prod
    gpu.close()


# ---- skew -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
@pytest.mark.parametrize("case", ["one_address", "all_none"])
def test_skewed_columns(sess, case, order):
    n = 16
    ra = np.full(1 << n, 5 if case == "one_address" else 0xFF, dtype=np.uint8)
    wa = np.full(1 << n, 9 if case == "one_address" else 0xFF, dtype=np.uint8)
    a, b, _, _, claim = _read_checking_pair(sess, n, order, 0x9900, ra, wa)
    _drive_pair(a, b, n, claim, 0x9910)
    if case == "all_none":
        assert a.final_evals()[:2] == [0, 0]


# ---- the batch engine and the scheduler ---------------------------------------------------------------------------
def _mixed_batch(sess, count, seed):
    """ragged members: sources (compact + one-hot + table, with eq), product, eq and expression members"""
    rng = np.random.Generator(np.random.PCG64(seed))
    dev, ref, desc = [], [], []
    for i in range(count):
        n = int(rng.integers(3, 8))
        kind = i % 4
        if kind == 0:
            a = address_column(n, 8, seed + i)
            c, rc = compact_column("i64", n, seed + i + 1)
            t = O.random_fr(seed * 100 + 10 * i, 1 << n)
            r = O.random_fr(seed * 100 + 10 * i + 1, 3)
            w = O.random_fr(seed * 100 + 10 * i + 9, n)
            mons = [(1, [0, 1]), (GAMMA, [2, 0]), (-1, [2])]
            rm = SR.SourcesMember([("one_hot", SR.addresses(a), 8, r), ("compact", rc), ("table", t)], mons, LOW_TO_HIGH, w)
            d = ExpressionMember.from_sources(sess, [Source.one_hot(a, 8, r), Source.compact(c),
                                                     Source.table(Polynomial.from_ints(sess, t))], mons, r_limbs(w),
                                              order=LOW_TO_HIGH)
        else:
            T, mons, eq = [(2, [(1, [0, 1])], False), (2, [(1, [0, 1])], True), (2, [(5, [0, 0, 1]), (1, [1])], False)][kind - 1]
            tabs = [O.random_fr(seed * 100 + 10 * i + j, 1 << n) for j in range(T)]
            w = O.random_fr(seed * 100 + 10 * i + 9, n) if eq else None
            rm = E.ExpressionMember(tabs, mons, LOW_TO_HIGH, w)
            polys = [Polynomial.from_ints(sess, t) for t in tabs]
            if kind == 1:
                d = ProductMember(sess, polys, LOW_TO_HIGH)
            elif kind == 2:
                d = EqProductMember(sess, polys, r_limbs(w), order=LOW_TO_HIGH)
            else:
                d = ExpressionMember(sess, polys, mons, order=LOW_TO_HIGH)
        dev.append(d)
        ref.append(rm)
        desc.append((rm.claim(), (i * 7 + 3) % P, n))
    return dev, ref, desc


def _challenge_fn(rnd, coeffs):
    return (sum(int(c) for c in coeffs) * 7 + 31 * rnd + 5) % P


@pytest.mark.parametrize("count", [4, 9])
def test_prove_batch_with_sources_matches_oracle_engine(sess, count):
    dev, ref, desc = _mixed_batch(sess, count, 0x60 + count)
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


def test_scheduler_with_sources_matches_oracle(sess):
    dev, ref, desc = _mixed_batch(sess, 9, 0x90)
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


# ---- errors -------------------------------------------------------------------------------------------------------
def _create(sess, srcs, monomials, length, w=None, order=LOW_TO_HIGH):
    arr = (_lib.SourceC * max(len(srcs), 1))()
    keep = []
    for i, s in enumerate(srcs):
        arr[i].type, arr[i].kind, arr[i].on_device = s.get("type", 1), s.get("kind", 1), s.get("on_device", 0)
        arr[i].table = s.get("table", 0)
        v = s.get("values")
        if isinstance(v, int):      # a raw (device) address
            arr[i].values = v
        elif v is not None:
            keep.append(v)
            arr[i].values = v.ctypes.data
        arr[i].K = s.get("K", 0)
        r = s.get("r_addr")
        if r is not None:
            keep.append(r)
            arr[i].r_addr = r.ctypes.data_as(_lib.c_u64p)
    mons = (_lib.MonomialC * max(len(monomials), 1))()
    for k, (coeff, tabs) in enumerate(monomials):
        mons[k].coeff[:] = [int(x) for x in F.to_limbs(coeff)]
        mons[k].degree = len(tabs)
        for j, t in enumerate(tabs):
            mons[k].table[j] = t
    h = ctypes.c_void_p()
    wp = None if w is None else np.ascontiguousarray(w, dtype=np.uint64)
    st = sess.lib.jb_member_create_expr_sources(sess.h, ctypes.cast(arr, ctypes.c_void_p), len(srcs), length,
                                                ctypes.cast(mons, ctypes.c_void_p), len(monomials),
                                                None if wp is None else wp.ctypes.data_as(_lib.c_u64p),
                                                0 if wp is None else wp.shape[0], None, order, ctypes.byref(h))
    if st == _lib.JB_OK:
        sess.lib.jb_member_destroy(h)
    return st


def test_errors_and_context_stays_usable(sess):
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    u8 = np.arange(16, dtype=np.uint8) % 4
    ok_r = r_limbs(O.random_fr(1, 2))
    bad_r = ok_r.copy()
    bad_r[1] = S.int_to_limbs(P)
    compact = dict(type=1, kind=1, values=u8)
    one_hot = dict(type=2, kind=1, values=u8, K=4, r_addr=ok_r)
    m1 = [(1, [0])]
    assert _create(sess, [compact], m1, 16) == _lib.JB_OK
    assert _create(sess, [one_hot], m1, 16) == _lib.JB_OK
    assert _create(sess, [dict(compact, type=3)], m1, 16) == INV                 # an unknown source type
    assert _create(sess, [dict(compact, kind=0)], m1, 16) == INV                 # JB_SCALAR_FR is not compact
    assert _create(sess, [dict(compact, kind=10)], m1, 16) == INV                # an unknown kind
    assert _create(sess, [dict(one_hot, kind=3)], m1, 16) == INV                 # one-hot addresses are u8 / u16
    assert _create(sess, [dict(one_hot, K=3)], m1, 16) == INV                    # K not a power of two
    assert _create(sess, [dict(one_hot, K=0)], m1, 16) == INV                    # K out of range
    assert _create(sess, [dict(one_hot, K=1 << 17, r_addr=r_limbs(O.random_fr(2, 17)))], m1, 16) == INV
    assert _create(sess, [dict(one_hot, r_addr=bad_r)], m1, 16) == INV           # r_addr not canonical
    assert _create(sess, [dict(one_hot, r_addr=None)], m1, 16) == INV            # a null r_addr
    assert _create(sess, [dict(compact, values=None)], m1, 16) == INV            # a null column
    assert _create(sess, [dict(compact, on_device=2)], m1, 16) == INV            # on_device not 0 / 1
    import torch
    dev = torch.zeros(64, dtype=torch.int64, device="cuda")
    assert _create(sess, [dict(compact, kind=4, values=dev.data_ptr() + 4, on_device=1)], m1, 16) == INV  # misaligned
    assert _create(sess, [dict(one_hot, kind=2, values=dev.data_ptr() + 1, on_device=1)], m1, 16) == INV  # misaligned
    assert _create(sess, [one_hot], m1, 1 << 31) == UNS                          # a one-hot column of 2^31 cycles
    assert _create(sess, [compact], m1, 12) == INV                               # len not a power of two
    assert _create(sess, [compact], m1, 1) == INV                                # len < 2
    p = Polynomial.new(sess, rand_limbs(3, 32))
    assert _create(sess, [dict(type=0, table=p.handle), compact], [(1, [0, 1])], 16) == INV   # a table of another length
    assert _create(sess, [dict(type=0, table=0xDEAD)], m1, 16) == INV            # an unknown table handle
    q = Polynomial.new(sess, rand_limbs(4, 16))
    assert _create(sess, [dict(type=0, table=q.handle)] * 2, [(1, [0, 1])], 16) == INV       # duplicate handles
    assert _create(sess, [compact], [(1, [0, 1])], 16) == INV                    # a table index out of range
    assert _create(sess, [compact, compact], m1, 16) == INV                      # a source no monomial uses
    assert _create(sess, [compact], m1, 16, w=r_limbs(O.random_fr(5, 3))) == INV  # nvars != log2(len)
    assert _create(sess, [compact], m1, 16, order=7) == INV                      # an unknown order
    assert _create(sess, [compact] * 9, [(1, list(range(6))), (1, [6, 7, 8])], 16) == UNS   # more than 8 sources
    # an address >= K that is not none: found on the device, nothing kept, the caller's table still usable
    bad_addr = u8.copy()
    bad_addr[7] = 4
    l0 = q.evals()
    assert _create(sess, [dict(type=0, table=q.handle), dict(one_hot, values=bad_addr)], [(1, [0, 1])], 16) == INV
    assert (q.evals() == l0).all() and len(q) == 16
    # the context still proves
    test_sources_without_claim_computes_every_point(sess, LOW_TO_HIGH)


def test_unbound_source_is_not_exported_and_partials_refused(sess):
    a = np.arange(16, dtype=np.uint8)
    torch = pytest.importorskip("torch")
    gpu = ExpressionMember.from_sources(sess, [Source.compact(a), Source.compact(a + 1)], [(1, [0, 1]), (3, [0])])
    lanes = torch.zeros(64, dtype=torch.int64, device="cuda")
    st = sess.lib.jb_member_prove_round_partials(gpu.h, None, 0, 0, ctypes.c_void_p(lanes.data_ptr()))
    assert st == _lib.JB_ERR_UNSUPPORTED
    out = ctypes.c_size_t()
    st = sess.lib.jb_member_export_table(gpu.h, 0, ctypes.c_void_p(lanes.data_ptr()), 8, ctypes.byref(out))
    assert st == _lib.JB_ERR_INVALID   # a compact source is a column until its bind
    gpu.close()


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW])
def test_device_columns_from_torch(sess, order):
    torch = pytest.importorskip("torch")
    n = 12
    a = address_column(n, 64, 0xA0)
    inc = np.random.default_rng(0xA1).integers(-(1 << 40), 1 << 40, 1 << n, dtype=np.int64)
    r = O.random_fr(0xA2, 6)
    mons = [(1, [0, 1]), (7, [1])]
    da = torch.from_numpy(a).cuda()
    di = torch.from_numpy(inc).cuda()
    g_host = ExpressionMember.from_sources(sess, [Source.one_hot(a, 64, r), Source.compact(inc)], mons, order=order)
    g_dev = ExpressionMember.from_sources(sess, [Source.one_hot(da, 64, r), Source.compact(di)], mons, order=order)
    torch.cuda.synchronize()
    ref = SR.SourcesMember([("one_hot", SR.addresses(a), 64, r), ("compact", [int(v) for v in inc])], mons, order)
    _drive_pair(g_host, g_dev, n, ref.claim(), 0xA3)
