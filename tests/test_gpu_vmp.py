"""Dory's vector-matrix product on the device (jb_lc_vector_matrix_product, Polynomial.vector_matrix_product), all
bit-exact: against tests/vmp_ref.py at small sizes for every row width; against the materialise-and-bind route
(jb_table_linear_combination bound HighToLow by the row coordinates) at scale; beyond what can be materialised, against
the combined evaluation claim; Dory's commitment identity against the row commitments; consistency; and every error
of the contract, after which the context keeps working."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (EqPolynomial, G1Bases, LinearTerm, Polynomial, _lib, evaluate_small, g1_jacobian_to_affine,
                       one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
import lincomb_ref as LR
import vmp_ref as V
from gpu_util import EDGE_INTS, rand_limbs
from test_gpu_lincomb import G, MAX125, NP_KIND, Terms, _scale_terms, _term, addresses, mixed

pytestmark = pytest.mark.gpu
R = O.R_MOD


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def arbitrary_left(sess, rows, seed):
    """Not an eq table: random values with the limb extremes of EDGE_INTS mixed in."""
    vals = O.random_fr(seed, rows)
    rng = np.random.default_rng(seed)
    for i in range(rows):
        if rng.random() < 0.5:
            vals[i] = EDGE_INTS[int(rng.integers(0, len(EDGE_INTS)))]
    return Polynomial.from_ints(sess, vals), vals


def vmp(sess, t, left, W, length=None):
    return Polynomial.vector_matrix_product(sess, t.dev, left, W, length=length)


# ---- 1. small sizes against the reference ----------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 3, 6, 10])
def test_matches_reference_for_every_row_width(sess, n):
    t = mixed(sess, n, 500 + n)
    for lw in range(n + 1):
        W = 1 << lw
        left, lv = arbitrary_left(sess, (1 << n) >> lw, 600 + n + lw)
        before = left.evals().copy()
        assert vmp(sess, t, left, W).to_ints() == V.vector_matrix_product(t.ref, 1 << n, W, lv), W
        assert np.array_equal(left.evals(), before)
    t.check_inputs()
    # a longer length: every term is a prefix
    W = max((2 << n) // 4, 1)
    left, lv = arbitrary_left(sess, (2 << n) // W, 700 + n)
    assert vmp(sess, t, left, W, length=2 << n).to_ints() == V.vector_matrix_product(t.ref, 2 << n, W, lv)


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
@pytest.mark.parametrize("dtype,K,lt", [(np.uint8, 1, 6), (np.uint8, 2, 6), (np.uint8, 16, 5), (np.uint8, 256, 3),
                                        (np.uint16, 1, 6), (np.uint16, 16, 5), (np.uint16, 256, 3),
                                        (np.uint16, 1 << 16, 2)])
@pytest.mark.parametrize("none_frac", [0.0, 0.3, 1.0])
def test_one_hot_every_shape(sess, dtype, K, lt, layout, none_frac):
    """W < K, W = K, W > K, W <= T and W > T, up to W = len (R = 1), with the coefficients 0, 1, p - 1 and 125 bits"""
    t = Terms(sess, 3 * K + lt)
    t.one_hot(dtype, K, lt, layout, none_frac)
    t.one_hot(dtype, K, lt, layout, none_frac)
    t.dev[0] = LinearTerm.one_hot(t.cref[0][1], K, MAX125, layout)
    t.ref[0] = t.ref[0][:-1] + (MAX125,)
    n = (K << lt).bit_length() - 1
    lk = K.bit_length() - 1
    widths = range(n + 1) if n <= 12 else sorted({0, 1, lt, lt + 1, lk - 1, lk, lk + 1, n - 1, n})
    for lw in widths:
        W = 1 << lw
        left, lv = arbitrary_left(sess, (K << lt) >> lw, K + lw)
        assert vmp(sess, t, left, W).to_ints() == V.vector_matrix_product(t.ref, K << lt, W, lv), W
    # with a prefix: the term covers part of row 0 only
    left, lv = arbitrary_left(sess, 2, 99)
    assert vmp(sess, t, left, K << lt, length=2 * K << lt).to_ints() == V.vector_matrix_product(t.ref, 2 * K << lt,
                                                                                                K << lt, lv)


# ---- 2. the materialise-and-bind route at scale ----------------------------------------------------------------------
def _bind_route(sess, terms, length, r_row):
    P = Polynomial.linear_combination(sess, terms, length=length)
    Q = P.clone()
    P.free()
    for r in r_row:
        Q.bind(r)
    return Q


def _check_against_route(sess, terms, n, lw, seed):
    r_row = O.random_fr(seed, n - lw)
    L = EqPolynomial.evals(sess, F.ints_to_limbs(r_row))
    v = Polynomial.vector_matrix_product(sess, terms, L, 1 << lw, length=1 << n)
    Q = _bind_route(sess, terms, 1 << n, r_row)
    assert np.array_equal(v.evals(), Q.evals())
    for p in (v, Q, L):
        p.free()


@pytest.mark.parametrize("n,count", [(22, 16), (24, 8)])
def test_at_scale_against_the_bind_route(sess, n, count):
    t = _scale_terms(sess, n, count, 800 + n)
    for lw in ((n + 1) // 2, 5):
        _check_against_route(sess, t.dev, n, lw, 810 + lw)
    t.check_inputs()


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
def test_one_hot_2_26_against_the_bind_route(sess, layout):
    t = Terms(sess, 900, big=True)
    t.one_hot(np.uint8, 256, 18, layout)
    for lw in (13, 20):
        _check_against_route(sess, t.dev, 26, lw, 901 + lw)


# ---- 3. beyond what can be materialised ------------------------------------------------------------------------------
def test_jolt_shape_2_32_against_the_combined_claim(sess):
    """one-hot K = 256 terms over T = 2^24 cycles in both layouts (2^32 coefficients, W = R = 2^16), compact u64 and
    i128 columns and a field table as prefixes: <v, eq(r_col)> = sum_i c_i prefix factor e_i"""
    import torch
    n, lt, K = 32, 24, 256
    rng = np.random.default_rng(1000)
    cs = [O.random_fr(1001, 1)[0], MAX125, R - 1, O.random_fr(1002, 1)[0], 1]
    cm = addresses(rng, 1 << lt, K, np.uint8, 0.3)
    am = addresses(rng, 1 << lt, K, np.uint8, 0.1)
    u64 = rng.integers(0, 1 << 64, 1 << lt, dtype=np.uint64)
    i128 = torch.from_numpy(rng.integers(0, 1 << 64, size=(1 << (lt - 1), 2), dtype=np.uint64).view(np.int64).copy()).cuda()
    tab = Polynomial.new(sess, rand_limbs(1003, 1 << lt))
    terms = [LinearTerm.one_hot(cm, K, cs[0], "cycle_major"), LinearTerm.one_hot(am, K, cs[1], "address_major"),
             LinearTerm.compact(u64, cs[2]), LinearTerm.compact(i128, cs[3], kind="i128"), LinearTerm.table(tab, cs[4])]
    for seed in (1010, 1020):
        point = O.random_fr(seed, n)
        L = EqPolynomial.evals(sess, F.ints_to_limbs(point[:16]))
        v = Polynomial.vector_matrix_product(sess, terms, L, 1 << 16)
        claims = [(cs[0], n, one_hot_evaluate(sess, cm, K, point, "cycle_major")[0]),
                  (cs[1], n, one_hot_evaluate(sess, am, K, point, "address_major")[0]),
                  (cs[2], lt, evaluate_small(sess, u64, point[n - lt:])[0]),
                  (cs[3], lt - 1, evaluate_small(sess, i128, point[n - lt + 1:], kinds="i128")[0]),
                  (cs[4], lt, tab.evaluate(point[n - lt:]))]
        assert v.evaluate(point[16:]) == LR.combined_claim(claims, point)
        v.free()
        L.free()


# ---- 4. Dory's commitment identity -----------------------------------------------------------------------------------
def _row_commitments(bases, claim, W):
    """The tier-1 row commitments of one term (rows of W; a term shorter than W is one row of its own length)."""
    kind, what, _c = claim
    if kind == "table":
        limbs = what.evals()
        return bases.msm_rows(limbs, max(limbs.shape[0] // W, 1), kind="fr")
    if kind == "compact":
        vals, k = what
        return bases.msm_rows(vals, max(len(vals) // W, 1), kind=None if k in NP_KIND else k)
    col, K, layout = what
    return bases.one_hot_rows(col, K, min(W, K * col.shape[0]), layout)[0]


@pytest.mark.parametrize("n,lw", [(12, 6), (14, 9), (16, 8)])
def test_commitment_identity(sess, n, lw):
    W = 1 << lw
    bases = G1Bases.generate_multiples(sess, G, W)
    t = mixed(sess, n, 1100 + n)
    left, lv = arbitrary_left(sess, (1 << n) >> lw, 1200 + n)
    v = Polynomial.vector_matrix_product(sess, t.dev, left, W)
    rows, scalars = [], []
    for claim in t.claims:
        for r, C in enumerate(_row_commitments(bases, claim, W)):
            if np.any(C[8:]):   # skip identity rows (Z = 0)
                rows.append(C)
                scalars.append(claim[2] * lv[r] % R)
    want = G1Bases.from_jacobian(sess, np.array(rows)).msm(F.ints_to_limbs(scalars))
    assert g1_jacobian_to_affine(bases.msm(v)) == g1_jacobian_to_affine(want)


# ---- 5. consistency --------------------------------------------------------------------------------------------------
def test_host_and_device_columns_repeated_calls_and_inputs(sess):
    n, W = 12, 1 << 5
    host, dev = mixed(sess, n, 7), mixed(sess, n, 7, device=True)
    left, _ = arbitrary_left(sess, (1 << n) // W, 8)
    before = left.evals().copy()
    a = vmp(sess, host, left, W).evals()
    b = vmp(sess, dev, left, W).evals()
    c = vmp(sess, dev, left, W).evals()
    assert np.array_equal(a, b) and np.array_equal(b, c)
    assert np.array_equal(left.evals(), before)
    host.check_inputs()
    dev.check_inputs()


# ---- 6. errors -------------------------------------------------------------------------------------------------------
def _raw(sess, terms, count=None, length=4, W=1, left=0):
    arr = (_lib.LcTermC * max(len(terms), 1))()
    for i, t in enumerate(terms):
        arr[i] = t
    out = ctypes.c_uint64(0)
    st = sess.lib.jb_lc_vector_matrix_product(sess.h, ctypes.cast(arr, ctypes.c_void_p),
                                              len(terms) if count is None else count, length, W, left, ctypes.byref(out))
    return st, out.value


def test_errors_leave_the_context_usable(sess):
    u8 = np.array([1, 2, 3, 4], dtype=np.uint8)
    u16 = np.array([0, 1, 0xFFFF, 3], dtype=np.uint16)
    poly = Polynomial.from_ints(sess, [5, 6, 7, 8])
    odd_h = ctypes.c_uint64()
    sess.check(sess.lib.jb_table_alloc(sess.h, 3, ctypes.byref(odd_h)))
    odd = Polynomial(sess, odd_h.value)
    lefts = {n: Polynomial.from_ints(sess, list(range(3, 3 + n))) for n in (1, 2, 4, 8, 16)}
    before = poly.evals().copy()
    vp = u8.ctypes.data
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    import torch
    dev16 = torch.zeros(8, dtype=torch.int16, device="cuda")
    OH = _lib.JB_LC_ONE_HOT
    # (terms, count, length, row width, left rows or a raw handle, status): W = 1 unless stated, left of len / W rows
    cases = [
        ([], 0, 4, 1, 4, INV),                                                                  # count == 0
        ([_term(type=7, values=vp)], None, 4, 1, 4, INV),                                      # unknown type
        ([_term(kind=0, values=vp)], None, 4, 1, 4, INV),                                      # FR is not compact
        ([_term(kind=10, values=vp)], None, 4, 1, 4, INV),                                     # unknown kind
        ([_term(values=vp)], None, 3, 1, 4, INV),                                              # len not a power of two
        ([_term(values=vp)], None, 2, 1, 2, INV),                                              # term longer than len
        ([_term(values=vp, len=3)], None, 4, 1, 4, INV),                                       # term length
        ([_term(values=None)], None, 4, 1, 4, INV),                                            # null column
        ([_term(values=vp, on_device=2)], None, 4, 1, 4, INV),                                 # on_device
        ([_term(values=vp, coeff=[int(x) for x in F.to_limbs(0)][:3] + [0xFFFFFFFFFFFFFFFF])], None, 4, 1, 4, INV),
        ([_term(type=_lib.JB_LC_TABLE, table=123456789)], None, 4, 1, 4, INV),                 # unknown handle
        ([_term(type=_lib.JB_LC_TABLE, table=odd.handle)], None, 4, 1, 4, INV),                # table length
        ([_term(kind=4, values=dev16.data_ptr() + 2, on_device=1)], None, 4, 1, 4, INV),       # misaligned column
        ([_term(type=OH, kind=4, values=vp)], None, 4, 1, 4, INV),                             # one-hot kind
        ([_term(type=OH, layout=2, values=vp)], None, 4, 1, 4, INV),                           # layout
        ([_term(type=OH, K=3, values=vp)], None, 16, 1, 16, INV),                              # K
        ([_term(type=OH, K=4, values=vp)], None, 8, 1, 8, INV),                                # K T > len
        ([_term(type=OH, kind=2, K=2, values=dev16.data_ptr() + 1, on_device=1)], None, 8, 1, 8, INV),
        ([_term(type=OH, kind=2, K=1 << 17, values=u16.ctypes.data)], None, 1 << 20, 1 << 16, 16, UNS),
        ([_term(type=OH, kind=2, K=1, len=1 << 31, values=u16.ctypes.data)], None, 1 << 31, 1 << 27, 16, UNS),
        # addresses >= K found on the device, in the scatter (cycle-major) and both gathers (address-major)
        ([_term(type=OH, K=2, values=vp)], None, 8, 1, 8, INV),
        ([_term(type=OH, K=2, values=vp)], None, 8, 4, 2, INV),
        ([_term(type=OH, K=2, layout=1, values=vp)], None, 8, 2, 4, INV),
        ([_term(type=OH, K=2, layout=1, values=vp)], None, 8, 8, 1, INV),
        ([_term(type=OH, kind=2, K=2, values=u16.ctypes.data)], None, 8, 2, 4, INV),
        # the row width and the left table
        ([_term(values=vp)], None, 4, 3, 1, INV),                                              # W not a power of two
        ([_term(values=vp)], None, 4, 0, 1, INV),                                              # W = 0
        ([_term(values=vp)], None, 4, 8, 1, INV),                                              # W > len
        ([_term(values=vp)], None, 4, 1, ("raw", 987654321), INV),                             # unknown left
        ([_term(values=vp)], None, 4, 1, 2, INV),                                              # left too short
        ([_term(values=vp)], None, 4, 2, 4, INV),                                              # left too long
        # the lane bound: count R < 2^32 (refused before the terms or left are read)
        ([_term(values=vp)], None, 1 << 32, 1, ("raw", 0), UNS),
        ([_term(values=vp)] * 4, None, 1 << 32, 4, ("raw", 0), UNS),
        ([_term(values=vp)] * 2, 1 << 31, 4, 2, ("raw", 0), UNS),
    ]
    good = [_term(type=_lib.JB_LC_TABLE, table=poly.handle, coeff=F.to_limbs(2)), _term(values=vp)]
    P = [(2 * a + 3 * b) % R for a, b in zip([5, 6, 7, 8], [1, 2, 3, 4])]
    last = None
    for i, (terms, count, length, W, left, want) in enumerate(cases):
        lh = left[1] if isinstance(left, tuple) else lefts[left].handle
        st, h = _raw(sess, terms, count, length, W, lh)
        assert st == want, (i, st, sess.lib.jb_last_error(sess.h))
        assert h == 0, i
        st, h = _raw(sess, good, None, 4, 2, lefts[2].handle)
        assert st == _lib.JB_OK, i
        if last is not None:
            assert h == last + 1, i   # the failed call created no table
        last = h
        assert Polynomial(sess, h).to_ints() == [(3 * P[0] + 4 * P[2]) % R, (3 * P[1] + 4 * P[3]) % R]
        Polynomial(sess, h).free()
    assert sess.lib.jb_lc_vector_matrix_product(sess.h, None, 1, 4, 1, lefts[4].handle,
                                                ctypes.byref(ctypes.c_uint64())) == INV
    assert np.array_equal(poly.evals(), before)
    with pytest.raises(ValueError):
        Polynomial.vector_matrix_product(sess, [], lefts[1], 1)
