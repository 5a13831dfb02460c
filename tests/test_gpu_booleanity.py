"""Booleanity member on the device (jb_member_create_booleanity), bit-exact against booleanity_ref: every round in
lockstep in both orders (with and without verify mode), the dense twin (the expression member over the materialised
ra tables), final values against one-hot evaluation, linearity at Jolt sizes, jb_prove_batch end to end, edge values,
host against device columns, and every refusal."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, BooleanityMember, ExpressionMember, JoltB200Error,
                       Polynomial, ProductMember, _lib, one_hot_evaluate)
from jolt_b200 import field as F
from jolt_b200.api import SCALAR_KINDS
from oracle import bn254 as O
import booleanity_ref as B

P = O.R_MOD
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def _hi4(seed, n):
    """125-bit challenges: Montgomery limbs [0, 0, lo, hi] (the device's HI4 bind path)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        lo, hi = int(rng.integers(0, 1 << 63)) * 2 + 1, int(rng.integers(0, 1 << 61))
        out.append(F.from_limbs(np.array([0, 0, lo, hi], dtype=np.uint64)))
    return out


def _drive(m, ch, claim=0):
    """Every round of a member at the challenges ch; returns (rounds, final claim)."""
    rounds, bind = [], None
    for rnd in range(len(ch)):
        got = m.prove_round_evals(bind, rnd, claim)
        assert (got[0] + got[1]) % P == claim, rnd
        rounds.append(got)
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    return rounds, claim


def _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order, verify=False, kind=None, cols=None):
    want_rounds, want_final = B.sparse_prove(K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order)
    cols = B.column_arrays(addrs, K, kind) if cols is None else cols
    m = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, scale, order)
    assert m.num_rounds() == len(ch) and m.degree() == 3
    sess.set_verify_rounds(verify)
    try:
        rounds, claim = _drive(m, ch)
        assert rounds == want_rounds
        fin = m.final_evals()
        assert fin == want_final
        e = m.eq_scalar()
        assert e == B.eq_scalar(K, T, r_addr, r_cycle, scale, ch, order)
        assert claim == B.final_claim(fin, coeffs, e)
        return rounds, fin
    finally:
        sess.set_verify_rounds(False)
        m.close()


def _inputs(seed, K, T, d):
    lk, lt = K.bit_length() - 1, T.bit_length() - 1
    return (O.random_fr(seed, d), O.random_fr(seed + 1, lk), O.random_fr(seed + 2, lt), O.random_fr(seed + 3, 1)[0],
            O.random_fr(seed + 4, lk + lt))


@pytest.mark.parametrize("K,T,d", [(1, 2, 1), (1, 1024, 9), (2, 4, 2), (2, 1024, 1), (16, 2, 9), (16, 1024, 9),
                                   (16, 4, 32), (256, 2, 32), (256, 1024, 32), (256, 4, 2), (8, 1, 3)])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("verify", [False, True])
def test_lockstep_with_reference(sess, K, T, d, order, verify):
    addrs = B.random_columns(K * 131 + T + d, K, T, d)
    coeffs, r_addr, r_cycle, scale, ch = _inputs(K + 3 * T + d, K, T, d)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale if verify else None, ch, order, verify)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_lockstep_u16_full_address_range(sess, order):
    K, T, d = 1 << 16, 4, 2
    addrs = B.random_columns(5, K, T, d, none_frac=0.1)
    addrs[1][0] = K - 2  # (K - 1 is the u16 none value)
    coeffs, r_addr, r_cycle, scale, ch = _inputs(17, K, T, d)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_lockstep_u16_small_k(sess, order):
    K, T, d = 64, 64, 3
    addrs = B.random_columns(6, K, T, d)
    coeffs, r_addr, r_cycle, scale, ch = _inputs(18, K, T, d)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order, kind=np.uint16)


def _dense_twin(sess, cols, K, coeffs, r_addr, r_cycle, order):
    one = F.to_limbs(1)
    polys = [Polynomial.new(sess, B.dense_ra_limbs(c, K, order, one)) for c in cols]
    mons = [m for i, c in enumerate(coeffs) for m in ((c, [i, i]), ((P - c) % P, [i]))]
    pt = list(r_addr) + list(r_cycle) if order == HIGH_TO_LOW else list(r_cycle) + list(r_addr)
    return ExpressionMember(sess, polys, mons, w_limbs=F.ints_to_limbs(pt), order=order)


@pytest.mark.parametrize("K,T,d,dtype", [(16, 1 << 16, 8, np.uint8), (256, 1 << 12, 4, np.uint8),
                                         (4, 1 << 18, 8, np.uint8), (1024, 1 << 10, 3, np.uint16)])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_bit_identical_with_dense_twin(sess, K, T, d, dtype, order):
    cols = B.random_column_arrays(K + T + d, K, T, d, dtype)
    coeffs, r_addr, r_cycle, _scale, _ch = _inputs(K + d, K, T, d)
    ch = _hi4(K + T, (K * T).bit_length() - 1)
    ch[1] = O.random_fr(9, 1)[0]
    m = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, order=order)
    tw = _dense_twin(sess, cols, K, coeffs, r_addr, r_cycle, order)
    got, claim = _drive(m, ch)
    want, claim_tw = _drive(tw, ch)
    assert got == want
    fin = m.final_evals()
    assert fin == tw.final_evals()
    assert m.eq_scalar() == tw.eq_scalar()
    ra, rc = B.bound_point(K, T, ch, order)
    assert fin == one_hot_evaluate(sess, cols, K, ra + rc, layout="address_major")
    assert claim == claim_tw == B.final_claim(fin, coeffs, m.eq_scalar())
    m.close()
    tw.close()


def test_linearity_at_jolt_sizes(sess):
    K, T, d = 16, 1 << 20, 32
    cols = B.random_column_arrays(77, K, T, d, np.uint8)
    coeffs, r_addr, r_cycle, scale, _ = _inputs(78, K, T, d)
    n = (K * T).bit_length() - 1
    ch = _hi4(79, n)
    for order in (HIGH_TO_LOW, LOW_TO_HIGH):
        full = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, scale, order)
        a = BooleanityMember(sess, cols[:13], K, coeffs[:13], r_addr, r_cycle, scale, order)
        b = BooleanityMember(sess, cols[13:], K, coeffs[13:], r_addr, r_cycle, scale, order)
        claims = [0, 0, 0]
        bind = None
        for rnd in range(n):
            polys = [m.prove_round_evals(bind, rnd, c) for m, c in zip((full, a, b), claims)]
            assert polys[0] == [(x + y) % P for x, y in zip(polys[1], polys[2])], (order, rnd)
            bind = ch[rnd]
            claims = [O.uni_evaluate(O.uni_from_evals(p), bind) for p in polys]
        for m in (full, a, b):
            m.finish_rounds(bind)
        assert full.final_evals() == a.final_evals() + b.final_evals()
        for m in (full, a, b):
            m.close()


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_prove_batch_end_to_end(sess, order):
    K, T, d = 256, 1 << 20, 16
    cols = B.random_column_arrays(91, K, T, d, np.uint8)
    coeffs, r_addr, r_cycle, scale, _ = _inputs(92, K, T, d)
    n = (K * T).bit_length() - 1
    m = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, scale, order)
    tabs = [O.random_fr(93 + j, 1 << 10) for j in range(2)]
    pm = ProductMember(sess, [Polynomial.from_ints(sess, x) for x in tabs], LOW_TO_HIGH)
    c_pm = sum(x * y for x, y in zip(*tabs)) % P
    k_b, k_pm = 5, 7
    claimed = k_pm * c_pm * pow(2, n - 10, P) % P
    got = jolt_b200.prove_batch_native([BatchMember(0, k_b, n, 0), BatchMember(c_pm, k_pm, 10, n - 10)], [m, pm], n, 3,
                                       claimed, seed=order + 1)
    fin = m.final_evals()
    e = m.eq_scalar()
    assert got.member_claims[0] == B.final_claim(fin, coeffs, e)
    assert e == B.eq_scalar(K, T, r_addr, r_cycle, scale, got.challenges, order)
    ra, rc = B.bound_point(K, T, got.challenges, order)
    assert fin == one_hot_evaluate(sess, cols, K, ra + rc, layout="address_major")
    pf = pm.final_evals()
    assert got.final_claim == (k_b * got.member_claims[0] + k_pm * pf[0] * pf[1]) % P
    m.close()
    pm.close()


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("K,kind", [(128, np.uint8), (256, np.uint8), (1 << 15, np.uint16), (1 << 16, np.uint16)])
def test_edge_columns(sess, order, K, kind):
    T = 8
    top = K - 1 if K < np.iinfo(kind).max + 1 else K - 2  # the largest address that is not the none value
    addrs = [[None] * T, [top] * T, [top if j % 2 else 0 for j in range(T)]]
    coeffs, r_addr, r_cycle, scale, ch = _inputs(31 + K, K, T, 3)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order, kind=kind)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_edge_values(sess, order):
    K, T, d = 16, 64, 3
    addrs = B.random_columns(41, K, T, d)
    n = 10
    edges = [0, 1, P - 1]
    ch = [edges[i % 3] for i in range(n)]
    coeffs = [P - 1, 1, 0]
    # points r - 1 (eq(r - 1, c) != 0 at every edge challenge) and 125-bit
    r_addr = [P - 1, _hi4(42, 1)[0], P - 1, P - 1]
    r_cycle = [P - 1] * 3 + _hi4(43, 3)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, P - 1, ch, order)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, None, _hi4(44, n), order)
    _lockstep(sess, K, T, addrs, O.random_fr(45, d), [1] * 4, [1] * 6, 1, O.random_fr(46, n), order)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_host_and_device_columns_agree(sess, order):
    torch = pytest.importorskip("torch")
    K, T, d = 256, 1 << 12, 5
    cols = B.random_column_arrays(51, K, T, d, np.uint8)
    coeffs, r_addr, r_cycle, scale, ch = _inputs(52, K, T, d)
    results = []
    for c in (cols, [torch.from_numpy(x).cuda() for x in cols]):
        m = BooleanityMember(sess, c, K, coeffs, r_addr, r_cycle, scale, order)
        rounds, _ = _drive(m, ch)
        results.append((rounds, m.final_evals(), m.eq_scalar()))
        m.close()
    assert results[0] == results[1]
    cols16 = [x.astype(np.uint16) for x in cols]
    cols16 = [np.where(x == 0xFF, 0xFFFF, x).astype(np.uint16) for x in cols16]
    m = BooleanityMember(sess, [torch.from_numpy(x.view(np.int16)).cuda() for x in cols16], K, coeffs, r_addr, r_cycle,
                         scale, order)
    rounds, _ = _drive(m, ch)
    assert (rounds, m.final_evals(), m.eq_scalar()) == results[0]
    m.close()


def _create(sess, cols, count, kind, dev, T, K, coeffs, r_addr, r_cycle, scale=None, order=LOW_TO_HIGH):
    h = ctypes.c_void_p()
    arr = None if cols is None else (ctypes.c_void_p * max(len(cols), 1))(*cols)
    lim = lambda xs: None if xs is None else np.ascontiguousarray(F.ints_to_limbs(xs) if xs else np.zeros((1, 4), np.uint64))
    cf, ra, rc = lim(coeffs), lim(r_addr), lim(r_cycle)
    sc = None if scale is None else np.ascontiguousarray(scale, dtype=np.uint64)
    p = lambda a: None if a is None else a.ctypes.data_as(_lib.c_u64p)
    st = sess.lib.jb_member_create_booleanity(sess.h, arr, count, kind, dev, T, K, p(cf), p(ra), p(rc), p(sc), order,
                                              ctypes.byref(h))
    if st == _lib.JB_OK:
        sess.lib.jb_member_destroy(h)
    return st


def test_refusals(sess):
    T, K = 8, 4
    col = np.zeros(T, dtype=np.uint8)
    ptr = [col.ctypes.data]
    u8, u16 = SCALAR_KINDS["u8"], SCALAR_KINDS["u16"]
    good = dict(coeffs=[3], r_addr=[5, 6], r_cycle=[7, 8, 9])
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    assert _create(sess, ptr, 1, u8, 0, T, K, **good) == _lib.JB_OK
    assert _create(sess, None, 1, u8, 0, T, K, **good) == INV
    assert _create(sess, ptr, 1, u8, 0, T, K, None, [5, 6], [7, 8, 9]) == INV
    assert _create(sess, ptr, 1, u8, 0, T, K, [3], None, [7, 8, 9]) == INV
    assert _create(sess, ptr, 1, u8, 0, T, K, [3], [5, 6], None) == INV
    assert _create(sess, [0], 1, u8, 0, T, K, **good) == INV  # a null column
    assert _create(sess, ptr, 0, u8, 0, T, K, **good) == INV
    assert _create(sess, ptr, 1, SCALAR_KINDS["u32"], 0, T, K, **good) == INV
    assert _create(sess, ptr, 1, u8, 0, T, K, **good, order=7) == INV
    assert _create(sess, ptr, 1, u8, 0, 6, K, **good) == INV
    assert _create(sess, ptr, 1, u8, 0, T, 3, **good) == INV
    assert _create(sess, ptr, 1, u16, 0, T, 1 << 17, **good) == INV
    assert _create(sess, ptr, 1, u8, 0, 1, 1, [3], [], []) == INV  # K T = 1
    assert _create(sess, ptr, 1, u8, 2, T, K, **good) == INV
    big = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)
    for bad in (dict(coeffs=None), dict(r_addr=None), dict(r_cycle=None)):
        args = dict(good)
        key = next(iter(bad))
        lim = np.ascontiguousarray(F.ints_to_limbs(args[key]))
        lim[0] = big
        h = ctypes.c_void_p()
        arrs = {k: np.ascontiguousarray(F.ints_to_limbs(v)) for k, v in args.items()}
        arrs[key] = lim
        p = lambda a: a.ctypes.data_as(_lib.c_u64p)
        st = sess.lib.jb_member_create_booleanity(sess.h, (ctypes.c_void_p * 1)(*ptr), 1, u8, 0, T, K, p(arrs["coeffs"]),
                                                  p(arrs["r_addr"]), p(arrs["r_cycle"]), None, LOW_TO_HIGH,
                                                  ctypes.byref(h))
        assert st == INV, key
    assert _create(sess, ptr, 1, u8, 0, T, K, **good, scale=big) == INV
    many = [col.ctypes.data] * 33
    assert _create(sess, many, 33, u8, 0, T, K, coeffs=[3] * 33, r_addr=[5, 6], r_cycle=[7, 8, 9]) == UNS
    assert _create(sess, ptr, 1, u8, 0, 1 << 31, K, coeffs=[3], r_addr=[5, 6], r_cycle=[7] * 31) == UNS
    torch = pytest.importorskip("torch")
    buf = torch.zeros(2 * T + 2, dtype=torch.uint8, device="cuda")
    assert _create(sess, [buf.data_ptr() + 1], 1, u16, 1, T, K, **good) == INV  # misaligned device column
    # an address >= K that is not none, found on the device; the context stays usable
    bad = col.copy()
    bad[3] = K
    assert _create(sess, [bad.ctypes.data], 1, u8, 0, T, K, **good) == INV
    bad_dev = torch.from_numpy(bad).cuda()
    assert _create(sess, [bad_dev.data_ptr()], 1, u8, 1, T, K, **good) == INV
    addrs = B.random_columns(61, K, T, 2)
    coeffs, r_addr, r_cycle, scale, ch = _inputs(62, K, T, 2)
    _lockstep(sess, K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, LOW_TO_HIGH)


def test_round_refusals(sess):
    K, T = 4, 8
    cols = B.column_arrays(B.random_columns(71, K, T, 2), K)
    # a zero eq factor at the current variable (LowToHigh binds the address LSB, r_addr[1], first) is refused
    m = BooleanityMember(sess, cols, K, [3, 4], [5, 0], [6, 7, 8])
    with pytest.raises(JoltB200Error) as e:
        m.prove_round_evals(None, 0, 0)
    assert e.value.status == _lib.JB_ERR_INVALID
    m.close()
    m = BooleanityMember(sess, cols, K, [3, 4], [2, 5], [6, 7, 8])
    with pytest.raises(JoltB200Error) as e:
        m.prove_round_evals(None, 0, None)  # the running claim is mandatory
    assert e.value.status == _lib.JB_ERR_INVALID
    out = np.zeros(64, dtype=np.uint64)
    assert sess.lib.jb_member_prove_round_partials(m.h, None, 0, 1, ctypes.c_void_p(out.ctypes.data)) == _lib.JB_ERR_UNSUPPORTED
    n = ctypes.c_size_t()
    assert sess.lib.jb_member_num_tables(m.h, ctypes.byref(n)) == _lib.JB_OK and n.value == 2
    assert sess.lib.jb_member_export_table(m.h, 0, ctypes.c_void_p(out.ctypes.data), 64, None) == _lib.JB_ERR_INVALID
    with pytest.raises(JoltB200Error):
        m.final_evals()  # NotFullyBound
    m.close()
