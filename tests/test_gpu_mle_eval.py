"""Multilinear evaluation on the device (jb_table_evaluate_batch, jb_small_evaluate_batch, jb_one_hot_evaluate,
jb_one_hot_pushforward) compared bit-exactly with tests/mle_eval_ref.py, with bind sequences and with closed forms at
scale; every error condition of the contract, after which the context keeps working."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, ONE_HOT_NONE, Polynomial, _lib, evaluate_small, one_hot_evaluate,
                       one_hot_pushforward)
from jolt_b200 import field as F
from jolt_b200.api import _p
from oracle import bn254 as O
from oracle import coracle as C
import mle_eval_ref as ref
from gpu_util import EDGE_INTS

pytestmark = pytest.mark.gpu
R = O.R_MOD
MAX125 = (1 << 125) - 1


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def point(kind, n, seed):
    """Canonical point values: random, 125-bit challenges, or the cycle 0, 1, p - 1, 2^125 - 1."""
    if kind == "random":
        return O.random_fr(seed, n)
    if kind == "125":
        return [int(F.from_limbs(C.rand_challenge(seed + i))) for i in range(n)]
    return [[0, 1, R - 1, MAX125][(i + seed) % 4] for i in range(n)]


def challenge_point(n, seed):
    """(values, limbs) of a 125-bit point; limbs [0,0,lo,hi]."""
    limbs = np.stack([C.rand_challenge(seed + i) for i in range(n)]) if n else np.zeros((0, 4), dtype=np.uint64)
    return [F.from_limbs(l) for l in limbs], limbs


# ---- field tables --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 9, 12, 17])
@pytest.mark.parametrize("batch", [1, 3, 8])
def test_field_tables(sess, n, batch):
    tabs = [O.random_fr(1000 * n + 10 * batch + b, 1 << n) for b in range(batch)]
    polys = [Polynomial.from_ints(sess, t) for t in tabs]
    before = [p.evals().copy() for p in polys]
    for pk in ("random", "125", "cycle"):
        pt = point(pk, n, 7 * n + batch)
        got = Polynomial.batch_evaluate(polys, pt)
        assert got == [ref.evaluate(t, pt) for t in tabs], pk
    for p, b in zip(polys, before):
        assert np.array_equal(p.evals(), b) and len(p) == 1 << n       # not bound, swapped or reallocated
    assert polys[0].evaluate(pt) == got[0]


@pytest.mark.parametrize("n", [1, 4, 12])
def test_field_tables_of_edge_values(sess, n):
    rng = np.random.Generator(np.random.PCG64(n))
    vals = [EDGE_INTS[i] for i in rng.integers(0, len(EDGE_INTS), size=1 << n)]
    limbs = np.full((1 << n, 4), np.uint64((1 << 64) - 1))
    limbs[:, 3] = np.uint64(0x30644E72E131A029 - 1)                    # limb-extreme canonical representatives
    extreme = F.limbs_to_ints(limbs)
    for tab in (vals, extreme, [R - 1] * (1 << n)):
        p = Polynomial.new(sess, F.ints_to_limbs(tab))
        for pk in ("random", "cycle"):
            pt = point(pk, n, 3)
            assert p.evaluate(pt) == ref.evaluate(tab, pt)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_a_bound_table_evaluates_at_its_remaining_variables(sess, order):
    n, k = 10, 3
    tab = O.random_fr(77 + order, 1 << n)
    pt = O.random_fr(78 + order, n)
    p = Polynomial.from_ints(sess, tab)
    binds = pt[:k] if order == HIGH_TO_LOW else pt[::-1][:k]
    for r in binds:
        p.bind(r, order)
    rest = pt[k:] if order == HIGH_TO_LOW else pt[:n - k]
    assert p.evaluate(rest) == ref.evaluate(tab, pt)


def test_point_limbs_are_taken_as_given(sess):
    vals, limbs = challenge_point(6, 90)
    tab = O.random_fr(91, 64)
    p = Polynomial.from_ints(sess, tab)
    assert p.evaluate(limbs) == p.evaluate(vals) == ref.evaluate(tab, vals)


# ---- compact columns -----------------------------------------------------------------------------------------------
KINDS = ["u8", "u16", "u32", "u64", "u128", "i64", "i128", "s64", "s128"]
_NP = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i64": np.int64}


def small_column(kind, n, seed):
    """(column as evaluate_small takes it, reference values): random entries with the kind's extremes mixed in."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind in _NP:
        info = np.iinfo(_NP[kind])
        a = rng.integers(info.min, info.max, size=n, dtype=_NP[kind], endpoint=True)
        a[:4 if n >= 4 else n] = np.array([0, info.max, info.min, 1], dtype=_NP[kind])[:min(n, 4)]
        return a, [int(v) for v in a]
    if kind in ("u128", "i128"):
        lo, hi = (0, 1 << 128) if kind == "u128" else (-(1 << 127), 1 << 127)
        vals = [int(x) for x in rng.integers(0, 1 << 63, size=n)]
        vals = [(v * 0x9E3779B97F4A7C15 ** 2) % (hi - lo) + lo for v in vals]
        vals[:4] = [0, hi - 1, lo, -1 if kind == "i128" else 1][:min(n, 4)]
        return vals, vals
    bits = 64 if kind == "s64" else 128
    recs = [((int(m) << (bits - 62)) | int(m), bool(s)) for m, s in zip(rng.integers(0, 1 << 62, size=n),
                                                                        rng.integers(0, 2, size=n))]
    recs[:4] = [(0, False), ((1 << bits) - 1, False), ((1 << bits) - 1, True), (0, True)][:min(n, 4)]
    return recs, recs


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [0, 2, 5, 13])
def test_compact_columns_of_every_kind(sess, kind, n):
    col, vals = small_column(kind, 1 << n, 500 + n)
    for pk in ("random", "125", "cycle"):
        pt = point(pk, n, n)
        want = ref.evaluate_small(vals, pt)
        assert evaluate_small(sess, [col], pt, kinds=kind) == [want], pk
    # the same as promoting on the device and evaluating the field table
    assert Polynomial.from_small(sess, col, kind=kind).evaluate(pt) == want


def test_mixed_kinds_in_one_batch_host_and_device(sess):
    torch = pytest.importorskip("torch")
    n = 11
    cols, vals = zip(*[small_column(k, 1 << n, 900 + i) for i, k in enumerate(KINDS)])
    pt = point("random", n, 4)
    want = [ref.evaluate_small(v, pt) for v in vals]
    assert evaluate_small(sess, list(cols), pt, kinds=KINDS) == want
    raw = [jolt_b200.small_scalars(c, k)[0] for c, k in zip(cols, KINDS)]
    dev = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda() for a in raw]
    assert evaluate_small(sess, dev, pt, kinds=KINDS) == want
    # a native torch dtype names its kind
    u8 = torch.from_numpy(np.asarray(cols[0])).cuda()
    assert evaluate_small(sess, u8, pt) == [want[0]]


# ---- one-hot -------------------------------------------------------------------------------------------------------
def address_column(K, T, dtype, seed, none_frac=0.0, single=None):
    rng = np.random.Generator(np.random.PCG64(seed))
    none = ONE_HOT_NONE[np.dtype(dtype)]
    col = rng.integers(0, min(K, none), size=T).astype(dtype)
    if single is not None:
        col[:] = single
    col[rng.random(T) < none_frac] = none
    return col, [None if a == none else int(a) for a in col.tolist()]


@pytest.mark.parametrize("K,dtype", [(1, np.uint8), (2, np.uint8), (16, np.uint8), (256, np.uint8), (1 << 16, np.uint16),
                                     (16, np.uint16)])
@pytest.mark.parametrize("T", [1, 2, 16, 1024])
def test_one_hot_evaluation_and_pushforward(sess, K, dtype, T):
    lt, lk = T.bit_length() - 1, K.bit_length() - 1
    cases = [address_column(K, T, dtype, 10 * T + i, f) for i, f in enumerate((0.0, 0.3, 1.0))]
    cases.append(address_column(K, T, dtype, 5, single=K // 2))
    cols = [c for c, _ in cases]
    # the materialised polynomial where it is small; beyond, its definition (the two agree: test_mle_eval_cpu.py)
    want = ref.one_hot_evaluate if K * T <= 1 << 14 else ref.one_hot_evaluate_direct
    for layout in ("cycle_major", "address_major"):
        pt = point("random", lt + lk, K + T)
        got = one_hot_evaluate(sess, cols, K, pt, layout)
        assert got == [want(a, K, T, pt, layout) for _, a in cases], layout
    r_cycle = point("125", lt, T)
    G = one_hot_pushforward(sess, cols, K, r_cycle)
    for g, (_, a) in zip(G, cases):
        assert len(g) == K and g.to_ints() == ref.pushforward(a, K, r_cycle)


def test_one_hot_device_columns(sess):
    torch = pytest.importorskip("torch")
    K, T = 256, 1 << 12
    col, a = address_column(K, T, np.uint8, 3, 0.3)
    pt = point("random", 20, 9)
    want = ref.one_hot_evaluate_direct(a, K, T, pt, "cycle_major")
    assert one_hot_evaluate(sess, torch.from_numpy(col).cuda(), K, pt) == [want]
    G = one_hot_pushforward(sess, torch.from_numpy(col).cuda(), K, pt[:12])
    assert G[0].to_ints() == ref.pushforward(a, K, pt[:12])


# ---- at scale ------------------------------------------------------------------------------------------------------
def test_field_table_2_22_against_the_c_oracle_binds(sess):
    n = 22
    tab = C.rand_limbs(22, 1 << n)
    vals, limbs = challenge_point(n, 2200)
    p = Polynomial.new(sess, tab)
    cur = tab
    for r in limbs:
        cur = C.bind(cur, r, HIGH_TO_LOW, threads=C.max_threads())
    assert p.evaluate(limbs) == F.from_limbs(cur[0])


def test_field_tables_2_24_against_device_binds_of_a_clone(sess):
    n = 24
    ps = [Polynomial.new(sess, C.rand_limbs(2400 + i, 1 << n)) for i in range(2)]
    pt = O.random_fr(2401, n)
    got = Polynomial.batch_evaluate(ps, pt)
    for p, g in zip(ps, got):
        q = p.clone()
        for r in pt:
            q.bind(r, HIGH_TO_LOW)
        assert q.to_ints() == [g]
        q.free()
    lo = ps[0].clone()
    for r in reversed(pt):
        lo.bind(r, LOW_TO_HIGH)
    assert lo.to_ints() == [got[0]]


def test_u64_column_2_24_against_upload_and_the_field_path(sess):
    n = 24
    col = np.random.Generator(np.random.PCG64(64)).integers(0, 1 << 64, size=1 << n, dtype=np.uint64)
    col[0] = np.uint64((1 << 64) - 1)
    pt = O.random_fr(65, n)
    want = Polynomial.from_small(sess, col).evaluate(pt)
    assert evaluate_small(sess, col, pt) == [want]


def test_one_hot_2_24_closed_forms(sess):
    K, T = 256, 1 << 24
    lt, lk = 24, 8
    r_cycle, r_addr = point("random", lt, 11), point("random", lk, 12)
    eq_addr = O.eq_evals(r_addr)
    const = np.full(T, 37, dtype=np.uint8)
    # address-major runs over all 256 addresses (u16: 255 is an address, not the u8 none value)
    block_u16 = (np.arange(T, dtype=np.uint64) >> np.uint64(lt - lk)).astype(np.uint16)
    e_a = [0] * K
    e_a[37] = 1
    assert one_hot_pushforward(sess, const, K, r_cycle)[0].to_ints() == e_a     # sum_j eq(r, j) = 1
    eq_top = O.eq_evals(r_cycle[:lk])
    assert one_hot_pushforward(sess, block_u16, K, r_cycle)[0].to_ints() == eq_top   # G[k] = eq(r_cycle[:log K], k)
    assert one_hot_evaluate(sess, const, K, r_cycle + r_addr) == [eq_addr[37]]
    assert one_hot_evaluate(sess, block_u16, K, r_cycle + r_addr) == [sum(a * b for a, b in zip(eq_addr, eq_top)) % R]
    # the global-bin and gather-through-L2 shapes (K > the shared-memory limits)
    Gw = one_hot_pushforward(sess, block_u16, 1 << 16, r_cycle)[0].to_ints()
    assert Gw[:K] == eq_top and not any(Gw[K:])
    # random addresses: the evaluation is the pushforward's dot product
    col = np.random.Generator(np.random.PCG64(13)).integers(0, 255, size=T).astype(np.uint8)
    col[::7] = ONE_HOT_NONE[np.dtype(np.uint8)]
    Gr = one_hot_pushforward(sess, col, K, r_cycle)[0].to_ints()
    assert one_hot_evaluate(sess, col, K, r_cycle + r_addr) == [sum(a * b for a, b in zip(eq_addr, Gr)) % R]


def test_results_are_deterministic(sess):
    K, T = 16, 1 << 20
    col = np.zeros(T, dtype=np.uint8)                       # skewed: every cycle at one address
    col[1::3] = 5
    pt = point("random", 24, 1)
    a = [one_hot_evaluate(sess, col, K, pt) for _ in range(3)]
    g = [one_hot_pushforward(sess, col, K, pt[:20])[0].to_ints() for _ in range(3)]
    assert a[0] == a[1] == a[2] and g[0] == g[1] == g[2]


# ---- errors --------------------------------------------------------------------------------------------------------
def _status(fn):
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        fn()
    return e.value.status


def test_errors_and_the_context_stays_usable(sess):
    lib, h = sess.lib, sess.h
    tab = O.random_fr(5, 16)
    p, q = Polynomial.from_ints(sess, tab), Polynomial.from_ints(sess, tab[:8])
    pt = point("random", 4, 5)
    bad_pt = F.ints_to_limbs(pt)
    bad_pt[1] = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)   # non-canonical
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    assert _status(lambda: Polynomial.batch_evaluate([p, q], pt[:4])) == INV          # different lengths
    assert _status(lambda: p.evaluate(pt[:3])) == INV                                # nvars != log2(len)
    assert _status(lambda: p.evaluate(bad_pt)) == INV
    assert lib.jb_table_evaluate_batch(h, None, 1, _p(F.ints_to_limbs(pt)), 4, None) == INV
    assert lib.jb_table_evaluate_batch(h, None, 0, None, 0, None) == _lib.JB_OK       # count == 0
    col = np.arange(16, dtype=np.uint8)
    assert _status(lambda: evaluate_small(sess, col, pt[:3])) == INV
    assert _status(lambda: evaluate_small(sess, col[:12], pt[:4])) == INV           # not a power of two
    ptrs = (ctypes.c_void_p * 1)(col.ctypes.data)
    ol = np.zeros((1, 4), dtype=np.uint64)
    assert lib.jb_small_evaluate_batch(h, ptrs, 1, (ctypes.c_int * 1)(0), 16, 0, _p(F.ints_to_limbs(pt)), 4, _p(ol)) == INV
    assert lib.jb_small_evaluate_batch(h, ptrs, 1, (ctypes.c_int * 1)(10), 16, 0, _p(F.ints_to_limbs(pt)), 4, _p(ol)) == INV
    import torch
    dev = torch.zeros(64, dtype=torch.int64, device="cuda")
    u8k, u64k = (ctypes.c_int * 1)(1), (ctypes.c_int * 1)(4)
    nul = (ctypes.c_void_p * 1)(None)
    assert lib.jb_small_evaluate_batch(h, ptrs, 1, u8k, 16, 2, _p(F.ints_to_limbs(pt)), 4, _p(ol)) == INV  # on_device
    assert lib.jb_small_evaluate_batch(h, nul, 1, u8k, 16, 0, _p(F.ints_to_limbs(pt)), 4, _p(ol)) == INV   # null column
    assert lib.jb_small_evaluate_batch(h, (ctypes.c_void_p * 1)(dev.data_ptr() + 4), 1, u64k, 16, 1,        # misaligned
                                       _p(F.ints_to_limbs(pt)), 4, _p(ol)) == INV
    addr = np.array([0, 1, 2, 3, 0xFF, 1, 0, 2], dtype=np.uint8)
    opt = point("random", 5, 6)
    with pytest.raises(ValueError):
        one_hot_evaluate(sess, addr, 4, opt[:4])                                     # wrong point length
    aptrs = (ctypes.c_void_p * 1)(addr.ctypes.data)
    o5 = F.ints_to_limbs(opt)
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 8, 3, 0, 0, _p(o5), _p(ol)) == INV  # K not a power of two
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 6, 4, 0, 0, _p(o5), _p(ol)) == INV  # T not a power of two
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 4, 8, 4, 0, 0, _p(o5), _p(ol)) == INV  # u64 addresses
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 8, 4, 2, 0, _p(o5), _p(ol)) == INV  # unknown layout
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 1 << 31, 4, 0, 0, _p(o5), _p(ol)) == UNS
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 8, 1 << 17, 0, 0, _p(o5), _p(ol)) == UNS   # K > 2^16
    assert lib.jb_one_hot_evaluate(h, aptrs, 1, 1, 8, 4, 0, 2, _p(o5), _p(ol)) == INV  # on_device
    assert lib.jb_one_hot_evaluate(h, nul, 1, 1, 8, 4, 0, 0, _p(o5), _p(ol)) == INV    # null column
    odd = (ctypes.c_void_p * 1)(dev.data_ptr() + 1)
    assert lib.jb_one_hot_evaluate(h, odd, 1, 2, 8, 4, 0, 1, _p(o5), _p(ol)) == INV    # misaligned u16 device column
    oh = np.zeros(1, dtype=np.uint64)
    assert lib.jb_one_hot_pushforward(h, odd, 1, 2, 8, 4, 1, _p(F.ints_to_limbs(opt[:3])), _p(oh)) == INV
    assert lib.jb_one_hot_pushforward(h, aptrs, 1, 1, 8, 4, 0, None, None) == INV
    assert lib.jb_one_hot_evaluate(h, aptrs, 0, 1, 8, 4, 0, 0, _p(o5), _p(ol)) == _lib.JB_OK
    # an address >= K that is not the none value: found on the device
    far = addr.copy()
    far[6] = 9
    assert _status(lambda: one_hot_evaluate(sess, far, 4, opt)) == INV
    assert _status(lambda: one_hot_pushforward(sess, far, 4, opt[:3])) == INV
    # the context keeps working
    a = [None if v == 0xFF else int(v) for v in addr]
    assert one_hot_evaluate(sess, addr, 4, opt) == [ref.one_hot_evaluate(a, 4, 8, opt, "cycle_major")]
    assert one_hot_pushforward(sess, addr, 4, opt[:3])[0].to_ints() == ref.pushforward(a, 4, opt[:3])
    assert p.evaluate(pt) == ref.evaluate(tab, pt)
