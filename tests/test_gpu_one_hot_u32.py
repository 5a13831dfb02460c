"""u32 address columns (JB_SCALAR_U32, K up to 2^24) on the device, in the entry points that take them -
jb_one_hot_evaluate, jb_one_hot_pushforward, product members over one-hot sources and read-write checking:
  - widening is exact: a u32 copy of a u8 / u16 column (its none value mapped to 0xFFFFFFFF) gives bit-identical
    evaluations, pushforward tables, round polynomials and final values;
  - above 2^16 (K = 2^17, 2^20, 2^24) against independent references: per-cycle eq(r_cycle, j) eq(r_addr, a_j) on the
    host, the pushforward's hit addresses and zeros elsewhere, the product over a table source of the host-gathered
    eq(r_addr, addr_j), read-write in lockstep with rw_ref.sparse_prove (the helpers for
    these sizes are tests/u32_ref.py's);
  - addresses 0 and K - 1, the none value, host and device columns, misaligned device columns, and every refusal;
  - RAM at real size: K = 2^22, T = 2^20, one u32 device column read and written (uniform and random-walk addresses),
    every read-write round from a claim computed outside the member and the final claim from independent evaluations
    (ra by one_hot_evaluate, Val by init~ plus a product member inc * wa * LT, inc by evaluate_small)."""
import ctypes

import numpy as np
import pytest
import torch

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, ONE_HOT_NONE, ExpressionMember, LtPolynomial, Polynomial,
                       ProductMember, ReadWriteCheckingMember, Source, _lib, evaluate_small, one_hot_evaluate,
                       one_hot_pushforward)
from jolt_b200 import field as F
from jolt_b200.api import _p
from oracle import bn254 as O
import rw_ref as R
import u32_ref as U

P = O.R_MOD
NONE32 = 0xFFFFFFFF
INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def widen(col):
    """The u32 copy of a u8 / u16 column: astype alone would turn the none value 0xFFFF into the address 65535."""
    w = col.astype(np.uint32)
    w[col == ONE_HOT_NONE[col.dtype]] = NONE32
    return w


def on_device(col):
    view = {np.dtype(np.uint8): np.uint8, np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32}[col.dtype]
    return torch.from_numpy(col.view(view)).cuda()


def column(T, K, seed, dtype=np.uint32, none_frac=0.2):
    """T addresses below K (also below the none value), a fraction none; cycles 0 and 1 touch addresses 0 and K - 1."""
    rng = np.random.default_rng(seed)
    top = min(K, int(np.iinfo(dtype).max))
    a = rng.integers(0, top, T).astype(dtype)
    a[rng.random(T) < none_frac] = np.iinfo(dtype).max
    a[0], a[1] = 0, min(K - 1, top - 1)
    return a


def addrs(col):
    none = ONE_HOT_NONE[col.dtype]
    return [None if int(a) == none else int(a) for a in col]


def _status(fn):
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        fn()
    return e.value.status


def _lockstep(a, b, n, claim, seed, order):
    """Runs two members round by round on the same challenges; both must publish the same values throughout."""
    ch = O.random_fr(seed, n)
    bind = None
    for rnd in range(n):
        ga = a.prove_round_evals(bind, rnd, claim)
        assert ga == b.prove_round_evals(bind, rnd, claim), rnd
        if claim is not None:
            assert (ga[0] + ga[1]) % P == claim, rnd
            claim = O.uni_evaluate(O.uni_from_evals(ga), ch[rnd])
        bind = ch[rnd]
    a.finish_rounds(bind)
    b.finish_rounds(bind)
    assert a.final_evals() == b.final_evals()
    a.close()
    b.close()


# ---- widening is exact ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,T,dtype", [(16, 1 << 10, np.uint8), (256, 1 << 12, np.uint8), (1 << 10, 1 << 12, np.uint16),
                                       (1 << 16, 1 << 12, np.uint16)])
@pytest.mark.parametrize("device", [False, True])
def test_widening_evaluate_and_pushforward(sess, K, T, dtype, device):
    cols = [column(T, K, 10 + s, dtype) for s in range(3)]
    wide = [widen(c) for c in cols]
    if device:
        cols, wide = [on_device(c) for c in cols], [on_device(c) for c in wide]
    lt, lk = T.bit_length() - 1, K.bit_length() - 1
    pt = O.random_fr(K + T, lt + lk)
    for layout in ("cycle_major", "address_major"):
        assert one_hot_evaluate(sess, wide, K, pt, layout) == one_hot_evaluate(sess, cols, K, pt, layout)
    r_cycle = pt[:lt]
    for g, w in zip(one_hot_pushforward(sess, cols, K, r_cycle), one_hot_pushforward(sess, wide, K, r_cycle)):
        assert np.array_equal(g.evals(), w.evals())


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("eq", [False, True])
def test_widening_product_sources(sess, order, eq):
    n = 10
    a8, a16 = column(1 << n, 256, 21, np.uint8), column(1 << n, 1 << 16, 22, np.uint16)
    r8, r16 = O.random_fr(23, 8), O.random_fr(24, 16)
    vals = np.random.default_rng(25).integers(0, 1 << 63, 1 << n).astype(np.uint64)
    w = O.random_fr(26, n) if eq else None

    def member(x8, x16):
        srcs = [Source.one_hot(x8, 256, r8), Source.compact(vals, "u64"), Source.one_hot(x16, 1 << 16, r16)]
        return ProductMember.from_sources(sess, srcs, None if w is None else F.ints_to_limbs(w), order=order)

    claim = None
    if eq:
        f = [U.eq_at(r8, a) if a is not None else 0 for a in addrs(a8)]
        g = [U.eq_at(r16, a) if a is not None else 0 for a in addrs(a16)]
        claim = sum(e * x * int(v) * y for e, x, v, y in zip(O.eq_evals(w), f, vals, g)) % P
    _lockstep(member(a8, a16), member(widen(a8), on_device(widen(a16))), n, claim, 27, order)


def _rw_member(sess, wl, w, wide, device=False):
    K, T, accesses, write, inc, init = wl
    dt = np.uint8 if K <= 256 else np.uint16 if K <= (1 << 16) else np.uint32
    cols, acc = {}, []
    for ad, values, c, d in accesses:
        if id(ad) not in cols:
            col = np.array([np.iinfo(dt).max if x is None else x for x in ad], dtype=dt)
            col = widen(col) if wide and dt != np.uint32 else col
            cols[id(ad)] = on_device(col) if device else col
        acc.append((cols[id(ad)], Source.table(Polynomial.from_ints(sess, values)), c, d))
    return ReadWriteCheckingMember(sess, acc, write, Source.table(Polynomial.from_ints(sess, inc)),
                                   Source.compact(np.array(init, dtype=np.uint64)), K, w)


@pytest.mark.parametrize("K,T,shape,A", [(8, 64, "registers", 3), (256, 32, "registers", 2), (1 << 16, 16, "ram", 2)])
def test_widening_read_write(sess, K, T, shape, A):
    wl = R.workload(31 + K, K, T, A, shape)
    w = O.random_fr(32 + K, T.bit_length() - 1)
    claim = R.claimed_sum(T, wl[2], wl[4], w)
    n = T.bit_length() - 1 + K.bit_length() - 1
    _lockstep(_rw_member(sess, wl, w, False), _rw_member(sess, wl, w, True, device=True), n, claim, 33, LOW_TO_HIGH)


# ---- above 2^16 ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1 << 17, 1 << 20, 1 << 24])
@pytest.mark.parametrize("device", [False, True])
def test_evaluate_above_2_16(sess, K, device):
    T = 1 << 12
    cols = [column(T, K, 40 + s) for s in range(2)]
    dcols = [on_device(c) for c in cols] if device else cols
    lt, lk = 12, K.bit_length() - 1
    r_cycle, r_addr = O.random_fr(41, lt), O.random_fr(42, lk)
    want = [U.one_hot_evaluate_sparse(addrs(c), r_cycle, r_addr) for c in cols]
    assert one_hot_evaluate(sess, dcols, K, r_cycle + r_addr, "cycle_major") == want
    assert one_hot_evaluate(sess, dcols, K, r_addr + r_cycle, "address_major") == want


@pytest.mark.parametrize("K", [1 << 17, 1 << 20, 1 << 24])
def test_pushforward_above_2_16(sess, K):
    T = 1 << 12
    col = column(T, K, 50 + K.bit_length())
    r_cycle = O.random_fr(51, 12)
    want = U.pushforward_sparse(addrs(col), r_cycle)
    for src in (col, on_device(col)):
        (g,) = one_hot_pushforward(sess, [src], K, r_cycle)
        ev = g.evals()
        g.free()
        hit = np.flatnonzero(ev.any(axis=1))
        assert hit.tolist() == sorted(want)            # the hit addresses (0 and K - 1 among them), zeros elsewhere
        assert F.limbs_to_ints(ev[hit]) == [want[k] for k in hit.tolist()]
        del ev


@pytest.mark.parametrize("K", [1 << 17, 1 << 20, 1 << 24])
@pytest.mark.parametrize("eq", [False, True])
def test_product_sources_above_2_16(sess, K, eq):
    n = 10
    col = column(1 << n, K, 60 + K.bit_length())
    r_addr = O.random_fr(61, K.bit_length() - 1)
    gathered = [0 if a is None else U.eq_at(r_addr, a) for a in addrs(col)]
    vals = np.random.default_rng(62).integers(-(1 << 62), 1 << 62, 1 << n).astype(np.int64)
    w = O.random_fr(63, n) if eq else None
    wl = None if w is None else F.ints_to_limbs(w)
    u32 = ProductMember.from_sources(sess, [Source.compact(vals, "i64"), Source.one_hot(on_device(col), K, r_addr)], wl,
                                     order=LOW_TO_HIGH)
    tab = ProductMember.from_sources(sess, [Source.compact(vals, "i64"), Source.table(Polynomial.from_ints(sess, gathered))],
                                     wl, order=LOW_TO_HIGH)
    claim = None
    if eq:
        claim = sum(e * (int(v) % P) * g for e, v, g in zip(O.eq_evals(w), vals, gathered)) % P
    _lockstep(u32, tab, n, claim, 64, LOW_TO_HIGH)


@pytest.mark.parametrize("device", [False, True])
def test_read_write_k_2_17_lockstep(sess, device):
    K, T = 1 << 17, 16
    wl = U.ram_workload_with_edges(71, K, T)
    t = T.bit_length() - 1
    w = O.random_fr(72, t)
    ch = O.random_fr(73, t + 17)
    want_rounds, want_final = R.sparse_prove(*wl, w, None, ch)
    m = _rw_member(sess, wl, w, True, device)
    claim = R.claimed_sum(T, wl[2], wl[4], w)
    bind = None
    for rnd in range(t + 17):
        got = m.prove_round_evals(bind, rnd, claim)
        assert got == want_rounds[rnd], rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    assert m.final_evals() == want_final
    m.close()


# ---- refusals -----------------------------------------------------------------------------------------------------
def test_refusals_and_the_context_keeps_working(sess):
    T = 1 << 10
    K = 1 << 24
    good = column(T, K, 80)
    r_cycle, r_addr = O.random_fr(81, 10), O.random_fr(82, 24)
    pt = r_cycle + r_addr
    want = one_hot_evaluate(sess, good, K, pt)
    bad_values = [K, 1 << 24, 0xFFFFFFFE]

    def check_good():
        assert one_hot_evaluate(sess, good, K, pt) == want

    for x in bad_values:           # an address >= K that is not the none value: found on the device
        bad = good.copy()
        bad[5] = x
        for b in (bad, on_device(bad)):
            assert _status(lambda: one_hot_evaluate(sess, b, K, pt)) == INV
            assert _status(lambda: one_hot_pushforward(sess, b, K, r_cycle)) == INV
            assert _status(lambda: ProductMember.from_sources(sess, [Source.one_hot(b, K, r_addr)])) == INV
            check_good()
    # K = 2^25: beyond the u32 limit
    big = O.random_fr(83, 25)
    assert _status(lambda: one_hot_evaluate(sess, good, 1 << 25, r_cycle + big)) == UNS
    assert _status(lambda: one_hot_pushforward(sess, good, 1 << 25, r_cycle)) == UNS
    assert _status(lambda: ProductMember.from_sources(sess, [Source.one_hot(good, 1 << 25, big)])) == INV
    check_good()
    # u8 / u16 columns keep K <= 2^16 where u32 reaches 2^24
    c16 = column(T, 1 << 16, 84, np.uint16)
    assert _status(lambda: one_hot_evaluate(sess, c16, 1 << 17, r_cycle + big[:17])) == UNS
    assert _status(lambda: ProductMember.from_sources(sess, [Source.one_hot(c16, 1 << 17, big[:17])])) == INV
    # expression members over sources keep u8 / u16
    assert _status(lambda: ExpressionMember.from_sources(sess, [Source.one_hot(good, K, r_addr)], [(1, [0])])) == INV
    assert _status(lambda: ExpressionMember.from_sources(sess, [Source.one_hot(column(T, 16, 85), 16, r_addr[:4])],
                                                         [(1, [0])])) == INV
    # misaligned u32 device columns (refused before anything is read)
    raw = torch.zeros(T + 1, dtype=torch.int32, device="cuda")
    ptrs = (ctypes.c_void_p * 1)(raw.data_ptr() + 2)
    out = np.zeros((1, 4), dtype=np.uint64)
    ptl = F.ints_to_limbs(pt)
    sess.after_torch()
    assert sess.lib.jb_one_hot_evaluate(sess.h, ptrs, 1, 3, T, K, 0, 1, _p(ptl), _p(out)) == INV
    oh = np.zeros(1, dtype=np.uint64)
    rcl = F.ints_to_limbs(r_cycle)
    assert sess.lib.jb_one_hot_pushforward(sess.h, ptrs, 1, 3, T, K, 1, _p(rcl), _p(oh)) == INV
    check_good()
    # read-write: K = 2^25 and addresses >= K
    wl = U.ram_columns_workload_u32(86, 1 << 17, 1 << 6)
    w = O.random_fr(87, 6)

    def rw(cols, K_):
        acc = [(cols, Source.compact(v, "u64"), c, d) for v, c, d in zip(wl["values"], wl["coeffs"], wl["ds"])]
        return ReadWriteCheckingMember(sess, acc, wl["write"], Source.compact(wl["inc"], "u64"),
                                       Source.compact(np.resize(wl["init"], K_), "u64"), K_, w)

    assert _status(lambda: rw(wl["addrs"][0], 1 << 25)) == INV
    for x in (1 << 17, 1 << 24, 0xFFFFFFFE):
        bad = wl["addrs"][0].copy()
        bad[3] = x
        assert _status(lambda: rw(bad, 1 << 17)) == INV
        assert _status(lambda: rw(on_device(bad), 1 << 17)) == INV
    m = rw(wl["addrs"][0], 1 << 17)
    ev = evaluate_small(sess, wl["values"] + [wl["inc"]], w, "u64")
    claim = sum(c * (v + d * ev[-1]) for c, v, d in zip(wl["coeffs"], ev, wl["ds"])) % P
    got = m.prove_round_evals(None, 0, claim)
    assert (got[0] + got[1]) % P == claim
    m.close()
    check_good()


# ---- RAM at real size -----------------------------------------------------------------------------------------------
def _val_at(sess, wl, r_addr, r_cycle):
    """Val(r_addr, r_cycle) = init~(r_addr) + sum_j inc(j) wa(r_addr, j) LT(j, r_cycle): s(0) + s(1) of the first round of
    a product member over inc, the u32 write column and the LT table."""
    lt = LtPolynomial.evals(sess, F.ints_to_limbs(r_cycle))
    m = ProductMember.from_sources(sess, [Source.compact(wl["inc"], "u64"),
                                          Source.one_hot(wl["addrs"][wl["write"]], wl["K"], r_addr), Source.table(lt)],
                                   order=LOW_TO_HIGH)
    s = m.prove_round_evals(None, 0, None)
    m.close()
    return (evaluate_small(sess, [wl["init"]], r_addr, "u64")[0] + s[0] + s[1]) % P


@pytest.mark.parametrize("K,T,local", [(1 << 20, 1 << 10, False), (1 << 22, 1 << 20, False), (1 << 22, 1 << 20, True)])
def test_ram_chain(sess, K, T, local):
    wl = U.ram_columns_workload_u32(90 + K.bit_length() + T.bit_length() + local, K, T, local=local)
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    w = O.random_fr(91, t)
    ch = O.random_fr(92 + local, t + kappa)
    col = on_device(wl["addrs"][0])                 # one device column, read and written
    acc = [(col, Source.compact(v, "u64"), c, d) for v, c, d in zip(wl["values"], wl["coeffs"], wl["ds"])]
    m = ReadWriteCheckingMember(sess, acc, wl["write"], Source.compact(wl["inc"], "u64"),
                                Source.compact(wl["init"], "u64"), K, w)
    ev = evaluate_small(sess, wl["values"] + [wl["inc"]], w, "u64")
    claim = sum(c * (v + d * ev[-1]) for c, v, d in zip(wl["coeffs"], ev, wl["ds"])) % P
    bind = None
    for rnd in range(t + kappa):
        got = m.prove_round_evals(bind, rnd, claim)
        assert (got[0] + got[1]) % P == claim, rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    fin = m.final_evals()
    e = m.eq_scalar()
    m.close()
    A = 2
    assert claim == e * sum(c * fin[a] * (fin[A] + d * fin[A + 1])
                            for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"]))) % P
    r_cycle, r_addr = ch[:t][::-1], ch[t:][::-1]
    ra = one_hot_evaluate(sess, col, K, r_addr + r_cycle, layout="address_major")[0]
    assert fin[0] == fin[1] == ra
    assert fin[A + 1] == evaluate_small(sess, [wl["inc"]], r_cycle, "u64")[0]
    assert fin[A] == _val_at(sess, wl, r_addr, r_cycle)
