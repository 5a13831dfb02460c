"""Read-write checking member on the device (jb_member_create_read_write), bit-exact against rw_ref: every round of
both phases in lockstep (with and without verify mode), edge values and access patterns, the claimed sum at 2^16
cycles, batching through the scheduler, and every refusal."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import LOW_TO_HIGH, HIGH_TO_LOW, Polynomial, ProductMember, ReadWriteCheckingMember, RoundScheduler, Source, _lib
from jolt_b200 import field as F
from oracle import bn254 as O
import rw_ref as R

P = O.R_MOD
MAX125 = F.from_limbs(np.array([0, 0, (1 << 64) - 1, (1 << 61) - 1], dtype=np.uint64))
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def _addr_col(ad, K):
    dt = np.uint8 if K <= 256 else np.uint16
    none = np.iinfo(dt).max
    return np.array([none if a is None else a for a in ad], dtype=dt)


def _signed(x):
    return x if x < (1 << 127) else x - P


def _member(sess, wl, w, scale, inc_kind="table", values_kind="table"):
    K, T, accesses, write, inc, init = wl
    cols = {}
    acc = []
    for ad, values, c, d in accesses:
        key = id(ad)
        if key not in cols:
            cols[key] = _addr_col(ad, K)
        if values_kind == "table":
            v = Source.table(Polynomial.from_ints(sess, values))
        else:
            v = Source.compact(np.array(values, dtype=np.uint64))
        acc.append((cols[key], v, c, d))
    if inc_kind == "table":
        inc_s = Source.table(Polynomial.from_ints(sess, inc))
    else:
        inc_s = Source.compact([_signed(x) for x in inc], inc_kind)
    init_s = Source.compact(np.array(init, dtype=np.uint64))
    return ReadWriteCheckingMember(sess, acc, write, inc_s, init_s, K, w, scale)


def _lockstep(sess, wl, w, scale, ch, verify=False, **kw):
    K, T, accesses, write, inc, init = wl
    want_rounds, want_final = R.sparse_prove(*wl, w, scale, ch)
    m = _member(sess, wl, w, scale, **kw)
    assert m.num_rounds() == len(ch) and m.degree() == 3
    sess.set_verify_rounds(verify)
    try:
        claim = R.claimed_sum(T, accesses, inc, w, scale)
        bind = None
        for rnd in range(len(ch)):
            got = m.prove_round_evals(bind, rnd, claim)
            assert got == want_rounds[rnd], rnd
            assert (got[0] + got[1]) % P == claim
            bind = ch[rnd]
            claim = O.uni_evaluate(O.uni_from_evals(got), bind)
        m.finish_rounds(bind)
        assert m.final_evals() == want_final
        t = T.bit_length() - 1
        assert m.eq_scalar() == O.evaluate(O.eq_evals(w, scale), ch[:t][::-1])
    finally:
        sess.set_verify_rounds(False)
        m.close()


@pytest.mark.parametrize("K,T,A,shape", [(1, 2, 1, "registers"), (2, 4, 2, "registers"), (8, 64, 3, "registers"),
                                         (128, 1024, 3, "registers"), (128, 64, 4, "registers"), (8, 1024, 2, "ram"),
                                         (128, 256, 2, "ram"), (1, 64, 3, "registers"), (1024, 512, 2, "ram")])
@pytest.mark.parametrize("verify", [False, True])
def test_lockstep_with_reference(sess, K, T, A, shape, verify):
    wl = R.workload(K * 31 + T + A, K, T, A, shape)
    t = T.bit_length() - 1
    w = O.random_fr(K + T, t)
    ch = O.random_fr(K + 2 * T, t + K.bit_length() - 1)
    _lockstep(sess, wl, w, O.random_fr(3, 1)[0] if verify else None, ch, verify)


@pytest.mark.parametrize("inc_kind", ["i64", "i128", "s64", "s128"])
def test_compact_increments(sess, inc_kind):
    bits = 64 if inc_kind in ("i64", "s64") else 128
    wl = R.workload(17, 16, 256, 3, "registers", inc_bits=bits)
    K, T, accesses, write, inc, init = wl
    # extremes, including negative ones, at a few written cycles
    lo, hi = -(1 << (bits - 1)) + (1 if inc_kind.startswith("s") else 0), (1 << (bits - 1)) - 1
    aw = accesses[write][0]
    for j, v in zip([j for j in range(T) if aw[j] is not None][:4], [lo, hi, -1, 0]):
        inc[j] = v % P
    val = R.val_table(K, T, accesses, write, inc, init)
    accesses = [(ad, [0 if ad[j] is None else val[ad[j]][j] for j in range(T)], c, d) for ad, _v, c, d in accesses]
    wl = (K, T, accesses, write, inc, init)
    _lockstep(sess, wl, O.random_fr(5, 8), None, O.random_fr(6, 12), inc_kind=inc_kind)


def test_edge_values_and_challenges(sess):
    K, T = 4, 16
    ad = [j % K if j % 3 else None for j in range(T)]
    accesses_addr = [ad, ad]
    inc = [0 if a is None else [P - 1, (1 << 64) - 1, 1, 0][j % 4] for j, a in enumerate(ad)]
    init = [(1 << 64) - 1, 0, 1, (1 << 63)]
    val = R.val_table(K, T, [(a, None, 0, 0) for a in accesses_addr], 1, inc, init)
    acc = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], c, d)
           for a, c, d in zip(accesses_addr, [1, P - 1], [0, 1])]
    wl = (K, T, acc, 1, inc, init)
    for ch in ([0, 1, P - 1, MAX125, 1, 0], [MAX125] * 6, [P - 1] * 6):
        _lockstep(sess, wl, [MAX125, P - 1, 1, 5], P - 1, ch)


@pytest.mark.parametrize("pattern", ["all_none", "one_key", "distinct", "rs1_rs2_rd", "write_only"])
def test_access_patterns(sess, pattern):
    K, T = 128, 128
    rng = np.random.default_rng(7)
    if pattern == "all_none":
        cols = [[None] * T] * 3
    elif pattern == "one_key":
        cols = [[5] * T] * 3
    elif pattern == "distinct":
        cols = [[(j + 40 * a) % K for j in range(T)] for a in range(3)]
    elif pattern == "rs1_rs2_rd":
        c = [int(x) for x in rng.integers(0, K, T)]
        cols = [c, c, c]
    else:  # writes to keys never read
        cols = [[int(x) for x in rng.integers(0, 16, T)]] * 2 + [[int(x) for x in rng.integers(64, K, T)]]
    inc = [0 if cols[2][j] is None else int(rng.integers(0, 1 << 40)) for j in range(T)]
    init = [int(x) for x in rng.integers(0, 1 << 60, K)]
    val = R.val_table(K, T, [(a, None, 0, 0) for a in cols], 2, inc, init)
    acc = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], c, d)
           for a, c, d in zip(cols, O.random_fr(9, 3), [0, 0, 1])]
    _lockstep(sess, (K, T, acc, 2, inc, init), O.random_fr(10, 7), None, O.random_fr(11, 14))


def test_u16_addresses_k_2_16(sess):
    wl = R.workload(21, 1 << 16, 64, 2, "ram", none_frac=0.05)
    _lockstep(sess, wl, O.random_fr(12, 6), None, O.random_fr(13, 22))


def test_claimed_sum_at_2_16_cycles(sess):
    # every round passes the s(0) + s(1) check against the host sum; the final claim matches the final values
    K, T = 128, 1 << 16
    wl = R.workload(33, K, T, 3, "registers")
    K, T, accesses, write, inc, init = wl
    t = T.bit_length() - 1
    w = O.random_fr(34, t)
    m = _member(sess, wl, w, None)
    claim = R.claimed_sum(T, accesses, inc, w)
    ch = O.random_fr(35, t + 7)
    bind = None
    for rnd in range(len(ch)):
        got = m.prove_round_evals(bind, rnd, claim)
        assert (got[0] + got[1]) % P == claim, rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    fin = m.final_evals()
    e = m.eq_scalar()
    assert claim == e * sum(c * fin[a] * (fin[-2] + d * fin[-1]) for a, (_x, _v, c, d) in enumerate(accesses)) % P
    # inc(r_cycle) and ra_a(r) by independent evaluations
    r_cycle = ch[:t][::-1]
    assert fin[-1] == O.evaluate([x % P for x in inc], r_cycle)
    r_addr = ch[t:][::-1]
    for a, (ad, _v, _c, _d) in enumerate(accesses):
        want = jolt_b200.one_hot_evaluate(sess, _addr_col(ad, K), K, r_addr + r_cycle, layout="address_major")[0]
        assert fin[a] == want
    m.close()


def test_scheduler_with_a_member_of_another_size(sess):
    wl = R.workload(41, 8, 32, 3, "registers")
    K, T, accesses, write, inc, init = wl
    w, ch = O.random_fr(42, 5), O.random_fr(43, 8)
    want_rounds, want_final = R.sparse_prove(*wl, w, None, ch)
    rw = _member(sess, wl, w, None)
    tabs = [O.random_fr(44 + j, 16) for j in range(2)]
    pm = ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tabs], LOW_TO_HIGH)
    sched = RoundScheduler(sess, [rw, pm])
    c_rw = R.claimed_sum(T, accesses, inc, w)
    c_pm = sum(a * b for a, b in zip(*tabs)) % P
    for rnd in range(8):
        work = [(0, rnd, None if rnd == 0 else ch[rnd - 1], c_rw)]
        if rnd < 4:
            work.append((1, rnd, None if rnd == 0 else ch[rnd - 1], c_pm))
        polys = sched.batch_prove_round(work)
        assert [polys[0].evaluate(x) for x in range(4)] == want_rounds[rnd]
        c_rw = polys[0].evaluate(ch[rnd])
        if rnd < 4:
            c_pm = polys[1].evaluate(ch[rnd])
    sched.batch_finish_rounds([(0, ch[7])])
    assert rw.final_evals() == want_final
    sched.close()
    rw.close()
    pm.close()


def _status(fn):
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        fn()
    return e.value.status


def test_refusals(sess):
    K, T = 8, 16
    wl = R.workload(51, K, T, 2, "registers")
    w = O.random_fr(52, 4)
    inc_poly = Polynomial.from_ints(sess, wl[4])
    base = [(_addr_col(ad, K), Source.compact(np.array([v % (1 << 64) for v in vals], dtype=np.uint64)), c, d)
            for ad, vals, c, d in wl[2]]
    init = np.array(wl[5], dtype=np.uint64)

    def make(acc=base, write=1, inc=None, init_=init, K_=K, w_=w, order=LOW_TO_HIGH, scale=None):
        return ReadWriteCheckingMember(sess, acc, write, Source.table(inc_poly) if inc is None else inc, init_, K_, w_,
                                       scale, order)

    assert _status(lambda: make(order=HIGH_TO_LOW)) == _lib.JB_ERR_UNSUPPORTED
    assert _status(lambda: make(acc=base * 3)) == _lib.JB_ERR_UNSUPPORTED
    assert _status(lambda: make(acc=[])) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(write=2)) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(K_=6)) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(K_=1 << 17)) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(w_=w[:3])) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(scale=np.full(4, (1 << 64) - 1, dtype=np.uint64))) == _lib.JB_ERR_INVALID
    assert _status(lambda: make(acc=[(a, v, np.array([0, 0, 0, 1 << 63], dtype=np.uint64), d)
                                     for a, v, _c, d in base])) == _lib.JB_ERR_INVALID
    odd = [(a[:15], v, c, d) for a, v, c, d in base]
    assert _status(lambda: make(acc=odd)) == _lib.JB_ERR_INVALID
    # found on the device: an address >= K; a nonzero increment at a cycle whose write address is none
    a0 = base[0][0].copy()
    a0[3] = K
    assert _status(lambda: make(acc=[(a0,) + base[0][1:], base[1]])) == _lib.JB_ERR_INVALID
    aw = base[1][0].copy()
    aw[5] = 0xFF
    inc2 = np.zeros(T, dtype=np.uint64)
    inc2[5] = 7
    assert _status(lambda: make(acc=[base[0], (aw,) + base[1][1:]], inc=Source.compact(inc2))) == _lib.JB_ERR_INVALID
    # the table sources stay the caller's, and the context is still usable
    assert len(inc_poly.to_ints()) == T
    m = make()
    assert m.num_rounds() == 4 + 3
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        m.prove_round_evals(None, 0, None)
    assert e.value.status == _lib.JB_ERR_INVALID
    m.close()
