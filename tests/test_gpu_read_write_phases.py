"""Read-write checking member with the address rounds after p cycle rounds (jb_member_create_read_write_phases) on the
device, bit-exact against rw_phases_ref: every round in lockstep for p in {0, 1, t/2, t-1, t} (with and without verify
mode, with a scale), p = t identical to jb_member_create_read_write, the same final values under every order at one
point, the sumcheck identities and independent evaluations at 2^16 cycles, the dense device route in the mixed layout,
compact increments, edge challenges at the phase boundaries, device-resident columns, batching and refusals."""
import numpy as np
import pytest
import torch

import jolt_b200
from jolt_b200 import (LOW_TO_HIGH, HIGH_TO_LOW, BatchMember, Polynomial, ProductMember, ReadWriteCheckingMember,
                       RoundScheduler, Source, _lib, evaluate_small, one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
import rw_ref as R
import rw_phases_ref as RP

P = O.R_MOD
MAX125 = F.from_limbs(np.array([0, 0, (1 << 64) - 1, (1 << 61) - 1], dtype=np.uint64))
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def _addr_col(ad, K):
    dt = np.uint8 if K <= 256 else np.uint16 if K <= 65536 else np.uint32
    none = np.iinfo(dt).max
    return np.array([none if a is None else a for a in ad], dtype=dt)


def _signed(x):
    return x if x < (1 << 127) else x - P


def _member(sess, wl, w, scale, p, inc_kind="table"):
    K, T, accesses, write, inc, init = wl
    cols = {}
    acc = []
    for ad, values, c, d in accesses:
        cols.setdefault(id(ad), _addr_col(ad, K))
        acc.append((cols[id(ad)], Source.table(Polynomial.from_ints(sess, values)), c, d))
    if inc_kind == "table":
        inc_s = Source.table(Polynomial.from_ints(sess, inc))
    else:
        inc_s = Source.compact([_signed(x) for x in inc], inc_kind)
    return ReadWriteCheckingMember(sess, acc, write, inc_s, Source.compact(np.array(init, dtype=np.uint64)), K, w, scale,
                                   cycle_rounds_first=p)


def _run(m, ch, claim):
    """Every round at the challenges ch, checking s(0) + s(1) = claim; (rounds, final values, eq scalar)."""
    rounds, bind = [], None
    for rnd in range(len(ch)):
        got = m.prove_round_evals(bind, rnd, claim)
        assert (got[0] + got[1]) % P == claim, rnd
        rounds.append(got)
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    m.finish_rounds(bind)
    return rounds, m.final_evals(), m.eq_scalar(), claim


def _lockstep(sess, wl, w, scale, ch, p, verify=False, **kw):
    K, T, accesses, write, inc, init = wl
    want_rounds, want_final = RP.sparse_prove(*wl, w, scale, ch, p)
    m = _member(sess, wl, w, scale, p, **kw)
    assert m.num_rounds() == len(ch) and m.degree() == 3
    sess.set_verify_rounds(verify)
    try:
        rounds, fin, e, _claim = _run(m, ch, R.claimed_sum(T, accesses, inc, w, scale))
        assert rounds == want_rounds
        assert fin == want_final
        assert e == O.evaluate(O.eq_evals(w, scale), RP.point(K, T, p, ch)[1])
    finally:
        sess.set_verify_rounds(False)
        m.close()


SHAPES = [(1, 2, 1, "registers"), (2, 4, 2, "registers"), (8, 64, 3, "registers"), (128, 1024, 3, "registers"),
          (128, 64, 4, "registers"), (8, 1024, 2, "ram"), (128, 256, 2, "ram"), (1, 64, 3, "registers"),
          (1024, 512, 2, "ram")]


@pytest.mark.parametrize("K,T,A,shape", SHAPES)
@pytest.mark.parametrize("verify", [False, True])
def test_lockstep_with_reference(sess, K, T, A, shape, verify):
    wl = R.workload(K * 31 + T + A, K, T, A, shape)
    t = T.bit_length() - 1
    w = O.random_fr(K + T, t)
    ch = O.random_fr(K + 2 * T, t + K.bit_length() - 1)
    for p in sorted({0, 1, t // 2, t - 1, t}):
        _lockstep(sess, wl, w, O.random_fr(3, 1)[0] if verify else None, ch, p, verify)


def test_u16_addresses_k_2_16(sess):
    wl = R.workload(21, 1 << 16, 64, 2, "ram", none_frac=0.05)
    for p in (0, 3, 6):
        _lockstep(sess, wl, O.random_fr(12, 6), 7, O.random_fr(13, 22), p)


@pytest.mark.parametrize("K,T,A,shape", [(8, 64, 3, "registers"), (1024, 512, 2, "ram"), (1, 64, 3, "registers")])
def test_p_t_identical_to_the_original_entry_point(sess, K, T, A, shape):
    wl = R.workload(K + 3 * T, K, T, A, shape)
    K, T, accesses, write, inc, init = wl
    t = T.bit_length() - 1
    w, ch = O.random_fr(K, t), O.random_fr(T, t + K.bit_length() - 1)
    claim = R.claimed_sum(T, accesses, inc, w, 11)
    a, b = _member(sess, wl, w, 11, None), _member(sess, wl, w, 11, t)
    assert _run(a, ch, claim) == _run(b, ch, claim)
    a.close()
    b.close()


def _ram_u32_workload(seed, K, T, none_frac=0.05):
    """One u32 address column read and written (RAM), u64 values and inc: Val(k, j) by prefix sums over the writes."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, K, T).astype(np.uint32)
    a[rng.random(T) < none_frac] = 0xFFFFFFFF
    wv = a != 0xFFFFFFFF
    inc = np.where(wv, rng.integers(0, 1 << 32, T), 0).astype(np.uint64)
    init = rng.integers(0, 1 << 40, K).astype(np.uint64)
    j_all = np.arange(T, dtype=np.int64)
    k = np.where(wv, a, 0).astype(np.int64)
    wkey = np.sort(k[wv] * T + j_all[wv])
    order = np.argsort(k[wv] * T + j_all[wv], kind="stable")
    cum = np.concatenate([[0], np.cumsum(inc[wv][order])]).astype(np.uint64)
    s = cum[np.searchsorted(wkey, k * T + j_all, "left")] - cum[np.searchsorted(wkey, k * T, "left")]
    values = np.where(wv, init[k] + s, 0).astype(np.uint64)
    coeffs = O.random_fr(seed + 1, 2)
    return dict(K=K, T=T, addrs=[a, a], values=[values, values], coeffs=coeffs, ds=[0, 1], write=1, inc=inc,
                init=init, none=0xFFFFFFFF)


def _cols_member(sess, wl, w, p, device=False):
    def col(x):
        if not device:
            return x
        return torch.from_numpy(x.view(np.int16) if x.dtype == np.uint16 else
                                x.view(np.int32) if x.dtype == np.uint32 else x).cuda()
    addr_cols = {id(a): col(a) for a in wl["addrs"]}
    acc = [(addr_cols[id(a)], Source.compact(col(v.view(np.int64)) if device else v, "u64"), c, d)
           for a, v, c, d in zip(wl["addrs"], wl["values"], wl["coeffs"], wl["ds"])]
    return ReadWriteCheckingMember(sess, acc, wl["write"], Source.compact(wl["inc"], "u64"),
                                   Source.compact(wl["init"], "u64"), wl["K"], w, cycle_rounds_first=p)


def _cols_claim(sess, wl, w):
    ev = evaluate_small(sess, wl["values"] + [wl["inc"]], w, "u64")
    return sum(c * (v + d * ev[-1]) for c, v, d in zip(wl["coeffs"], ev, wl["ds"])) % P


@pytest.mark.parametrize("K,T,shape", [(128, 1 << 16, "registers"), (1 << 20, 1 << 14, "ram_u32")])
def test_same_point_under_every_order(sess, K, T, shape):
    wl = _ram_u32_workload(5, K, T) if shape == "ram_u32" else R.columns_workload(5, K, T, shape)
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    w = O.random_fr(6, t)
    r_addr, r_cycle = O.random_fr(7, kappa), O.random_fr(8, t)
    claim = _cols_claim(sess, wl, w)
    seen = []
    for p in (0, 1, t // 2, t - 1, t):
        m = _cols_member(sess, wl, w, p)
        _rounds, fin, e, last = _run(m, RP.challenges_for(K, T, p, r_addr, r_cycle), claim)
        m.close()
        A = len(wl["addrs"])
        assert last == e * sum(c * fin[a] * (fin[A] + d * fin[A + 1]) for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"]))) % P
        seen.append((fin, e))
    assert all(x == seen[0] for x in seen)


@pytest.mark.parametrize("p", [0, 8, 16])
def test_identities_and_independent_evaluations_at_2_16_cycles(sess, p):
    K, T = 128, 1 << 16
    wl = R.columns_workload(33, K, T, "registers")
    t, kappa = 16, 7
    w = O.random_fr(34, t)
    ch = O.random_fr(35, t + kappa)
    m = _cols_member(sess, wl, w, p)
    _rounds, fin, e, last = _run(m, ch, _cols_claim(sess, wl, w))
    m.close()
    A = len(wl["addrs"])
    assert last == e * sum(c * fin[a] * (fin[A] + d * fin[A + 1]) for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"]))) % P
    r_addr, r_cycle = RP.point(K, T, p, ch)
    assert e == O.evaluate(O.eq_evals(w), r_cycle)
    for a in range(A):
        assert fin[a] == one_hot_evaluate(sess, wl["addrs"][a], K, r_addr + r_cycle, layout="address_major")[0], a
    assert fin[A + 1] == evaluate_small(sess, [wl["inc"]], r_cycle, "u64")[0]


@pytest.mark.parametrize("p", [0, 5, 10])
@pytest.mark.parametrize("device", [False, True])
def test_matches_dense_device_route(sess, p, device):
    K, T = 128, 1 << 10
    wl = R.columns_workload(K + T + p, K, T, "registers")
    t, kappa = 10, 7
    w = O.random_fr(K * 3 + T, t)
    ch = O.random_fr(K * 5 + T + p, t + kappa)
    rw = _cols_member(sess, wl, w, p, device)
    dense = RP.dense_member(sess, wl, w, p)
    claim = _cols_claim(sess, wl, w)
    bind = None
    for rnd in range(t + kappa):
        got = rw.prove_round_evals(bind, rnd, claim)
        assert got == dense.prove_round_evals(bind, rnd, claim), rnd
        bind = ch[rnd]
        claim = O.uni_evaluate(O.uni_from_evals(got), bind)
    rw.finish_rounds(bind)
    dense.finish_rounds(bind)
    want = dense.final_evals()
    assert rw.final_evals() == want[:-1]
    assert rw.eq_scalar() == want[-1]
    rw.close()
    dense.close()


def test_device_columns_u32_ram(sess):
    K, T = 1 << 20, 1 << 12
    wl = _ram_u32_workload(9, K, T)
    w, ch = O.random_fr(10, 12), O.random_fr(11, 32)
    claim = _cols_claim(sess, wl, w)
    got = []
    for device in (False, True):
        m = _cols_member(sess, wl, w, 6, device)
        got.append(_run(m, ch, claim))
        m.close()
    assert got[0] == got[1]


@pytest.mark.parametrize("inc_kind", ["i64", "i128", "s64", "s128"])
def test_compact_increments(sess, inc_kind):
    bits = 64 if inc_kind in ("i64", "s64") else 128
    K, T, accesses, write, inc, init = R.workload(17, 16, 256, 3, "registers", inc_bits=bits)
    lo, hi = -(1 << (bits - 1)) + (1 if inc_kind.startswith("s") else 0), (1 << (bits - 1)) - 1
    aw = accesses[write][0]
    for j, v in zip([j for j in range(T) if aw[j] is not None][:4], [lo, hi, -1, 0]):
        inc[j] = v % P
    val = R.val_table(K, T, accesses, write, inc, init)
    accesses = [(ad, [0 if ad[j] is None else val[ad[j]][j] for j in range(T)], c, d) for ad, _v, c, d in accesses]
    for p in (0, 4, 7):
        _lockstep(sess, (K, T, accesses, write, inc, init), O.random_fr(5, 8), None, O.random_fr(6, 12), p,
                  inc_kind=inc_kind)


def test_edge_challenges_at_the_phase_boundaries(sess):
    K, T = 4, 16
    ad = [j % K if j % 3 else None for j in range(T)]
    inc = [0 if a is None else [P - 1, (1 << 64) - 1, 1, 0][j % 4] for j, a in enumerate(ad)]
    init = [(1 << 64) - 1, 0, 1, (1 << 63)]
    val = R.val_table(K, T, [(a, None, 0, 0) for a in (ad, ad)], 1, inc, init)
    acc = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], c, d) for a, c, d in zip((ad, ad), [1, P - 1], [0, 1])]
    wl = (K, T, acc, 1, inc, init)
    edges = [0, 1, P - 1, MAX125]
    for p in range(5):
        # the edge values on the rounds on either side of each phase boundary (p - 1, p, p + 1, p + 2, p + 3)
        for e in edges:
            ch = O.random_fr(20 + p, 6)
            for r in (p - 1, p, p + 1, p + 2, p + 3):
                if 0 <= r < 6:
                    ch[r] = e
            _lockstep(sess, wl, [MAX125, P - 1, 2, 5], P - 1, ch, p)  # (no edge challenge makes an eq factor vanish)


def test_scheduler_with_a_member_of_another_size(sess):
    wl = R.workload(41, 8, 32, 3, "registers")
    K, T, accesses, write, inc, init = wl
    w, ch = O.random_fr(42, 5), O.random_fr(43, 8)
    for p in (0, 2):
        want_rounds, want_final = RP.sparse_prove(*wl, w, None, ch, p)
        rw = _member(sess, wl, w, None, p)
        tabs = [O.random_fr(44 + j, 16) for j in range(2)]
        pm = ProductMember(sess, [Polynomial.from_ints(sess, x) for x in tabs], LOW_TO_HIGH)
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


def test_prove_batch_with_a_member_of_fewer_variables(sess):
    wl = R.workload(61, 8, 64, 3, "registers")
    K, T, accesses, write, inc, init = wl
    w = O.random_fr(62, 6)
    p = 2
    rw = _member(sess, wl, w, None, p)
    tabs = [O.random_fr(63 + j, 16) for j in range(2)]
    pm = ProductMember(sess, [Polynomial.from_ints(sess, x) for x in tabs], LOW_TO_HIGH)
    c_rw = R.claimed_sum(T, accesses, inc, w)
    c_pm = sum(a * b for a, b in zip(*tabs)) % P
    k_rw, k_pm, n = 3, 5, 9
    claimed = (k_rw * c_rw + k_pm * c_pm * pow(2, n - 4, P)) % P
    got = jolt_b200.prove_batch_native([BatchMember(c_rw, k_rw, n, 0), BatchMember(c_pm, k_pm, 4, n - 4)], [rw, pm], n, 3,
                                       claimed, absorb_round=lambda r, poly: (sum(poly.coefficients) * 7 + r + 3) % P)
    want_rounds, want_final = RP.sparse_prove(*wl, w, None, got.challenges, p)
    assert rw.final_evals() == want_final
    e = rw.eq_scalar()
    member = e * sum(c * want_final[a] * (want_final[-2] + d * want_final[-1]) for a, (_x, _v, c, d) in enumerate(accesses)) % P
    assert got.member_claims[0] == member
    pf = pm.final_evals()
    assert got.final_claim == (k_rw * member + k_pm * pf[0] * pf[1]) % P
    for rnd, poly in enumerate(got.round_polynomials[:n - 4]):
        half = c_pm * pow(2, n - 4 - rnd - 1, P) % P
        assert [poly.evaluate(x) for x in range(4)] == [(k_rw * s + k_pm * half) % P for s in want_rounds[rnd]]
    rw.close()
    pm.close()


def test_refusals(sess):
    K, T = 8, 16
    wl = R.workload(51, K, T, 2, "registers")
    w = O.random_fr(52, 4)
    base = [(_addr_col(ad, K), Source.compact(np.array([v % (1 << 64) for v in vals], dtype=np.uint64)), c, d)
            for ad, vals, c, d in wl[2]]
    inc = Source.table(Polynomial.from_ints(sess, wl[4]))
    init = np.array(wl[5], dtype=np.uint64)

    def status(p, order=LOW_TO_HIGH, K_=K):
        with pytest.raises(jolt_b200.JoltB200Error) as e:
            ReadWriteCheckingMember(sess, base, 1, inc, init, K_, w, None, order, cycle_rounds_first=p)
        return e.value.status

    assert status(5) == _lib.JB_ERR_INVALID
    assert status(1 << 40) == _lib.JB_ERR_INVALID
    assert status(2, HIGH_TO_LOW) == _lib.JB_ERR_UNSUPPORTED
    assert status(5, HIGH_TO_LOW) == _lib.JB_ERR_UNSUPPORTED  # (the order is checked first, as before)
    assert status(2, K_=6) == _lib.JB_ERR_INVALID
    # the context is still usable: a member at p = 0 proves its rounds
    _lockstep(sess, wl, w, None, O.random_fr(53, 7), 0)
