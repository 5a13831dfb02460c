"""ORACLE (test infrastructure, NOT product code) for the read-write checking member (jb_member_create_read_write).

The relation, index x = k T + j (cycle in the low bits), bound LowToHigh:
    sum_{k<K} sum_{j<T} scale eq(w, j) sum_a c_a ra_a(k, j) (Val(k, j) + d_a inc(j))
with ra_a(k, j) = [addr_a(j) = k] and Val(k, j) = init(k) + sum_{j' < j, addr_w(j') = k} inc(j').

Two references that must agree on every round polynomial (as s(0..3)) and every final value:
  * `dense_prove`: materialises ra_a, Val, inc and the eq table over K T and runs the sumcheck on them;
  * `sparse_prove`: a restatement of the member's algorithm - entries per (row, key) with val, vs (Val before the
    row's block) and ve (Val after it), adjacent rows paired with a missing key taking its partner's boundary value, the
    eq factor kept split - then the dense address rounds.
A workload is (K, T, accesses, write, inc, init): accesses = [(addr, values, c, d)] with addr[j] an int or None (no
access), values[j] = Val(addr[j], j) (the precondition; `workload` builds them), ints mod P throughout."""
from __future__ import annotations

import numpy as np

from jolt_b200 import LOW_TO_HIGH, EqPolynomial, ExpressionMember, Polynomial
from jolt_b200 import field as F

from oracle import bn254 as O

P = O.R_MOD


def val_table(K, T, accesses, write, inc, init):
    """Val[k][j] by the definition."""
    aw = accesses[write][0]
    val = []
    for k in range(K):
        row, cur = [], init[k] % P
        for j in range(T):
            row.append(cur)
            if aw[j] == k:
                cur = (cur + inc[j]) % P
        val.append(row)
    return val


def workload(seed, K, T, A, shape="registers", none_frac=0.1, inc_bits=64, local=False):
    """A random workload satisfying the precondition. shape: "registers" (A distinct columns, the last one the write)
    or "ram" (one column read and written: A = 2)."""
    rng = np.random.default_rng(seed)
    hi = K - 1 if K in (256, 65536) else K  # (the all-ones value of the column width is the none value)

    def column():
        if local:
            a = np.cumsum(rng.integers(-2, 3, T)) % hi
        else:
            a = rng.integers(0, hi, T)
        return [None if rng.random() < none_frac else int(x) for x in a]

    cols = [column()] if shape == "ram" else [column() for _ in range(A)]
    addrs = [cols[0], cols[0]] if shape == "ram" else cols
    write = len(addrs) - 1
    inc = [0 if addrs[write][j] is None else
           (int.from_bytes(rng.bytes(inc_bits // 8), "little") - (1 << (inc_bits - 1))) % P for j in range(T)]
    init = [int(x) for x in rng.integers(0, 1 << 62, K)]
    val = val_table(K, T, [(a, None, 0, 0) for a in addrs], write, inc, init)
    coeffs = O.random_fr(seed + 11, len(addrs))
    accesses = []
    for a, ad in enumerate(addrs):
        values = [0 if ad[j] is None else val[ad[j]][j] for j in range(T)]
        accesses.append((ad, values, coeffs[a], 1 if a == write else 0))
    return K, T, accesses, write, inc, init


def claimed_sum(T, accesses, inc, w, scale=None):
    """sum_j scale eq(w, j) sum_a c_a (v_a(j) + d_a inc(j)) over the accessing cycles: the relation's value."""
    e = O.eq_evals(w, scale)
    tot = 0
    for ad, values, c, d in accesses:
        for j in range(T):
            if ad[j] is not None:
                tot += e[j] * c * (values[j] + d * inc[j])
    return tot % P


def _interp(lo, hi, t):
    return (lo + t * (hi - lo)) % P


def _round_from_q(q0, q1, qinf, scalar, wc):
    """s(t) = l(t) q(t), t = 0..3, for q of degree 2 and the eq factor l(t) = scalar ((1 - wc) + t (2 wc - 1))."""
    out = []
    for t in range(4):
        q = (q0 + (q1 - q0 - qinf) * t + qinf * t * t) % P
        out.append(scalar * ((1 - wc) + t * (2 * wc - 1)) % P * q % P)
    return out


def dense_prove(K, T, accesses, write, inc, init, w, scale, challenges):
    """(round evaluations s(0..3) per round, final values [ra_0 .. ra_{A-1}, Val, inc]) with challenges[i] bound after
    round i (len(challenges) = log2(K T))."""
    A = len(accesses)
    val = val_table(K, T, accesses, write, inc, init)
    e = O.eq_evals(w, scale)
    ra = [[1 if ad[j] == k else 0 for k in range(K) for j in range(T)] for ad, _v, _c, _d in accesses]
    tabs = ra + [[val[k][j] for k in range(K) for j in range(T)], [inc[j] % P for _k in range(K) for j in range(T)],
                 [e[j] for _k in range(K) for j in range(T)]]
    cs = [c for _a, _v, c, _d in accesses]
    ds = [d for _a, _v, _c, d in accesses]
    rounds = []
    for r in challenges:
        n = len(tabs[0]) // 2
        s = [0, 0, 0, 0]
        for i in range(n):
            for t in range(4):
                x = [_interp(tb[2 * i], tb[2 * i + 1], t) for tb in tabs]
                s[t] += x[A + 2] * sum(cs[a] * x[a] * (x[A] + ds[a] * x[A + 1]) for a in range(A))
        rounds.append([v % P for v in s])
        tabs = [[_interp(tb[2 * i], tb[2 * i + 1], r) for i in range(n)] for tb in tabs]
    return rounds, [tb[0] for tb in tabs[:A + 2]]


def sparse_prove(K, T, accesses, write, inc, init, w, scale, challenges):
    """The member's algorithm; same result as dense_prove."""
    A = len(accesses)
    t = T.bit_length() - 1
    cs = [c for _a, _v, c, _d in accesses]
    ds = [d for _a, _v, _c, d in accesses]
    aw = accesses[write][0]
    # the unbound matrix: rows[j] = {key: [ra list, val, vs, ve]}
    rows = []
    for j in range(T):
        row = {}
        for a, (ad, values, _c, _d) in enumerate(accesses):
            k = ad[j]
            if k is None:
                continue
            if k not in row:
                v = values[j] % P
                row[k] = [[0] * A, v, v, (v + inc[j]) % P if aw[j] == k else v]
            row[k][0][a] = 1
        rows.append(row)
    incs = [x % P for x in inc]
    scalar = 1 if scale is None else scale % P
    rounds = []

    def sides(lo, hi, k):
        L = lo.get(k)
        H = hi.get(k)
        if L is None:
            b = H[2]
            L = [[0] * A, b, b, b]
        if H is None:
            b = L[3]
            H = [[0] * A, b, b, b]
        return L, H

    for m in range(t):
        wc = w[t - 1 - m]
        E = O.eq_evals(w[:t - 1 - m])
        q = [0, 0, 0]
        for y in range(len(rows) // 2):
            lo, hi = rows[2 * y], rows[2 * y + 1]
            for k in set(lo) | set(hi):
                L, H = sides(lo, hi, k)
                for idx, (S, ic) in enumerate(((L, incs[2 * y]), (H, incs[2 * y + 1]))):
                    q[idx] += E[y] * sum(cs[a] * S[0][a] * (S[1] + ds[a] * ic) for a in range(A))
                q[2] += E[y] * sum(cs[a] * (H[0][a] - L[0][a]) * ((H[1] - L[1]) + ds[a] * (incs[2 * y + 1] - incs[2 * y]))
                                   for a in range(A))
        rounds.append(_round_from_q(q[0] % P, q[1] % P, q[2] % P, scalar, wc))
        r = challenges[m]
        new = []
        for y in range(len(rows) // 2):
            lo, hi = rows[2 * y], rows[2 * y + 1]
            row = {}
            for k in sorted(set(lo) | set(hi)):
                L, H = sides(lo, hi, k)
                row[k] = [[_interp(L[0][a], H[0][a], r) for a in range(A)], _interp(L[1], H[1], r), L[2], H[3]]
            new.append(row)
        rows = new
        incs = [_interp(incs[2 * y], incs[2 * y + 1], r) for y in range(len(incs) // 2)]
        scalar = scalar * ((1 - wc) * (1 - r) + wc * r) % P
    # address phase: dense K-entry tables
    (row,) = rows
    ra = [[row[k][0][a] if k in row else 0 for k in range(K)] for a in range(A)]
    val = [row[k][1] if k in row else init[k] % P for k in range(K)]
    inc_r = incs[0]
    for r in challenges[t:]:
        n = len(val) // 2
        s = [0, 0, 0, 0]
        for i in range(n):
            for tt in range(4):
                v = _interp(val[2 * i], val[2 * i + 1], tt)
                s[tt] += scalar * sum(cs[a] * _interp(ra[a][2 * i], ra[a][2 * i + 1], tt) * (v + ds[a] * inc_r)
                                      for a in range(A))
        rounds.append([x % P for x in s])
        ra = [[_interp(x[2 * i], x[2 * i + 1], r) for i in range(n)] for x in ra]
        val = [_interp(val[2 * i], val[2 * i + 1], r) for i in range(n)]
    return rounds, [x[0] for x in ra] + [val[0], inc_r]


# ---- large workloads (numpy) and the dense device route they are compared with ----------------------------------


def columns_workload(seed, K, T, shape, none_frac=0.05):
    """Address columns (u8 / u16, all-ones = none), u64 value columns v_a(j) = Val(addr_a(j), j) (0 at none), a u64 inc
    column (0 where the write is none) and u64 init, built with numpy: non-negative increments keep every Val in u64."""
    rng = np.random.default_rng(seed)
    dt = np.uint8 if K <= 256 else np.uint16
    none = np.iinfo(dt).max
    hi = min(K, int(none))
    ncols = 1 if shape == "ram" else 3
    cols = []
    for _ in range(ncols):
        a = rng.integers(0, hi, T).astype(dt)
        a[rng.random(T) < none_frac] = none
        cols.append(a)
    addrs = [cols[0], cols[0]] if shape == "ram" else cols
    write = len(addrs) - 1
    aw = addrs[write]
    wv = aw != none
    inc = np.where(wv, rng.integers(0, 1 << 32, T), 0).astype(np.uint64)
    init = rng.integers(0, 1 << 40, K).astype(np.uint64)
    # Val(k, j) = init(k) + the increments of the earlier writes to k: prefix sums over the writes sorted by (k, j)
    j_all = np.arange(T, dtype=np.int64)
    wkey = aw[wv].astype(np.int64) * T + j_all[wv]
    order = np.argsort(wkey, kind="stable")
    wkey = wkey[order]
    cum = np.concatenate([[0], np.cumsum(inc[wv][order].astype(np.uint64))]).astype(np.uint64)
    values = []
    for ad in addrs:
        valid = ad != none
        k = ad.astype(np.int64)
        q = k * T + j_all
        s = cum[np.searchsorted(wkey, q, "left")] - cum[np.searchsorted(wkey, k * T, "left")]
        values.append(np.where(valid, init[np.minimum(k, K - 1)] + s, 0).astype(np.uint64))
    coeffs = O.random_fr(seed + 1, len(addrs))
    ds = [1 if a == write else 0 for a in range(len(addrs))]
    return dict(K=K, T=T, addrs=addrs, values=values, coeffs=coeffs, ds=ds, write=write, inc=inc, init=init, none=none)


def dense_member(sess, wl, w):
    """The device expression member (jolt_b200, not the oracle) over the materialised K T tables (index k T + j) with a replicated eq table."""
    K, T = wl["K"], wl["T"]
    keys = np.arange(K, dtype=np.int64)[:, None]
    aw = wl["addrs"][wl["write"]]
    # Val over the matrix: init + exclusive prefix sums of each address's increments
    M = np.zeros((K, T), dtype=np.uint64)
    wv = aw != wl["none"]
    M[aw[wv].astype(np.int64), np.arange(T)[wv]] = wl["inc"][wv]
    val = wl["init"][:, None] + np.cumsum(M, axis=1, dtype=np.uint64) - M
    # (at K = 2^16 the none value 0xFFFF is also a key: it must not count as an access)
    tabs = [Polynomial.from_small(sess, ((a.astype(np.int64)[None, :] == keys) & (a != wl["none"])[None, :])
                                  .astype(np.uint8).reshape(-1), "u8") for a in wl["addrs"]]
    tabs.append(Polynomial.from_small(sess, val.reshape(-1), "u64"))
    tabs.append(Polynomial.from_small(sess, np.tile(wl["inc"], K), "u64"))
    eq = EqPolynomial.evals(sess, F.ints_to_limbs(w)).evals()
    tabs.append(Polynomial.new(sess, np.tile(eq, (K, 1))))
    A = len(wl["addrs"])
    monos = [(c, [a, A, A + 2]) for a, c in enumerate(wl["coeffs"])]
    monos += [(c, [a, A + 1, A + 2]) for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"])) if d]
    return ExpressionMember(sess, tabs, monos, order=LOW_TO_HIGH)


