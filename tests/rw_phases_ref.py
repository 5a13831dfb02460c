"""ORACLE (test infrastructure, NOT product code) for the read-write checking member with its address rounds after
p = cycle_rounds_first cycle rounds (jb_member_create_read_write_phases).

The relation is rw_ref's; the rounds bind, LSB first, cycle bits 0 .. p-1, then address bits 0 .. kappa-1, then cycle
bits p .. t-1: LowToHigh over the index x = (j >> p) K 2^p + k 2^p + (j mod 2^p). Workloads are rw_ref's.

Two references that must agree on every round polynomial (as s(0..3)) and every final value [ra_0 .. ra_{A-1}, Val,
inc]:
  * `dense_prove`: materialises ra_a, Val, inc and the eq table in the mixed layout and runs the sumcheck on them;
  * `sparse_prove`: a restatement of the member's algorithm - p cycle rounds over entries per (row, key) as rw_ref's,
    then the address rounds over entries per (key, row), a key absent at a row taking ra = 0 and Val = the ve of its
    own last entry at an earlier row (else its bound init value), each row weighted by eq, then dense tables over the
    remaining rows. At p = t it is rw_ref.sparse_prove.
`dense_member` is the device route: an ExpressionMember over the materialised mixed-layout tables."""
from __future__ import annotations

import bisect

import numpy as np

from jolt_b200 import LOW_TO_HIGH, EqPolynomial, ExpressionMember, Polynomial
from jolt_b200 import field as F

from oracle import bn254 as O
import rw_ref as R

P = O.R_MOD


def _interp(lo, hi, t):
    return (lo + t * (hi - lo)) % P


def mixed_index(K, T, p):
    """[(k, j)] in the order of x = (j >> p) K 2^p + k 2^p + (j mod 2^p)."""
    lo_n = 1 << p
    return [(k, jh * lo_n + jl) for jh in range(T >> p) for k in range(K) for jl in range(lo_n)]


def point(K, T, p, challenges):
    """(r_addr, r_cycle), each MSB first, of the challenges of a p-first order."""
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    return challenges[p:p + kappa][::-1], (challenges[:p] + challenges[p + kappa:])[::-1]


def challenges_for(K, T, p, r_addr, r_cycle):
    """The challenges under which a p-first order ends at (r_addr, r_cycle) (both MSB first)."""
    cyc, adr = r_cycle[::-1], r_addr[::-1]
    return cyc[:p] + adr + cyc[p:]


def _dense_rounds(tabs, A, cs, ds, challenges):
    """Rounds over tables [ra_0 .. ra_{A-1}, Val, inc, eq]: s(0..3) per round, then the bound tables."""
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
    return rounds, tabs


def dense_prove(K, T, accesses, write, inc, init, w, scale, challenges, p):
    A = len(accesses)
    val = R.val_table(K, T, accesses, write, inc, init)
    e = O.eq_evals(w, scale)
    idx = mixed_index(K, T, p)
    tabs = [[1 if ad[j] == k else 0 for k, j in idx] for ad, _v, _c, _d in accesses]
    tabs += [[val[k][j] for k, j in idx], [inc[j] % P for _k, j in idx], [e[j] for _k, j in idx]]
    cs = [c for _a, _v, c, _d in accesses]
    ds = [d for _a, _v, _c, d in accesses]
    rounds, tabs = _dense_rounds(tabs, A, cs, ds, challenges)
    return rounds, [tb[0] for tb in tabs[:A + 2]]


def sparse_prove(K, T, accesses, write, inc, init, w, scale, challenges, p):
    A = len(accesses)
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    if K == 1:
        p = t  # no address rounds: every order is the same
    cs = [c for _a, _v, c, _d in accesses]
    ds = [d for _a, _v, _c, d in accesses]
    aw = accesses[write][0]
    rows = []  # rows[j] = {key: [ra list, val, vs, ve]}
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
    E = O.eq_evals(w, scale)  # the eq table over the rows, bound alongside (degree 1 per variable: as a split factor)
    rounds = []

    def sides(lo, hi, k):
        L, H = lo.get(k), hi.get(k)
        if L is None:
            b = H[2]
            L = [[0] * A, b, b, b]
        if H is None:
            b = L[3]
            H = [[0] * A, b, b, b]
        return L, H

    # phase 1: p cycle rounds, adjacent rows paired
    for m in range(p):
        s = [0, 0, 0, 0]
        for y in range(len(rows) // 2):
            lo, hi = rows[2 * y], rows[2 * y + 1]
            for tt in range(4):
                et = _interp(E[2 * y], E[2 * y + 1], tt)
                it = _interp(incs[2 * y], incs[2 * y + 1], tt)
                for k in set(lo) | set(hi):
                    L, H = sides(lo, hi, k)
                    v = _interp(L[1], H[1], tt)
                    s[tt] += et * sum(cs[a] * _interp(L[0][a], H[0][a], tt) * (v + ds[a] * it) for a in range(A))
        rounds.append([x % P for x in s])
        r = challenges[m]
        new = []
        for y in range(len(rows) // 2):
            lo, hi = rows[2 * y], rows[2 * y + 1]
            new.append({k: [[_interp(L[0][a], H[0][a], r) for a in range(A)], _interp(L[1], H[1], r), L[2], H[3]]
                        for k in sorted(set(lo) | set(hi)) for L, H in [sides(lo, hi, k)]})
        rows = new
        incs = [_interp(incs[2 * y], incs[2 * y + 1], r) for y in range(len(incs) // 2)]
        E = [_interp(E[2 * y], E[2 * y + 1], r) for y in range(len(E) // 2)]
    # phase 2: address-major, keys[k] = (sorted rows, {row: [ra, val, ve]}); absent (k, i) -> ve of k's last row < i,
    # else k's bound init value
    Tp = len(rows)
    keys = [dict() for _ in range(K)]
    for i, row in enumerate(rows):
        for k, (ra, v, _vs, ve) in row.items():
            keys[k][i] = [ra, v, ve]
    ini = [x % P for x in init]

    def at(kd, srt, ik, i):
        if i in kd:
            return kd[i]
        pos = bisect.bisect_left(srt, i)
        b = kd[srt[pos - 1]][2] if pos else ik
        return [[0] * A, b, b]

    for m in range(kappa):
        s = [0, 0, 0, 0]
        new = []
        r = challenges[p + m]
        for y in range(len(keys) // 2):
            lo, hi = keys[2 * y], keys[2 * y + 1]
            slo, shi = sorted(lo), sorted(hi)
            kd = {}
            for i in sorted(set(lo) | set(hi)):
                L, H = at(lo, slo, ini[2 * y], i), at(hi, shi, ini[2 * y + 1], i)
                for tt in range(4):
                    v = _interp(L[1], H[1], tt)
                    s[tt] += E[i] * sum(cs[a] * _interp(L[0][a], H[0][a], tt) * (v + ds[a] * incs[i]) for a in range(A))
                kd[i] = [[_interp(L[0][a], H[0][a], r) for a in range(A)], _interp(L[1], H[1], r), _interp(L[2], H[2], r)]
            new.append(kd)
        rounds.append([x % P for x in s])
        keys = new
        ini = [_interp(ini[2 * y], ini[2 * y + 1], r) for y in range(len(ini) // 2)]
    # phase 3: dense tables over the remaining rows
    (kd,) = keys
    srt = sorted(kd)
    ent = [at(kd, srt, ini[0], i) for i in range(Tp)]
    tabs = [[x[0][a] for x in ent] for a in range(A)] + [[x[1] for x in ent], incs, E]
    more, tabs = _dense_rounds(tabs, A, cs, ds, challenges[p + kappa:])
    return rounds + more, [tb[0] for tb in tabs[:A + 2]]


def dense_member(sess, wl, w, p):
    """The device expression member (jolt_b200, not the oracle) over the tables of rw_ref.columns_workload materialised
    in the mixed layout, with a replicated eq table."""
    K, T = wl["K"], wl["T"]
    keys = np.arange(K, dtype=np.int64)[:, None]
    aw = wl["addrs"][wl["write"]]
    M = np.zeros((K, T), dtype=np.uint64)
    wv = aw != wl["none"]
    M[aw[wv].astype(np.int64), np.arange(T)[wv]] = wl["inc"][wv]
    val = wl["init"][:, None] + np.cumsum(M, axis=1, dtype=np.uint64) - M

    def mixed(kt):  # (K, T) -> the mixed layout: axes (j >> p, k, j mod 2^p)
        return kt.reshape(K, T >> p, 1 << p).transpose(1, 0, 2).reshape(-1)

    tabs = [Polynomial.from_small(sess, mixed(((a.astype(np.int64)[None, :] == keys) & (a != wl["none"])[None, :])
                                              .astype(np.uint8)), "u8") for a in wl["addrs"]]
    tabs.append(Polynomial.from_small(sess, mixed(val), "u64"))
    tabs.append(Polynomial.from_small(sess, mixed(np.tile(wl["inc"], (K, 1))), "u64"))
    eq = EqPolynomial.evals(sess, F.ints_to_limbs(w)).evals()  # (T, 4) limbs
    eqm = np.broadcast_to(eq.reshape(T >> p, 1, 1 << p, 4), (T >> p, K, 1 << p, 4)).reshape(-1, 4)
    tabs.append(Polynomial.new(sess, np.ascontiguousarray(eqm)))
    A = len(wl["addrs"])
    monos = [(c, [a, A, A + 2]) for a, c in enumerate(wl["coeffs"])]
    monos += [(c, [a, A + 1, A + 2]) for a, (c, d) in enumerate(zip(wl["coeffs"], wl["ds"])) if d]
    return ExpressionMember(sess, tabs, monos, order=LOW_TO_HIGH)
