"""Big-int references for the booleanity member (jb_member_create_booleanity):

    sum_{k<K} sum_{j<T} scale * eq(r_addr, k) * eq(r_cycle, j) * sum_i c_i * (ra_i(k, j)^2 - ra_i(k, j)),
    ra_i(k, j) = [addr_i(j) = k]   (addresses are ints or None).

  * dense_prove: the plain sumcheck over the materialised K T tables and the eq table - HighToLow over the
    address-major index k T + j with eq point r_addr || r_cycle, or LowToHigh over the cycle-major index j K + k with
    eq point r_cycle || r_addr;
  * sparse_prove: the member's algorithm - the address rounds from the pushforward G (bound linearly) and its copy Q
    (bound by the squared rule), then the cycle rounds from H_i(j) = F[addr_i(j)], F = eq(rho_addr, .).
Both return (round polynomials as s(0..3), [ra_i at the bound point]). Also numpy builders for the device's dense twin.
"""
import random

import numpy as np

from oracle import bn254 as O

P = O.R_MOD
HIGH_TO_LOW, LOW_TO_HIGH = 0, 1


def eq_table(w):
    """eq(w, x) over x in [0, 2^n), w[0] <-> the most significant bit of x."""
    t = [1]
    for wi in w:
        t = [v for x in t for v in (x * (1 - wi) % P, x * wi % P)]
    return t


def _interp(lo, hi, t):
    return (lo + t * (hi - lo)) % P


def _pair(order, n):
    return (lambda y: (y, y + n)) if order == HIGH_TO_LOW else (lambda y: (2 * y, 2 * y + 1))


def _bind(tab, r, order):
    n = len(tab) // 2
    pr = _pair(order, n)
    return [_interp(tab[pr(y)[0]], tab[pr(y)[1]], r) for y in range(n)]


def dense_prove(K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order):
    d = len(addrs)
    if order == HIGH_TO_LOW:
        idx, w = (lambda k, j: k * T + j), list(r_addr) + list(r_cycle)
    else:
        idx, w = (lambda k, j: j * K + k), list(r_cycle) + list(r_addr)
    tabs = []
    for col in addrs:
        t = [0] * (K * T)
        for j, a in enumerate(col):
            if a is not None:
                t[idx(a, j)] = 1
        tabs.append(t)
    e = [x * (1 if scale is None else scale) % P for x in eq_table(w)]
    tabs.append(e)
    rounds = []
    for r in ch:
        n = len(tabs[0]) // 2
        pr = _pair(order, n)
        s = [0] * 4
        for y in range(n):
            a, b = pr(y)
            for t in range(4):
                x = [_interp(tb[a], tb[b], t) for tb in tabs]
                s[t] += x[d] * sum(c * (x[i] * x[i] - x[i]) for i, c in enumerate(coeffs))
        rounds.append([v % P for v in s])
        tabs = [_bind(tb, r, order) for tb in tabs]
    return rounds, [tb[0] for tb in tabs[:d]]


def sparse_prove(K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order):
    d, lk, lt = len(addrs), K.bit_length() - 1, T.bit_length() - 1
    assert len(ch) == lk + lt
    ec = eq_table(r_cycle)
    G = [[0] * K for _ in range(d)]
    for i, col in enumerate(addrs):
        for j, a in enumerate(col):
            if a is not None:
                G[i][a] = (G[i][a] + ec[j]) % P
    Q = [g[:] for g in G]
    ea = [x * (1 if scale is None else scale) % P for x in eq_table(r_addr)]
    rounds = []
    for m in range(lk):
        r, n = ch[m], len(ea) // 2
        pr = _pair(order, n)
        s = [0] * 4
        for y in range(n):
            a, b = pr(y)
            for t in range(4):
                inner = sum(c * ((1 - t) ** 2 * Q[i][a] + t * t * Q[i][b] - _interp(G[i][a], G[i][b], t))
                            for i, c in enumerate(coeffs))
                s[t] += _interp(ea[a], ea[b], t) * inner
        rounds.append([v % P for v in s])
        ea = _bind(ea, r, order)
        G = [_bind(g, r, order) for g in G]
        Q = [[((1 - r) ** 2 * q[pr(y)[0]] + r * r * q[pr(y)[1]]) % P for y in range(n)] for q in Q]
    rho_a = ch[:lk] if order == HIGH_TO_LOW else ch[:lk][::-1]
    F = eq_table(rho_a)
    scal = ea[0]
    H = [[0 if a is None else F[a] for a in col] for col in addrs]
    e = ec[:]
    for m in range(lt):
        r, n = ch[lk + m], len(e) // 2
        pr = _pair(order, n)
        s = [0] * 4
        for y in range(n):
            a, b = pr(y)
            for t in range(4):
                inner = 0
                for i, c in enumerate(coeffs):
                    h = _interp(H[i][a], H[i][b], t)
                    inner += c * (h * h - h)
                s[t] += _interp(e[a], e[b], t) * inner
        rounds.append([v * scal % P for v in s])
        e = _bind(e, r, order)
        H = [_bind(h, r, order) for h in H]
    if lt == 0:  # T = 1: G holds ra_i(rho, 0)
        return rounds, [g[0] for g in G]
    return rounds, [h[0] for h in H]


def bound_point(K, T, ch, order):
    """(rho_addr, rho_cycle), each MSB first, of the challenges of a run."""
    lk = K.bit_length() - 1
    ra, rc = list(ch[:lk]), list(ch[lk:])
    if order == LOW_TO_HIGH:
        ra, rc = ra[::-1], rc[::-1]
    return ra, rc


def eq_scalar(K, T, r_addr, r_cycle, scale, ch, order):
    ra, rc = bound_point(K, T, ch, order)
    return (1 if scale is None else scale) * O.evaluate(eq_table(r_addr), ra) * O.evaluate(eq_table(r_cycle), rc) % P


def final_claim(finals, coeffs, eq_s):
    return eq_s * sum(c * (v * v - v) for c, v in zip(coeffs, finals)) % P


def random_columns(seed, K, T, d, none_frac=0.25):
    """Addresses below min(K, the none value of the width column_arrays picks for K)."""
    rng = random.Random(seed)
    top = min(K, 0xFF if K <= 256 else 0xFFFF)
    return [[None if rng.random() < none_frac else rng.randrange(top) for _ in range(T)] for _ in range(d)]


def column_arrays(addrs, K, kind=None):
    """uint8 (K <= 256) or uint16 numpy columns; the all-ones value is None."""
    dt = (np.uint8 if K <= 256 else np.uint16) if kind is None else kind
    none = np.iinfo(dt).max
    return [np.array([none if a is None else a for a in col], dtype=dt) for col in addrs]


def random_column_arrays(seed, K, T, d, dtype, none_frac=0.25):
    """Large random columns straight in numpy."""
    rng = np.random.default_rng(seed)
    none = np.iinfo(dtype).max
    cols = []
    for _ in range(d):
        c = rng.integers(0, min(K, int(none)), size=T, dtype=np.int64).astype(dtype)
        c[rng.random(T) < none_frac] = none
        cols.append(c)
    return cols


def dense_ra_limbs(col, K, order, one_limbs):
    """The materialised ra table of one numpy column as (K T, 4) Montgomery limbs: address-major (HighToLow) or
    cycle-major (LowToHigh)."""
    T = col.shape[0]
    none = np.iinfo(col.dtype).max
    out = np.zeros((K * T, 4), dtype=np.uint64)
    j = np.nonzero(col != none)[0]
    k = col[j].astype(np.int64)
    idx = k * T + j if order == HIGH_TO_LOW else j * K + k
    out[idx] = one_limbs
    return out
