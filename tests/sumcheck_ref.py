"""Reference inputs and answers for the sumcheck edge tests: full-range and limb-extreme Montgomery tables, extreme
challenges, the sum-of-products oracle, and closed-form round polynomials of sign-tensor tables (for sizes the C
oracle cannot reach). Everything here is pinned against Python big ints by tests/test_sumcheck_ref_cpu.py."""
import math

import numpy as np

from oracle import bn254 as O
from oracle import coracle as C

P = O.R_MOD
MASK64 = (1 << 64) - 1
_P_LIMBS = [(P >> (64 * k)) & MASK64 for k in range(4)]


def int_to_limbs(v: int) -> np.ndarray:
    """A raw 256-bit integer as 4 little-endian u64 limbs (no Montgomery encoding)."""
    return np.array([(v >> (64 * k)) & MASK64 for k in range(4)], dtype=np.uint64)


def raw_ints(a: np.ndarray) -> list[int]:
    """The raw integers held in (n, 4) limbs."""
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
    return [O.mont_raw(row) for row in a]


def below_p(a: np.ndarray) -> np.ndarray:
    """Row-wise raw value < p, vectorised over (n, 4) limbs."""
    lt = np.zeros(a.shape[0], dtype=bool)
    eq = np.ones(a.shape[0], dtype=bool)
    for k in (3, 2, 1, 0):
        pk = np.uint64(_P_LIMBS[k])
        lt |= eq & (a[:, k] < pk)
        eq &= a[:, k] == pk
    return lt


def rand_limbs_full(seed: int, n: int) -> np.ndarray:
    """n canonical Montgomery elements uniform over all of [0, p): 254-bit draws, rejected when >= p. Unlike
    rand_limbs (which stays below 2^253) about a third of them lie in [2^253, p)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty((n, 4), dtype=np.uint64)
    filled = 0
    while filled < n:
        want = n - filled
        a = rng.integers(0, 1 << 64, size=(want + want // 3 + 16, 4), dtype=np.uint64)
        a[:, 3] &= np.uint64(MASK64 >> 2)
        a = a[below_p(a)][:want]
        out[filled:filled + a.shape[0]] = a
        filled += a.shape[0]
    return out


R_MONT = (1 << 256) % P      # Montgomery one
EXTREME_RAW = [
    0, 1, 2,
    P - 1, P - 2, P - (1 << 32),
    (1 << 253) - 1, 1 << 253, (1 << 64) - 1,
    ((P >> 224) << 224) - 1,  # the largest value below p with every 32-bit word 0xFFFFFFFF except the top one
    R_MONT, R_MONT * R_MONT % P,
]
extreme_limbs = np.stack([int_to_limbs(v) for v in EXTREME_RAW])


def extreme_pairs(rotate: int = 0) -> list[tuple[int, int]]:
    """Every ordered pair (lo, hi) of extreme_limbs indices; `rotate` shifts which hi meets which lo, so that tables
    of one product put different extremes side by side."""
    k = len(EXTREME_RAW)
    return [(a, (b + rotate) % k) for a in range(k) for b in range(k)]


def extreme_table(seed: int, n: int, order: int, rotate: int = 0) -> np.ndarray:
    """2^n Montgomery limbs: every ordered pair of extreme_limbs as one (lo, hi) pair of the first round under
    `order` (LowToHigh pairs (2i, 2i+1), HighToLow pairs (i, i + 2^(n-1))), repeated at four places spread over the
    table when it is long enough (so several blocks of a multi-block pass meet them); the rest is rand_limbs_full."""
    t = rand_limbs_full(seed, 1 << n)
    half = 1 << (n - 1)
    pairs = extreme_pairs(rotate)
    assert len(pairs) <= half, "table too short for every extreme pair"
    bases = [0] if half < 4 * len(pairs) else [0, half // 4, half // 2, half - len(pairs)]
    for base in bases:
        for i, (a, b) in enumerate(pairs):
            y = base + i
            lo, hi = (2 * y, 2 * y + 1) if order == O.LOW_TO_HIGH else (y, y + half)
            t[lo] = extreme_limbs[a]
            t[hi] = extreme_limbs[b]
    return t


# ---- challenges (raw Montgomery limbs) --------------------------------------------------------------------
EXTREME_CHALLENGES = np.stack([
    int_to_limbs(0),                                            # zero: the 4-row [0, 0, lo, hi] product with lo = hi = 0
    np.array([0, 0, MASK64, (1 << 61) - 1], dtype=np.uint64),   # the largest 125-bit challenge
    np.array([0, 0, 1, 0], dtype=np.uint64),
    int_to_limbs(R_MONT),                                       # one (full-width path)
    int_to_limbs(P - 1),
])


def extreme_point(seed: int, n: int, kind: str = "full", zero: bool = True) -> np.ndarray:
    """n point coordinates (eq points), shuffled so the extremes land on both sides of an inner / outer split.
    "full": canonical 0 (unless zero=False), 1 and p - 1, the limb-extreme values and the extreme challenges, then
    random elements; "challenge": 125-bit [0, 0, lo, hi] coordinates with extreme and random lo / hi."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind == "full":
        special = [int_to_limbs(0)] if zero else []
        special += [int_to_limbs(R_MONT), np.array(O.to_mont_limbs(P - 1), dtype=np.uint64)]
        special += [v for v in extreme_limbs[2:] if O.mont_raw(v) != R_MONT] + list(EXTREME_CHALLENGES[1:3])
    else:
        lo_hi = [(0, 0), (MASK64, (1 << 61) - 1), (1, 0), (0, (1 << 61) - 1), (MASK64, 0), (0, 1)]
        special = [np.array([0, 0, lo, hi], dtype=np.uint64) for lo, hi in lo_hi]
    pts = special[:max(n - 4, 0)]
    for k in range(n - len(pts)):
        pts.append(C.rand_challenge(seed + k) if kind != "full" or k % 2 else rand_limbs_full(seed + k, 1)[0])
    return np.stack([pts[i] for i in rng.permutation(n)])


def extreme_challenge(rnd: int, seed: int = 0) -> np.ndarray:
    """Round `rnd`'s challenge: the extreme challenges interleaved with random 125-bit and 254-bit ones."""
    k = rnd % 7
    if k < len(EXTREME_CHALLENGES):
        return EXTREME_CHALLENGES[k].copy()
    if k == 5:
        return C.rand_challenge(seed * 1000 + rnd)
    return rand_limbs_full(seed * 1000 + rnd, 1)[0]


# ---- sum of products --------------------------------------------------------------------------------------
def sop_round_evals(tables: list[np.ndarray], factors: int, order: int, threads: int = 1) -> list[int]:
    """Round evaluations (t = 0..factors) of sum_k prod_j f_{k*factors+j}: the mod-p sum over terms of the C
    oracle's product round evaluations (the round polynomial is linear in the terms)."""
    acc = [0] * (factors + 1)
    for k in range(len(tables) // factors):
        ev = C.mont_to_ints(C.product_round_evals(tables[k * factors:(k + 1) * factors], factors, order, threads))
        acc = [(a + e) % P for a, e in zip(acc, ev)]
    return acc


# ---- sign-tensor tables: closed-form sumchecks ------------------------------------------------------------
# f_j(x) = c * prod_i g_{j,i}(x_i) with g_{j,i}(0), g_{j,i}(1) in {+1, -1} and x_0 the MSB of the table index
# (r[0] <-> MSB, as eq.rs). c is chosen so its Montgomery limbs are p - 1; -c then has limbs 1.
C_SIGN = (P - 1) * pow(1 << 256, -1, P) % P
LIMBS_POS = int_to_limbs(P - 1)
LIMBS_NEG = int_to_limbs(1)


def sign_patterns(seed: int, n: int, m: int, terms: int = 1) -> list[list[list[tuple[int, int]]]]:
    """terms x m tables x n variables of (g(0), g(1)) sign pairs with prod_j g_{j,i}(0) == prod_j g_{j,i}(1) for
    every variable i, so that no factor sum_b prod_j g_{j,i}(b) vanishes (else every round polynomial would be
    zero). Every term gets the same per-variable products, so the terms of a sum of products cannot cancel."""
    rng = np.random.Generator(np.random.PCG64(seed))
    target = rng.choice([-1, 1], size=n)
    out = []
    for _ in range(terms):
        pats = [[None] * n for _ in range(m)]
        for i in range(n):
            s = rng.choice([-1, 1], size=(m, 2))
            s[m - 1, 0] = target[i] * math.prod(int(v) for v in s[:m - 1, 0])
            s[m - 1, 1] = target[i] * math.prod(int(v) for v in s[:m - 1, 1])
            for j in range(m):
                pats[j][i] = (int(s[j, 0]), int(s[j, 1]))
        out.append(pats)
    return out


def sign_table(pat: list[tuple[int, int]]) -> np.ndarray:
    """The 2^n Montgomery limbs of c * prod_i g_i(x_i): entries are limbs p - 1 (+c) or 1 (-c)."""
    sign = np.ones(1, dtype=np.int8)
    for g0, g1 in pat:            # x_0 first: np.kron's left factor is the most significant index bit
        sign = np.kron(sign, np.array([g0, g1], dtype=np.int8))
    out = np.empty((sign.size, 4), dtype=np.uint64)
    out[:] = LIMBS_NEG
    out[sign > 0] = LIMBS_POS
    return out


def _g(pair: tuple[int, int], r: int) -> int:
    g0, g1 = pair
    return (g0 + r * (g1 - g0)) % P


def sign_sumcheck(terms: list[list[list[tuple[int, int]]]], order: int, challenges: list[int]) -> dict:
    """Closed-form run of the sumcheck of sum_k prod_j f_{k,j} for sign-tensor tables (terms[k][j] is table
    (k, j)'s pattern; a product member is one term). Round k binds variable k (HighToLow) or n-1-k (LowToHigh).
    s_k(t) = sum_terms c^D * prod_j [prod_{bound i} g_{j,i}(r_i)] * g_{j,v}(t) * prod_{free i != v} sum_b prod_j g_{j,i}(b).
    Returns the round evaluations at t = 0..D, the final evaluations of every table and the final claim."""
    D = len(terms[0])
    n = len(terms[0][0])
    cD = pow(C_SIGN, D, P)
    var = (lambda k: k) if order == O.HIGH_TO_LOW else (lambda k: n - 1 - k)
    bound: dict[int, int] = {}
    rounds = []
    for k in range(n):
        v = var(k)
        evals = [0] * (D + 1)
        for tm in terms:
            fixed = cD
            for i, r in bound.items():
                for j in range(D):
                    fixed = fixed * _g(tm[j][i], r) % P
            for i in range(n):
                if i != v and i not in bound:
                    fixed = fixed * (math.prod(tm[j][i][0] for j in range(D)) + math.prod(tm[j][i][1] for j in range(D))) % P
            for t in range(D + 1):
                e = fixed
                for j in range(D):
                    e = e * _g(tm[j][v], t) % P
                evals[t] = (evals[t] + e) % P
        rounds.append(evals)
        if k < len(challenges):
            bound[v] = challenges[k] % P
    finals = []
    for tm in terms:
        for j in range(D):
            f = C_SIGN
            for i in range(n):
                f = f * _g(tm[j][i], bound[i]) % P
            finals.append(f)
    claim = 0
    for k in range(len(terms)):
        claim = (claim + math.prod(finals[k * D:(k + 1) * D])) % P
    return dict(rounds=rounds, finals=finals, final_claim=claim)


def trimmed_coeffs(evals: list[int]) -> list[int]:
    """Coefficients of the round polynomial through evals as the batch engine reports it (trailing zero
    coefficients dropped down to degree 1, prover.rs:163-168)."""
    c = O.uni_from_evals(evals)
    while len(c) > 2 and c[-1] == 0:
        c.pop()
    return c
