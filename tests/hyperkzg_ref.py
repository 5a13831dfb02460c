"""Reference HyperKZG verifier for the tests, in G1 alone.

The tests generate the SRS, so they know its secret tau. The verifier's pairing check e(L, [1]_2) = e(R, [tau]_2)
holds iff L = tau R in G1 (G1 has prime order and the pairing is non-degenerate), so checking L = tau R is exact.

Derived from the fold definition (SURVEY "HyperKZG"): P_0 = the evaluation table, P_i[j] = P_(i-1)[2j] +
x (P_(i-1)[2j+1] - P_(i-1)[2j]) with x = point[ell - i], read as univariate coefficient vectors. Writing
P_i(X) = E(X^2) + X O(X^2), the fold is P_(i+1)(X^2) = (1 - x) E(X^2) + x O(X^2), and folding P_(ell-1) with point[0]
gives y = the multilinear evaluation at `point` (point[0] the most significant index bit, as O.evaluate).

Group elements are affine (x, y) integer pairs, None for the identity (oracle/bn254.py). Scalars are ints mod r."""
import numpy as np

from oracle import bn254 as O
from oracle import coracle as C

R = O.R_MOD
GEN = (1, 2)


def g_mul(P, k):
    return O.g1_scalar_mul(P, k % R)


def g_sum(terms):
    """sum_i k_i P_i over (k_i, P_i) pairs"""
    acc = None
    for k, P in terms:
        acc = O.g1_add(acc, g_mul(P, k))
    return acc


def oracle_affine(xy, inf):
    return None if inf else (O.from_mont_limbs(xy[:4], O.Q_MOD), O.from_mont_limbs(xy[4:], O.Q_MOD))


def fold_tables(evals_limbs, point_limbs):
    """P_0 .. P_(ell-1) as Montgomery limbs: P_i = P_(i-1) bound LowToHigh by point[ell - i] (C oracle)."""
    thr = C.max_threads()
    ell = point_limbs.shape[0]
    polys = [evals_limbs]
    for i in range(1, ell):
        polys.append(C.bind(polys[-1], point_limbs[ell - i], O.LOW_TO_HIGH, thr))
    return polys


def host_eval(evals_limbs, point_limbs) -> int:
    """y: the last fold, P_(ell-1) bound by point[0]."""
    last = fold_tables(evals_limbs, point_limbs)[-1]
    return C.mont_to_ints(C.bind(last, point_limbs[0], O.LOW_TO_HIGH))[0]


def oracle_open(srs_xy, evals_limbs, point_limbs, r_int, q_int):
    """The prover restated with the C oracle doing the table-sized work: com (ell - 1 affine points), w (3 affine
    points) and v[3][ell] (ints), for the challenges r and q."""
    thr = C.max_threads()
    polys = fold_tables(evals_limbs, point_limbs)
    com = [oracle_affine(*C.g1_msm_pippenger(srs_xy[: p.shape[0]], p, 0, thr)) for p in polys[1:]]
    u = [r_int % R, (-r_int) % R, r_int * r_int % R]
    v = [[C.mont_to_ints(C.eval_univariate(p, C.ints_to_mont([ui])[0]))[0] for p in polys] for ui in u]
    n = evals_limbs.shape[0]
    b = np.zeros((n, 4), dtype=np.uint64)
    qj = 1
    for p in polys:
        scaled = C.f_vec(0, 2, p, np.tile(C.ints_to_mont([qj]), (p.shape[0], 1)))
        b[: p.shape[0]] = C.f_vec(0, 0, b[: p.shape[0]], scaled)
        qj = qj * q_int % R
    w = []
    for ui in u:
        h = C.witness_polynomial(b, C.ints_to_mont([ui])[0])
        w.append(oracle_affine(*C.g1_msm_pippenger(srs_xy[: h.shape[0]], h, 0, thr)) if h.shape[0] else None)
    return com, w, v


def challenges(r):
    return [r % R, (-r) % R, r * r % R]


def consistency(point, y, v, r) -> list[bool]:
    """2 r Y[i+1] = r (1 - x) (v0[i] + v1[i]) + x (v0[i] - v1[i]), x = point[ell - 1 - i], Y = v[2] ++ [y]: one entry
    per i. Vacuous when r = 0."""
    ell = len(point)
    Y = list(v[2]) + [y % R]
    out = []
    for i in range(ell):
        x = point[ell - 1 - i]
        lhs = 2 * r * Y[i + 1]
        rhs = r * (1 - x) * (v[0][i] + v[1][i]) + x * (v[0][i] - v[1][i])
        out.append((lhs - rhs) % R == 0)
    return out


def batched_values(v, q):
    """B(u_t) = sum_j q^j v[t][j]"""
    return [sum(pow(q, j, R) * vj for j, vj in enumerate(vt)) % R for vt in v]


def kzg_per_point(tau, C0, com, w, v, r, q) -> list[bool]:
    """(tau - u_t) w_t = B_C - B(u_t) G for each t, B_C = sum_j q^j C_j."""
    BC = g_sum((pow(q, j, R), Cj) for j, Cj in enumerate([C0] + list(com)))
    Bu = batched_values(v, q)
    return [g_mul(w[t], tau - ut) == O.g1_add(BC, g_mul(GEN, -Bu[t])) for t, ut in enumerate(challenges(r))]


def kzg_batched(tau, C0, com, w, v, r, q, d0) -> bool:
    """The reference verifier's one check with d = (1, d0, d0^2):
    L = sum_j q^j (1 + d0 + d0^2) C_j + sum_t d_t u_t w_t - (sum_t d_t B(u_t)) G, R = sum_t d_t w_t, L = tau R."""
    d = [1, d0 % R, d0 * d0 % R]
    Bu = batched_values(v, q)
    u = challenges(r)
    L = g_sum([(pow(q, j, R) * sum(d), Cj) for j, Cj in enumerate([C0] + list(com))]
              + [(d[t] * u[t], w[t]) for t in range(3)] + [(-sum(d[t] * Bu[t] for t in range(3)), GEN)])
    Rt = g_sum((d[t], w[t]) for t in range(3))
    return L == g_mul(Rt, tau)


def verify(tau, C0, point, y, com, w, v, r, q, d0) -> bool:
    """Accept iff the shapes are right, every consistency equation holds and the batched KZG check passes.
    `point`: ints, point[0] the most significant variable."""
    ell = len(point)
    if ell == 0 or len(com) != ell - 1 or len(w) != 3 or len(v) != 3 or any(len(vt) != ell for vt in v):
        return False
    return all(consistency(point, y, v, r)) and kzg_batched(tau, C0, com, w, v, r, q, d0)


def expected(tau, polys, v, q, r):
    """Closed forms of a proof over a power SRS, to say which element of a failing proof is wrong: com_j = P_j(tau) G
    and w_t = ((B(tau) - B(u_t)) / (tau - u_t)) G (tau != u_t). `polys`: fold_tables' output."""
    t_m = C.ints_to_mont([tau % R])[0]
    at_tau = [C.mont_to_ints(C.eval_univariate(p, t_m))[0] for p in polys]
    com = [g_mul(GEN, a) for a in at_tau[1:]]
    B_tau = sum(pow(q, j, R) * a for j, a in enumerate(at_tau)) % R
    w = [g_mul(GEN, (B_tau - Bu) * pow((tau - ut) % R, -1, R)) for ut, Bu in zip(challenges(r), batched_values(v, q))]
    return com, w


def diagnose(tau, evals_limbs, point_limbs, C0, y, com, w, v, r, q) -> list[str]:
    """The elements of a proof that differ from their closed forms (empty if none does)."""
    polys = fold_tables(evals_limbs, point_limbs)
    bad = []
    if C0 != g_mul(GEN, C.mont_to_ints(C.eval_univariate(polys[0], C.ints_to_mont([tau % R])[0]))[0]):
        bad.append("C0")
    if y % R != host_eval(evals_limbs, point_limbs):
        bad.append("y")
    u = challenges(r)
    for t in range(3):
        for j, p in enumerate(polys):
            if v[t][j] != C.mont_to_ints(C.eval_univariate(p, C.ints_to_mont([u[t]])[0]))[0]:
                bad.append(f"v[{t}][{j}]")
    ecom, ew = expected(tau, polys, v, q, r)
    bad += [f"com[{j}]" for j in range(len(ecom)) if j >= len(com) or com[j] != ecom[j]]
    bad += [f"w[{t}]" for t in range(3) if w[t] != ew[t]]
    return bad
