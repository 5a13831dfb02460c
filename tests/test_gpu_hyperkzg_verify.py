"""Device HyperKZG proofs checked by the reference verifier (tests/hyperkzg_ref.py) over a power SRS whose secret tau
the test knows: every proof must verify with y computed on the host, and y must equal the device's own evaluation.

Covers ell = 1..24 over an SRS of exactly 2^ell bases (plain and precomputed) and over one precomputed 2^24 SRS shared by
smaller opens (which then mix the shared-window, per-window and 8-bit-table MSM paths); ell = 23 is the largest open
whose Horner scan keeps chunks of 32 (1024 blocks), ell = 24 the first with chunks of 64. Edge challenges (r in {0, 1,
p - 1, ...}, where two or three of r, -r, r^2 coincide; q in {0, 1, p - 1}), edge points and edge polynomials; tampered
device proofs must be rejected. A batched opening ties the linear combination, the three commitment paths, the three
evaluation entry points and the open together in one equation."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (G1Bases, HyperKZG, LinearTerm, Polynomial, evaluate_small, g1_jacobian_to_affine,
                       one_hot_evaluate)
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
import hyperkzg_ref as HK
import sumcheck_ref as SR
from gpu_util import rand_challenge, rand_limbs

pytestmark = pytest.mark.gpu
R = O.R_MOD
G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
TAU = O.random_fr(0x5E7A, 1)[0]
MAX_ELL = 24
MAX125 = O.from_mont_limbs([0, 0, (1 << 64) - 1, (1 << 61) - 1])   # the largest 125-bit challenge, as a field value
EVAL_MAX_ELL = 20      # Polynomial.evaluate is compared up to here


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def srs():
    """tau^i G for i < 2^24 on the host; its prefixes are the SRS of every smaller open"""
    return C.g1_powers_fast(1 << MAX_ELL, G, C.ints_to_mont([TAU])[0])


@pytest.fixture(scope="module")
def shared(sess, srs):
    """one precomputed 2^24 SRS on the device, shared by opens of every size"""
    b = G1Bases.from_affine(sess, srs).precompute()
    yield b
    b.free()


def mixed_point(ell, seed):
    return np.stack([rand_challenge(seed + i) if i % 2 else rand_limbs(seed + 50 + i, 1)[0] for i in range(ell)])


def open_and_verify(sess, bases, evals, point, r, q, d0=None):
    """Commit and open on the device; assert the proof verifies (naming the elements that differ from their closed
    forms if it does not), C0 = P(tau) G, and y = Polynomial.evaluate. Returns the proof as the verifier takes it."""
    ell = point.shape[0]
    poly = Polynomial.new(sess, evals)
    try:
        C0 = g1_jacobian_to_affine(HyperKZG.commit(bases, poly))
        proof = HyperKZG.open(bases, poly, point, lambda com: r, lambda v: q)
        y = HK.host_eval(evals, point)
        if ell <= EVAL_MAX_ELL:
            assert poly.evaluate(point) == y
    finally:
        poly.free()
    p = dict(C0=C0, point=C.mont_to_ints(point), y=y, com=[g1_jacobian_to_affine(c) for c in proof.com],
             w=[g1_jacobian_to_affine(x) for x in proof.w], v=proof.v, r=r % R, q=q % R,
             d0=O.random_fr(ell + 77, 1)[0] if d0 is None else d0)
    if not check(p):
        bad = HK.diagnose(TAU, evals, point, p["C0"], p["y"], p["com"], p["w"], p["v"], p["r"], p["q"])
        pytest.fail(f"device proof at ell = {ell} does not verify; differs from the closed forms: {bad}")
    assert C0 == HK.g_mul(HK.GEN, C.mont_to_ints(C.eval_univariate(evals, C.ints_to_mont([TAU])[0]))[0])
    return p


def check(p, **change):
    a = dict(p, **change)
    return HK.verify(TAU, a["C0"], a["point"], a["y"], a["com"], a["w"], a["v"], a["r"], a["q"], a["d0"])


def assert_tampered_rejected(p, point_matters=True):
    """y + 1, w0 <-> w1, a perturbed com_j and the reversed point must each be rejected (the point only where the
    polynomial depends on the order of its variables)"""
    ell = len(p["point"])
    assert not check(p, y=(p["y"] + 1) % R)
    if ell >= 2:
        assert not check(p, w=[p["w"][1], p["w"][0], p["w"][2]])
        if point_matters:
            assert not check(p, point=p["point"][::-1])
        for j in sorted({0, ell // 2 - 1, ell - 2}):
            assert not check(p, com=[O.g1_add(c, HK.GEN) if i == j else c for i, c in enumerate(p["com"])])


SIZES = [(1, False), (2, False), (3, True), (4, False), (8, True), (13, False), (14, False), (15, True), (16, True),
         (17, False), (19, False), (20, True), (22, False), (23, True), (24, False)]


@pytest.mark.parametrize("ell,precompute", SIZES)
def test_open_verifies_exact_srs(sess, srs, ell, precompute):
    bases = G1Bases.from_affine(sess, srs[: 1 << ell])
    try:
        if precompute:
            bases.precompute()
        r, q = O.random_fr(500 + ell, 2)
        p = open_and_verify(sess, bases, rand_limbs(400 + ell, 1 << ell), mixed_point(ell, 600 + ell), r, q)
    finally:
        bases.free()
    assert_tampered_rejected(p)


@pytest.mark.parametrize("ell", [8, 14, 17, 20, 24])
def test_open_verifies_shared_srs(sess, shared, ell):
    r, q = O.random_fr(700 + ell, 2)
    p = open_and_verify(sess, shared, rand_limbs(800 + ell, 1 << ell), mixed_point(ell, 900 + ell), r, q)
    assert_tampered_rejected(p)


EDGE_R = [0, 1, R - 1, MAX125, 1 << 128]
EDGE_Q = [0, 1, R - 1]


def edge_point(ell, seed):
    """coordinates cycling through 0, 1, p - 1 and 125-bit challenges (the largest, small, random)"""
    special = [F.to_limbs(0), F.to_limbs(1), F.to_limbs(R - 1), SR.EXTREME_CHALLENGES[1], SR.EXTREME_CHALLENGES[2]]
    return np.stack([special[i % len(special)] if i % 3 != 2 else rand_challenge(seed + i) for i in range(ell)])


@pytest.mark.parametrize("ell", [5, 15])
@pytest.mark.parametrize("r", EDGE_R, ids=["r0", "r1", "r-1", "r125", "r2^128"])
def test_edge_challenges(sess, srs, ell, r):
    bases = G1Bases.from_affine(sess, srs[: 1 << ell])
    try:
        evals = rand_limbs(1000 + ell, 1 << ell)
        for q in EDGE_Q:
            p = open_and_verify(sess, bases, evals, edge_point(ell, 1100 + ell), r, q)
            assert check(p, d0=0) and check(p, d0=R - 1)
            if r % R:      # r = 0 leaves y unbound (every u_t is 0)
                assert not check(p, y=(p["y"] + 1) % R)
    finally:
        bases.free()


def edge_polynomials(ell):
    n = 1 << ell
    ext = SR.extreme_table(1200 + ell, ell, O.LOW_TO_HIGH)
    const = np.tile(SR.extreme_limbs[6], (n, 1))
    last = np.zeros((n, 4), dtype=np.uint64)
    last[-1] = SR.extreme_limbs[3]
    return {"extreme": ext, "zero": np.zeros((n, 4), dtype=np.uint64), "constant": const, "last_only": last}


@pytest.mark.parametrize("ell", [10, 15])
@pytest.mark.parametrize("kind", ["extreme", "zero", "constant", "last_only"])
def test_edge_polynomials(sess, srs, ell, kind):
    bases = G1Bases.from_affine(sess, srs[: 1 << ell])
    try:
        evals = edge_polynomials(ell)[kind]
        r, q = O.random_fr(1300 + ell, 2)
        p = open_and_verify(sess, bases, evals, mixed_point(ell, 1400 + ell), r, q)
    finally:
        bases.free()
    if kind == "zero":
        assert p["C0"] is None and p["com"] == [None] * (ell - 1) and p["w"] == [None] * 3
        assert not check(p, C0=HK.GEN)
    else:   # a constant table folds to itself at any point, so its proof holds for every point
        assert_tampered_rejected(p, point_matters=kind != "constant")


# ---- batched openings -------------------------------------------------------------------------------------------------
def fval(v):
    return O.signed_to_fr(*v) if isinstance(v, tuple) else int(v) % R


def compact_column(kind, m, rng):
    """m entries of `kind` in small_scalars' form, extremes (negatives included) first"""
    if kind in ("u8", "u64", "i64"):
        dt = {"u8": np.uint8, "u64": np.uint64, "i64": np.int64}[kind]
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, m, dtype=dt, endpoint=True)
        ext = [info.min, info.max, 0, 1] + ([-1] if kind == "i64" else [])
        v[: len(ext)] = ext
        return v, None
    if kind == "i128":
        v = [int(rng.integers(-(1 << 62), 1 << 62)) << int(rng.integers(0, 65)) for _ in range(m)]
        v[:4] = [-(1 << 127), (1 << 127) - 1, -1, 0]
        return v, kind
    v = [(int(rng.integers(0, 1 << 63)), bool(rng.integers(0, 2))) for _ in range(m)]     # s64
    v[:4] = [(0, True), (0, False), ((1 << 64) - 1, False), ((1 << 64) - 1, True)]
    return v, kind


def one_hot_column(rng, K, T):
    none = 0xFF if K <= 255 else 0xFFFF
    col = rng.integers(0, K, T).astype(np.uint8 if none == 0xFF else np.uint16)
    col[rng.random(T) < 0.25] = none
    return col


def at_tau(values):
    """sum_i values[i] tau^i for field ints"""
    return C.mont_to_ints(C.eval_univariate(C.ints_to_mont([v % R for v in values]), C.ints_to_mont([TAU])[0]))[0]


@pytest.mark.parametrize("ell", [12, 17])
def test_batched_opening(sess, srs, ell):
    """C = sum gamma^i C_i (each term committed in its own format) and y = sum gamma^i p_i(x) (each term evaluated by
    its own entry point, a shorter term times prod (1 - x_k) over the high variables it lacks) must verify as the
    opening of Polynomial.linear_combination at x."""
    rng = np.random.default_rng(ell)
    bases = G1Bases.from_affine(sess, srs[: 1 << ell])
    point = mixed_point(ell, 1500 + ell)
    x = C.mont_to_ints(point)
    gamma = O.random_fr(1600 + ell, 1)[0]
    terms, commits, evals, scal_tau = [], [], [], []
    keep = []
    host = np.zeros((1 << ell, 4), dtype=np.uint64)      # sum_i gamma^i p_i, built on the host from dense tables

    def add(term, n_i, commit, value, tau_value, dense):
        # each entry point against the host evaluation of the term's dense table
        assert value == HK.host_eval(dense, point[ell - n_i:]), f"term {len(terms)}: evaluation"
        g = np.tile(C.ints_to_mont([pow(gamma, len(terms), R)]), (dense.shape[0], 1))
        host[: dense.shape[0]] = C.f_vec(0, 0, host[: dense.shape[0]], C.f_vec(0, 2, dense, g))
        terms.append(term)
        pad = 1
        for k in range(ell - n_i):
            pad = pad * (1 - x[k]) % R
        commits.append(commit)
        evals.append(value * pad % R)
        scal_tau.append(tau_value)

    try:
        for n_i, seed in ((ell, 1), (ell - 3, 2)):                  # field tables
            limbs = rand_limbs(1700 + ell + seed, 1 << n_i)
            poly = Polynomial.new(sess, limbs)
            keep.append(poly)
            add(LinearTerm.table(poly, pow(gamma, len(terms), R)), n_i, g1_jacobian_to_affine(bases.msm(poly)),
                poly.evaluate(point[ell - n_i:]), C.mont_to_ints(C.eval_univariate(limbs, C.ints_to_mont([TAU])[0]))[0],
                limbs)
        for kind, n_i in (("u8", ell), ("i64", ell - 1), ("u64", ell - 2), ("i128", ell), ("s64", ell - 4)):
            vals, k = compact_column(kind, 1 << n_i, rng)
            keep.append(vals)
            field = [fval(v) for v in vals]
            add(LinearTerm.compact(vals, pow(gamma, len(terms), R), kind=k), n_i,
                g1_jacobian_to_affine(bases.msm_small(vals, kind=k)),
                evaluate_small(sess, [vals], point[ell - n_i:], kinds=[k])[0], at_tau(field), C.ints_to_mont(field))
        for K, log_t, layout in ((16, ell - 4, "cycle_major"), (8, ell - 5, "address_major"), (256, ell - 8, "address_major"),
                                 (512, ell - 10, "cycle_major")):
            T = 1 << log_t
            col = one_hot_column(rng, K, T)
            keep.append(col)
            n_i = (K * T).bit_length() - 1
            hot = [(j * K + int(a)) if layout == "cycle_major" else (int(a) * T + j)
                   for j, a in enumerate(col) if int(a) < K]
            dense = np.zeros((K * T, 4), dtype=np.uint64)
            dense[hot] = C.ints_to_mont([1])[0]
            row = bases.one_hot_rows(col, K, K * T, layout=layout)
            assert row.shape[:2] == (1, 1)
            add(LinearTerm.one_hot(col, K, pow(gamma, len(terms), R), layout=layout), n_i, g1_jacobian_to_affine(row[0, 0]),
                one_hot_evaluate(sess, col, K, point[ell - n_i:], layout=layout)[0],
                sum(pow(TAU, h, R) for h in hot) % R, dense)
        for Ci, s in zip(commits, scal_tau):       # each term's own commitment is p_i(tau) G
            assert Ci == HK.g_mul(HK.GEN, s)
        combined = Polynomial.linear_combination(sess, terms)
        keep.append(combined)
        assert len(combined) == 1 << ell
        assert (combined.evals() == host).all()
        C_comb = HK.g_sum((pow(gamma, i, R), Ci) for i, Ci in enumerate(commits))
        y = sum(pow(gamma, i, R) * e for i, e in enumerate(evals)) % R
        r, q = O.random_fr(1800 + ell, 2)
        proof = HyperKZG.open(bases, combined, point, lambda com: r, lambda v: q)
        p = dict(C0=C_comb, point=x, y=y, com=[g1_jacobian_to_affine(c) for c in proof.com],
                 w=[g1_jacobian_to_affine(c) for c in proof.w], v=proof.v, r=r, q=q, d0=O.random_fr(1900 + ell, 1)[0])
        assert combined.evaluate(point) == y
        assert g1_jacobian_to_affine(bases.msm(combined)) == C_comb
        if not check(p):
            bad = HK.diagnose(TAU, host, point, C_comb, y, p["com"], p["w"], p["v"], r, q)
            pytest.fail(f"batched opening at ell = {ell} does not verify; differs from the closed forms: {bad}")
        assert not check(p, y=(y + 1) % R)
        assert not check(p, C0=O.g1_add(C_comb, HK.g_mul(HK.GEN, 1)))
    finally:
        for obj in keep:
            if isinstance(obj, Polynomial):
                obj.free()
        bases.free()
