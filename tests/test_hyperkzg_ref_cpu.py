"""The reference HyperKZG verifier (tests/hyperkzg_ref.py) on the host: honest proofs of the oracle prover verify over a
power SRS, the per-point and batched checks agree, y is the multilinear evaluation, and every single-element change
to a proof is rejected. Also pins the threaded power-SRS generator (orc_g1_powers_fast) against the sequential one."""
import numpy as np
import pytest

from oracle import bn254 as O
from oracle import coracle as C
import hyperkzg_ref as HK
from gpu_util import rand_challenge, rand_limbs

R = O.R_MOD
G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
TAU = O.random_fr(0x7A75, 1)[0]
MAX_ELL = 10


@pytest.fixture(scope="module")
def srs():
    return C.g1_powers_fast(1 << MAX_ELL, G, C.ints_to_mont([TAU])[0])


def make_proof(srs, ell, seed):
    evals = rand_limbs(seed, 1 << ell)
    point = np.stack([rand_challenge(seed + i) if i % 2 else rand_limbs(seed + 50 + i, 1)[0] for i in range(ell)])
    r, q, d0 = O.random_fr(seed + 7, 3)
    com, w, v = HK.oracle_open(srs[: 1 << ell], evals, point, r, q)
    C0 = HK.oracle_affine(*C.g1_msm_pippenger(srs[: 1 << ell], evals, 0, C.max_threads()))
    pt = C.mont_to_ints(point)
    y = HK.host_eval(evals, point)
    return dict(C0=C0, point=pt, y=y, com=com, w=w, v=v, r=r, q=q, d0=d0), evals, point


def check(p, **change):
    a = dict(p, **change)
    return HK.verify(TAU, a["C0"], a["point"], a["y"], a["com"], a["w"], a["v"], a["r"], a["q"], a["d0"])


@pytest.mark.parametrize("ell", range(1, MAX_ELL + 1))
def test_honest_proofs_verify(srs, ell):
    p, evals, point = make_proof(srs, ell, 100 + ell)
    assert p["y"] == O.evaluate(C.mont_to_ints(evals), p["point"])
    assert all(HK.consistency(p["point"], p["y"], p["v"], p["r"]))
    assert HK.kzg_per_point(TAU, p["C0"], p["com"], p["w"], p["v"], p["r"], p["q"]) == [True] * 3
    assert HK.kzg_batched(TAU, p["C0"], p["com"], p["w"], p["v"], p["r"], p["q"], p["d0"])
    assert check(p)
    # the closed forms agree with the oracle prover's group elements
    assert HK.diagnose(TAU, evals, point, p["C0"], p["y"], p["com"], p["w"], p["v"], p["r"], p["q"]) == []


def bump(P):
    return O.g1_add(P, HK.GEN)


@pytest.mark.parametrize("ell", [1, 2, 3, 6, 10])
def test_every_single_change_is_rejected(srs, ell):
    p, evals, point = make_proof(srs, ell, 300 + ell)
    assert check(p)
    bad = []

    def expect_reject(what, **change):
        if check(p, **change):
            bad.append(what)
        # the per-point checks localise a change to a group element or an evaluation
        a = dict(p, **change)
        if what.startswith(("com", "w", "v", "C0", "q")) and all(
                HK.kzg_per_point(TAU, a["C0"], a["com"], a["w"], a["v"], a["r"], a["q"])):
            bad.append(what + " (per point)")

    expect_reject("C0", C0=bump(p["C0"]))
    for j in range(ell - 1):
        expect_reject(f"com[{j}]", com=[bump(c) if i == j else c for i, c in enumerate(p["com"])])
    for t in range(3):
        expect_reject(f"w[{t}]", w=[bump(x) if i == t else x for i, x in enumerate(p["w"])])
        for j in range(ell):
            v = [list(vt) for vt in p["v"]]
            v[t][j] = (v[t][j] + 1) % R
            expect_reject(f"v[{t}][{j}]", v=v)
    expect_reject("y", y=(p["y"] + 1) % R)
    if ell >= 2:
        expect_reject("reversed point", point=p["point"][::-1])
        sw = list(p["point"])
        sw[0], sw[1] = sw[1], sw[0]
        expect_reject("swapped point", point=sw)
    expect_reject("point[-1] + 1", point=p["point"][:-1] + [(p["point"][-1] + 1) % R])
    expect_reject("r", r=(p["r"] + 1) % R)
    expect_reject("-r", r=(-p["r"]) % R)
    if ell >= 2:    # at ell = 1 there is one polynomial and q never enters
        expect_reject("q", q=(p["q"] + 1) % R)
    if ell >= 2:    # at ell = 1 the three quotients are the same constant
        expect_reject("w0 <-> w1", w=[p["w"][1], p["w"][0], p["w"][2]])
    expect_reject("shape", com=p["com"] + [HK.GEN])
    assert bad == []


@pytest.mark.parametrize("r", [0, 1, R - 1])
def test_coinciding_challenges(srs, r):
    """r = 0 (u all 0: the consistency equations are vacuous, the KZG checks still bind every v), r = 1 and p - 1
    (two of r, -r, r^2 coincide)."""
    ell = 4
    evals = rand_limbs(900, 1 << ell)
    point = rand_limbs(901, ell)
    q, d0 = O.random_fr(902, 2)
    com, w, v = HK.oracle_open(srs[: 1 << ell], evals, point, r, q)
    C0 = HK.oracle_affine(*C.g1_msm_pippenger(srs[: 1 << ell], evals, 0, 1))
    pt, y = C.mont_to_ints(point), HK.host_eval(evals, point)
    assert HK.verify(TAU, C0, pt, y, com, w, v, r, q, d0)
    for t in range(3):
        for j in range(ell):
            vv = [list(vt) for vt in v]
            vv[t][j] = (vv[t][j] + 1) % R
            assert not HK.verify(TAU, C0, pt, y, com, w, vv, r, q, d0)
    assert HK.verify(TAU, C0, pt, (y + 1) % R, com, w, v, r, q, d0) == (r == 0)


@pytest.mark.parametrize("tau", [1, R - 1, O.random_fr(0x51, 1)[0]])
@pytest.mark.parametrize("n", [1, 2, 3, 1000, 1 << 12])
def test_fast_powers_match_sequential(tau, n):
    t = C.ints_to_mont([tau])[0]
    assert (C.g1_powers_fast(n, G, t) == C.g1_powers(n, G, t)).all()


def test_fast_powers_of_zero():
    out = C.g1_powers_fast(5, G, C.ints_to_mont([0])[0])
    assert (out[0] == G).all() and not out[1:].any()


def test_fast_powers_sampled_2_20():
    """the 16-bit-window table (n >= 2^16) at sampled indices up to 2^20"""
    n = 1 << 20
    out = C.g1_powers_fast(n, G, C.ints_to_mont([TAU])[0])
    for i in [0, 1, 2, 1023, 1024, 1025, 65535, 65536, 777777, n - 1]:
        want = O.g1_scalar_mul(HK.GEN, pow(TAU, i, R))
        assert HK.oracle_affine(out[i], False) == want, i
