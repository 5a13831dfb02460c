"""EqPolynomial::evals on the device vs the oracle (mirrors eq.rs:496-756, 238-263)."""
import numpy as np
import pytest

import jolt_b200
from jolt_b200 import EqPolynomial
from oracle import bn254 as O
from oracle import coracle as C
from gpu_util import rand_limbs
import sumcheck_ref as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 8, 11, 12, 13, 17])
@pytest.mark.parametrize("scaled", [False, True])
def test_eq_matches_oracle(sess, n, scaled):
    r = rand_limbs(300 + n, n)
    sc = rand_limbs(77, 1)[0] if scaled else None
    got = EqPolynomial.evals(sess, r, sc).evals()
    want = C.eq_evals(r, sc, threads=4 if n > 12 else 1)
    assert got.shape == want.shape and (got == want).all()


def test_eq_sums_to_one_and_pointwise(sess):
    n = 12
    r_int = O.random_fr(9, n)
    tab = EqPolynomial.evals(sess, C.ints_to_mont(r_int)).to_ints()
    assert sum(tab) % O.R_MOD == 1
    for x in (0, 1, 1234, (1 << n) - 1):
        v = 1
        for i in range(n):
            bit = (x >> (n - 1 - i)) & 1          # r[0] <-> MSB
            v = v * (r_int[i] if bit else 1 - r_int[i]) % O.R_MOD
        assert tab[x] == v


def test_eq_aligned_block_is_slice(sess):
    n = 14
    r = rand_limbs(5, n)
    full = EqPolynomial.evals(sess, r).evals()
    for start, size in ((0, 1 << 11), (3 << 11, 1 << 11), (3 << 12, 1 << 12), (1 << 13, 1 << 13), (0, 1 << 14), (7, 1)):
        got = EqPolynomial.evals_for_aligned_block(sess, r, start, size).evals()
        assert (got == full[start:start + size]).all()


@pytest.mark.parametrize("kind", ["full254", "challenge125", "mixed"])
def test_eq_2pow22(sess, kind):
    """BASELINE size; the point as full elements, as 125-bit challenges [0,0,lo,hi] (the 4-row product
    path, mod.rs:172-184), and mixed."""
    n = 22
    r = rand_limbs(0xE0, n)
    if kind != "full254":
        r[:, 0] = 0
        r[:, 1] = 0
        r[:, 3] &= np.uint64((1 << 61) - 1)
    if kind == "mixed":
        r[12] = rand_limbs(5, 1)[0]
    got = EqPolynomial.evals(sess, r).evals()
    want = C.eq_evals(r, None, threads=C.max_threads())
    assert (got == want).all()


@pytest.mark.parametrize("n", [17, 22])
@pytest.mark.parametrize("kind", ["full", "challenge"])
def test_eq_extreme_point_coordinates(sess, n, kind):
    """coordinates 0, 1, p - 1 and limb-extreme values as full elements, and extreme 125-bit [0,0,lo,hi]
    challenges, shuffled over the point"""
    r = S.extreme_point(0xE0E + n, n, kind)
    got = EqPolynomial.evals(sess, r).evals()
    want = C.eq_evals(r, None, threads=C.max_threads())
    assert (got == want).all()
