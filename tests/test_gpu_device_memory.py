"""Every entry point gives back the device memory it allocates for itself: after a call, and after the handles it
returned are freed, the device's default memory pool (which the context allocates from, stream-ordered, and which never
releases memory) holds exactly as much as before - on success and on refusals the device finds after the call has
allocated. A leaked buffer would stay allocated for the life of the process."""
import ctypes
import os

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (EqPolynomial, ExpressionMember, G1Bases, HyperKZG, LinearTerm, LtPolynomial, Polynomial, Source,
                       _lib, evaluate_small, one_hot_evaluate, one_hot_pushforward)
from oracle import bn254 as O
from gpu_util import rand_limbs

pytestmark = pytest.mark.gpu

G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
N = 1 << 14                               # bases of the SRS
BAD_ADDRESS = "one-hot: an address >= K that is not the none value"
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7      # cuda.h (CUDA 12.9)


class PoolUsage:
    """The bytes of a device's default memory pool in use, read through the driver API."""

    def __init__(self, device: int):
        self.cu = ctypes.CDLL("libcuda.so.1")
        assert self.cu.cuInit(0) == 0
        dev = ctypes.c_int()
        assert self.cu.cuDeviceGet(ctypes.byref(dev), device) == 0
        self.pool = ctypes.c_void_p()
        assert self.cu.cuDeviceGetDefaultMemPool(ctypes.byref(self.pool), dev) == 0
        self.cu.cuMemPoolGetAttribute.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]

    def used(self) -> int:
        v = ctypes.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, ctypes.byref(v)) == 0
        return v.value


@pytest.fixture(scope="module")
def env():
    conf = os.environ.get("PYTORCH_CUDA_ALLOC_CONF", "") + os.environ.get("PYTORCH_ALLOC_CONF", "")
    if "cudaMallocAsync" in conf:
        pytest.skip("torch's allocator shares the default memory pool (PYTORCH_CUDA_ALLOC_CONF selects cudaMallocAsync)")
    sess = jolt_b200.Session(0)
    plain = G1Bases.generate_multiples(sess, G, N)          # bases[i] = (i + 1) G
    pre = G1Bases.generate_multiples(sess, G, N).precompute()
    yield sess, PoolUsage(sess.device), plain, pre
    sess.close()


def _release(made):
    for m in made or []:
        if hasattr(m, "free"):
            m.free()
        else:
            m.close()


def assert_gives_back(sess, pool, call):
    """call() once to warm up (grow-once buffers: the partial sums, an SRS's small table), then again between two
    readings of the pool; call returns what it made (tables, bases, members), freed before the second reading."""
    _release(call())
    sess.synchronize()
    before = pool.used()
    _release(call())
    sess.synchronize()
    assert pool.used() == before


def assert_refusal_gives_back(sess, pool, call, status, message):
    """As assert_gives_back for a call that the device refuses after the call has allocated."""
    def refused():
        with pytest.raises(jolt_b200.JoltB200Error, match=message) as e:
            call()
        assert e.value.status == status
    assert_gives_back(sess, pool, refused)


def _discard(f, *args, **kw):
    """Calls f for its effect on the pool: what it returns holds no handle."""
    f(*args, **kw)


def _ints(seed, n):
    return O.random_fr(seed, n)


def _addresses(seed, T, K, dtype=np.uint8, bad=False):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, K, size=T).astype(dtype)
    a[::7] = np.iinfo(dtype).max                     # cycles that touched no address
    if bad:
        a[T // 2] = K                                # not the none value, >= K
    return a


# ---- MSMs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["plain", "precomputed"])
def test_msm_g1(env, which):
    sess, pool, plain, pre = env
    bases = plain if which == "plain" else pre
    sc = rand_limbs(0xD3E0, N)
    assert_gives_back(sess, pool, lambda: _discard(bases.msm, sc))
    assert_gives_back(sess, pool, lambda: _discard(bases.msm, sc[:1000], offset=17))


@pytest.mark.parametrize("kind", ["u8_binary", "u8", "i64"])
def test_msm_g1_small(env, kind):
    sess, pool, plain, _ = env
    rng = np.random.default_rng(0xD3E1)
    if kind == "u8_binary":   # all <= 1 after the u8 max pass: the selection sum
        values = rng.integers(0, 2, size=N).astype(np.uint8)
    elif kind == "u8":        # the max pass, then the general path
        values = rng.integers(0, 256, size=N).astype(np.uint8)
    else:
        values = rng.integers(-(1 << 62), 1 << 62, size=N).astype(np.int64)
    assert_gives_back(sess, pool, lambda: _discard(plain.msm_small, values))


def test_msm_g1_rows(env):
    sess, pool, plain, _ = env
    sc = rand_limbs(0xD3E2, 4 << 10)
    assert_gives_back(sess, pool, lambda: _discard(plain.msm_rows, sc, 4, kind="fr"))
    # u8 rows of N entries go 2^14 rows to a pass: 2^14 + 1 rows end in a lone row, committed as a single MSM
    rows = (1 << 14) + 1
    values = np.zeros(rows * N, dtype=np.uint8)
    values[::4099] = 3
    assert_gives_back(sess, pool, lambda: _discard(plain.msm_rows, values, rows))


def test_msm_g1_one_hot_rows(env):
    sess, pool, plain, _ = env
    cols = [_addresses(0xD3E3 + i, 1 << 10, 16) for i in range(3)]
    assert_gives_back(sess, pool, lambda: _discard(plain.one_hot_rows, cols, 16, 1 << 7))
    bad = [cols[0], _addresses(0xD3E4, 1 << 10, 16, bad=True)]
    assert_refusal_gives_back(sess, pool, lambda: plain.one_hot_rows(bad, 16, 1 << 7), _lib.JB_ERR_INVALID, BAD_ADDRESS)
    assert plain.one_hot_rows(cols, 16, 1 << 7).shape == (3, 128, 12)


def test_msm_g1_device_and_table(env):
    sess, pool, plain, pre = env
    poly = Polynomial.new(sess, rand_limbs(0xD3E5, N))
    out = np.zeros(12, dtype=np.uint64)
    d_scalars = ctypes.c_void_p(poly.device_ptr())

    def device():
        sess.check(sess.lib.jb_msm_g1_device(sess.h, pre.handle, 0, d_scalars, N, out.ctypes.data_as(_lib.c_u64p)))
    assert_gives_back(sess, pool, device)
    assert_gives_back(sess, pool, lambda: _discard(plain.msm, poly))
    poly.free()


def test_srs_upload_and_generate(env):
    sess, pool, plain, _ = env
    xy = plain.affine()[:1 << 10]
    one = np.array(O.to_mont_limbs(1, O.Q_MOD), dtype=np.uint64)
    xyz = np.concatenate([xy, np.tile(one, (xy.shape[0], 1))], axis=1)
    assert_gives_back(sess, pool, lambda: [G1Bases.from_jacobian(sess, xyz)])
    assert_gives_back(sess, pool, lambda: [G1Bases.generate_multiples(sess, G, 1 << 12)])


def test_g1_batch_add(env):
    sess, pool, plain, _ = env
    sets = [[100, 2000, 5000, 9000], [7], [], [300, 4000, 11000]]
    assert_gives_back(sess, pool, lambda: _discard(plain.batch_add, sets))


# ---- HyperKZG -----------------------------------------------------------------------------------------------------
def _open_raw(sess, bases, poly, pt, r_fn, q_fn):
    ell = pt.shape[0]
    com = np.zeros((ell - 1, 12), dtype=np.uint64)
    w = np.zeros((3, 12), dtype=np.uint64)
    v = np.zeros((3, ell, 4), dtype=np.uint64)
    cb_r, cb_q = _lib.HKZG_R_FN(r_fn), _lib.HKZG_Q_FN(q_fn)
    p = lambda a: a.ctypes.data_as(_lib.c_u64p)  # noqa: E731
    sess.check(sess.lib.jb_hyperkzg_open(sess.h, bases.handle, poly.handle, p(pt), ell, ctypes.cast(cb_r, ctypes.c_void_p),
                                         ctypes.cast(cb_q, ctypes.c_void_p), None, p(com), p(w), p(v)))


def _challenge(value):
    def fn(_user, _vals, _n, out):
        for i, limb in enumerate(value):
            out[i] = limb
        return 0
    return fn


def test_hyperkzg_open(env):
    sess, pool, _, pre = env
    ell = 10
    poly = Polynomial.new(sess, rand_limbs(0xD3E6, 1 << ell))
    pt = rand_limbs(0xD3E7, ell)
    assert_gives_back(sess, pool, lambda: _discard(HyperKZG.open, pre, poly, pt, lambda com: 5, lambda v: 7))
    ok = _challenge([5, 0, 0, 0])
    assert_refusal_gives_back(sess, pool, lambda: _open_raw(sess, pre, poly, pt, lambda *a: 1, ok),
                              _lib.JB_ERR_INVALID, "challenge_r callback failed")
    assert_refusal_gives_back(sess, pool, lambda: _open_raw(sess, pre, poly, pt, ok, _challenge([2**64 - 1] * 4)),
                              _lib.JB_ERR_INVALID, "challenge q not canonical")
    _open_raw(sess, pre, poly, pt, ok, ok)
    poly.free()


# ---- tables -------------------------------------------------------------------------------------------------------
def _terms(sess, poly, bad=False):
    K, T = 4, 64
    return [LinearTerm.table(poly, 3),
            LinearTerm.compact(np.arange(K * T, dtype=np.uint16), 5),
            LinearTerm.one_hot(_addresses(0xD3E8, T, K, bad=bad), K, 7)]


def test_linear_combination_and_vmp(env):
    sess, pool, _, _ = env
    poly = Polynomial.new(sess, rand_limbs(0xD3E9, 256))
    left = Polynomial.new(sess, rand_limbs(0xD3EA, 16))
    lc = lambda bad=False: [Polynomial.linear_combination(sess, _terms(sess, poly, bad))]  # noqa: E731
    vmp = lambda bad=False: [Polynomial.vector_matrix_product(sess, _terms(sess, poly, bad), left, 16)]  # noqa: E731
    assert_gives_back(sess, pool, lc)
    assert_gives_back(sess, pool, vmp)
    assert_refusal_gives_back(sess, pool, lambda: lc(True), _lib.JB_ERR_INVALID, BAD_ADDRESS)
    assert_refusal_gives_back(sess, pool, lambda: vmp(True), _lib.JB_ERR_INVALID, BAD_ADDRESS)
    _release(lc() + vmp())
    poly.free()
    left.free()


def test_structured_tables_above_one_block(env):
    sess, pool, _, _ = env
    r = rand_limbs(0xD3EB, 13)    # > EQ_BLOCK_VARS = 11: the prefix tables are built for the call
    assert_gives_back(sess, pool, lambda: [EqPolynomial.evals(sess, r)])
    assert_gives_back(sess, pool, lambda: [LtPolynomial.evals(sess, r)])


def test_evaluations_and_pushforward(env):
    sess, pool, _, _ = env
    n = 10
    cols = [np.arange(1 << n, dtype=np.uint16), np.arange(1 << n, dtype=np.int64) - 300, np.ones(1 << n, dtype=np.uint8)]
    assert_gives_back(sess, pool, lambda: _discard(evaluate_small, sess, cols, _ints(0xD3EC, n)))
    K, T = 16, 1 << n
    addr = [_addresses(0xD3ED, T, K), _addresses(0xD3EE, T, K)]
    point = _ints(0xD3EF, n + 4)
    assert_gives_back(sess, pool, lambda: _discard(one_hot_evaluate, sess, addr, K, point))
    assert_refusal_gives_back(sess, pool, lambda: one_hot_evaluate(sess, [addr[0], _addresses(0xD3F0, T, K, bad=True)],
                                                                   K, point), _lib.JB_ERR_INVALID, BAD_ADDRESS)
    assert_gives_back(sess, pool, lambda: one_hot_pushforward(sess, addr, K, _ints(0xD3F1, n)))
    assert len(one_hot_evaluate(sess, addr, K, point)) == 2


def test_vec_op(env):
    sess, pool, _, _ = env
    a, b = rand_limbs(0xD3F2, 1000), rand_limbs(0xD3F3, 1000)
    assert_gives_back(sess, pool, lambda: _discard(sess.vec_op, 0, 2, a, b))


def test_expression_member_over_sources(env):
    sess, pool, _, _ = env
    K, T = 4, 256
    srcs = lambda: [Source.compact(np.arange(T, dtype=np.uint16)),  # noqa: E731
                    Source.one_hot(_addresses(0xD3F4, T, K), K, _ints(0xD3F5, 2))]
    assert_gives_back(sess, pool, lambda: [ExpressionMember.from_sources(sess, srcs(), [(1, [0, 1])])])
