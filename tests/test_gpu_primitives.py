"""The device primitives every kernel is built from, tested directly against Python big integers: the BN254 Fr / Fq
Montgomery arithmetic (canonical and lazy forms), the 544-bit deferred-reduction accumulators and reduce_wide17, the
lane bins (pf_flush, bins_to_fr_kernel), the XYZZ group law and fq_inverse. tests/native/primitives_harness.cu
includes the library headers unmodified and is built here with the library's nvcc flags, so it sees the same code
generation. Every comparison is bit-exact, on raw limbs: a Montgomery operand is the integer its limbs hold.

The inputs are the ones where carry chains and stated bounds fail: values in [2^253, p), lazy operands up to 2p - 1,
hi4 multipliers up to the largest canonical value with two zero low limbs, accumulators at 2^544 - 1 and group-law
operands that are equal or opposite only projectively (different ZZ / ZZZ)."""
import ctypes
import os
import pathlib
import random
import shutil
import subprocess

import numpy as np
import pytest

from oracle import bn254 as O
from oracle import coracle as C

ROOT = pathlib.Path(__file__).resolve().parents[1]
CSRC = ROOT / "jolt_b200" / "csrc"
# the library's flags (jolt_b200/csrc/Makefile): the carry chains are only as right as what ptxas makes of them
NVFLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-O2,-Wall",
           "-cudart", "static"]

FIELDS = [pytest.param(0, O.R_MOD, id="fr"), pytest.param(1, O.Q_MOD, id="fq")]
R = 1 << 256
W17 = 1 << 544
N_RANDOM = 1 << 18
N_BLOCK = 1 << 14

# field_op_kernel's operations (primitives_harness.cu)
ADD, SUB, MUL, SQR, NEG, DBL, FROM_MONT, TO_MONT, EQ, SUB_LAZY, MUL_LAZY, MUL_HI4_LAZY, MUL_HI4, INVERSE = range(14)
W_REG, W_SMEM, W_BW1, W_BW2, W_BW4, W_BW8 = range(6)
G_ADD_AFFINE, G_ADD, G_DOUBLE = range(3)


def find_nvcc():
    default = "/usr/local/cuda/bin/nvcc"
    return shutil.which("nvcc") or (default if os.path.exists(default) else None)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = find_nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    so = tmp_path_factory.mktemp("primitives") / "libprimitives_harness.so"
    cmd = [nvcc, *NVFLAGS, "-shared", "-I", str(CSRC), str(ROOT / "tests/native/primitives_harness.cu"), "-o", str(so), "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, f"primitives harness does not build against the current headers:\n{res.stderr[-4000:]}"
    return Harness(ctypes.CDLL(str(so)))


class Harness:
    """The harness's extern "C" entry points over numpy arrays; each asserts the call returned cudaSuccess."""

    def __init__(self, lib):
        self.lib = lib
        vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.ph_field_op.argtypes = [i, i, vp, vp, vp, sz]
        lib.ph_wide_acc.argtypes = [i, vp, vp, vp, i, i, vp, sz]
        lib.ph_reduce_wide17.argtypes = [i, vp, vp, sz]
        lib.ph_bins_to_fr.argtypes = [vp, vp, sz]
        lib.ph_pf_flush.argtypes = [vp, vp, vp, sz, vp, sz]
        lib.ph_g1.argtypes = [i, vp, vp, vp, vp, sz]

    @staticmethod
    def _p(a):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data

    def _ok(self, err, what):
        assert err == 0, f"{what}: cudaError {err}"

    def field_op(self, fld, op, a, b=None):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        b = np.ascontiguousarray(a if b is None else b, dtype=np.uint64)
        out = np.zeros_like(a)
        self._ok(self.lib.ph_field_op(fld, op, self._p(a), self._p(b), self._p(out), a.shape[0]), f"field op {op}")
        return out

    def wide_acc(self, mode, seed, a, b, reps=1):
        """seed: (n, 17) u32; a, b: (n, count, 8) u32."""
        seed, a, b = (np.ascontiguousarray(x, dtype=np.uint32) for x in (seed, a, b))
        n, count = a.shape[0], a.shape[1]
        out = np.zeros_like(seed)
        self._ok(self.lib.ph_wide_acc(mode, self._p(seed), self._p(a), self._p(b), count, reps, self._p(out), n),
                 f"wide acc mode {mode}")
        return out

    def reduce_wide17(self, fld, acc):
        """acc: (n, 17) u32 words; passed word-major, so reduce_wide17 reads it at stride n."""
        acc_t = np.ascontiguousarray(np.asarray(acc, dtype=np.uint32).T)
        out = np.zeros((acc.shape[0], 4), dtype=np.uint64)
        self._ok(self.lib.ph_reduce_wide17(fld, self._p(acc_t), self._p(out), acc.shape[0]), "reduce_wide17")
        return out

    def bins_to_fr(self, lanes):
        lanes = np.ascontiguousarray(lanes, dtype=np.uint64)
        out = np.zeros((lanes.shape[0], 4), dtype=np.uint64)
        self._ok(self.lib.ph_bins_to_fr(self._p(lanes), self._p(out), lanes.shape[0]), "bins_to_fr")
        return out

    def pf_flush(self, emit, key, val, nbins):
        emit, key = (np.ascontiguousarray(x, dtype=np.uint32) for x in (emit, key))
        val = np.ascontiguousarray(val, dtype=np.uint64)
        bins = np.zeros((nbins, 8), dtype=np.uint64)
        self._ok(self.lib.ph_pf_flush(self._p(emit), self._p(key), self._p(val), emit.shape[0], self._p(bins), nbins),
                 "pf_flush")
        return bins

    def g1(self, op, a, b, neg=None):
        a, b = (np.ascontiguousarray(x, dtype=np.uint64) for x in (a, b))
        neg = np.ascontiguousarray(np.zeros(a.shape[0]) if neg is None else neg, dtype=np.uint32)
        out = np.zeros_like(a)
        self._ok(self.lib.ph_g1(op, self._p(a), self._p(b), self._p(neg), self._p(out), a.shape[0]), f"g1 op {op}")
        return out


# ---- integers <-> words ------------------------------------------------------------------------------------------

def to_ints(a, bits=64):
    """(n, w) little-endian words -> object array of the n integers they hold."""
    a = np.asarray(a)
    out = np.zeros(a.shape[0], dtype=object)
    for k in range(a.shape[1] - 1, -1, -1):
        out = (out << bits) | a[:, k].astype(object)
    return out


def to_words(vals, words=4, bits=64):
    """Integers -> (n, words) little-endian words (u64 for 64-bit words, u32 for 32-bit ones)."""
    v = np.array(list(vals), dtype=object)
    mask, dt = (1 << bits) - 1, np.uint64 if bits == 64 else np.uint32
    return np.stack([((v >> (bits * k)) & mask).astype(dt) for k in range(words)], axis=1)


def rand_range(seed, n, lo, hi):
    """n integers uniform on [lo, hi)."""
    rng = random.Random(seed)
    return np.array([rng.randrange(lo, hi) for _ in range(n)], dtype=object)


def canonical_edges(p):
    top = ((p >> 224) - 1) << 224 | ((1 << 224) - 1)  # every word all ones, the top word one below p's
    vals = [0, 1, 2, p - 1, p - 2, p - (1 << 32), (1 << 253) - 1, 1 << 253, (1 << 64) - 1, top,
            R % p, R * R % p, R * R * R % p]
    assert all(0 <= v < p for v in vals)
    return vals


def lazy_edges(p):
    return canonical_edges(p) + [p, p + 1, 2 * p - 2, 2 * p - 1]


def operands(p, edges, seed, extra=()):
    """(a, b) object arrays: every ordered pair of edges, then N_RANDOM pairs uniform on [0, p), N_BLOCK on
    [2^253, p) and N_BLOCK on each (lo, hi) range of `extra`, a and b drawn independently."""
    k = len(edges)
    a = [np.repeat(np.array(edges, dtype=object), k)]
    b = [np.tile(np.array(edges, dtype=object), k)]
    blocks = [(0, p, N_RANDOM), (1 << 253, p, N_BLOCK)] + [(lo, hi, N_BLOCK) for lo, hi in extra]
    for j, (lo, hi, n) in enumerate(blocks):
        a.append(rand_range(seed + 2 * j, n, lo, hi))
        b.append(rand_range(seed + 2 * j + 1, n, lo, hi))
    return np.concatenate(a), np.concatenate(b)


def mismatches(got, want):
    bad = np.nonzero(got != want)[0]
    return f"{bad.size} mismatches, first at {bad[:5].tolist()}"


def cios(a, b, p, bits=256):
    """The exact word-serial Montgomery product of integers a, b (b < 2^bits): (a b + m p) / 2^bits with
    m = -a b p^-1 mod 2^bits, the one value the carry chains compute when nothing is lost."""
    rb = 1 << bits
    pinv = pow(p, -1, rb)
    t = a * b
    return (t + ((-t * pinv) % rb) * p) >> bits


# ---- build (no GPU) -----------------------------------------------------------------------------------------------

def test_harness_builds_against_current_headers(harness):
    """The harness compiles and links against field.cuh, ec.cuh and lane_bins.cuh as they stand, so a header change
    that breaks it fails here, without a GPU."""
    for name in ("ph_field_op", "ph_wide_acc", "ph_reduce_wide17", "ph_bins_to_fr", "ph_pf_flush", "ph_g1"):
        assert hasattr(harness.lib, name)


# ---- field: canonical forms ---------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_canonical_ops(harness, fld, p):
    """add, sub, mul, sqr, neg (-0 = 0), dbl, from_mont, to_mont on canonical operands: each result equals the big-int
    value, which is below p, so the device result is canonical too."""
    a, b = operands(p, canonical_edges(p), 100 + fld)
    da, db = to_words(a), to_words(b)
    rinv = pow(R, -1, p)
    want = {
        ADD: (a + b) % p,
        SUB: (a - b) % p,
        MUL: a * b * rinv % p,
        SQR: a * a * rinv % p,
        NEG: (-a) % p,
        DBL: 2 * a % p,
        FROM_MONT: a * rinv % p,
        TO_MONT: a * R % p,
    }
    for op, w in want.items():
        got = to_ints(harness.field_op(fld, op, da, db))
        assert (got == w).all(), f"field {fld} op {op}: {mismatches(got, w)}"
        assert (got < p).all()


@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_equality_and_is_zero(harness, fld, p):
    """operator== and is_zero compare all eight words: pairs equal, differing in one bit of any one word, and the
    ordered edge pairs (whose diagonal is equal)."""
    edges = canonical_edges(p)
    a = np.concatenate([np.repeat(np.array(edges, dtype=object), len(edges)), rand_range(7 + fld, 4096, 0, p)])
    b = np.concatenate([np.tile(np.array(edges, dtype=object), len(edges)), a[len(edges) ** 2:]])
    rng = np.random.default_rng(fld)
    flip = rng.integers(0, 256, size=b.size)
    flip[::2] = -1                                          # half stay equal
    b = np.array([x if f < 0 else x ^ (1 << int(f)) for x, f in zip(b, flip)], dtype=object)
    out = harness.field_op(fld, EQ, to_words(a), to_words(b))
    assert ((out[:, 0] & np.uint64(0xffffffff)) == (a == b)).all(), "operator=="
    assert ((out[:, 0] >> np.uint64(32)) == (a == 0)).all(), "is_zero"


# ---- field: lazy forms --------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_lazy_ops(harness, fld, p):
    """fp_sub_lazy is exactly a - b + p, in (0, 2p) for canonical operands; fp_mul_lazy on operands up to 2p - 1 is the
    exact Montgomery product, congruent to a b R^-1 and below 2p."""
    a, b = operands(p, lazy_edges(p), 200 + fld, extra=[(p, 2 * p)])
    b = np.where(b >= p, b - p, b)                           # the subtrahend stays canonical: b <= a + p
    got = to_ints(harness.field_op(fld, SUB_LAZY, to_words(a), to_words(b)))
    assert (got == a - b + p).all(), mismatches(got, a - b + p)
    canon = a < p
    assert ((got[canon] > 0) & (got[canon] < 2 * p)).all()

    a, b = operands(p, lazy_edges(p), 300 + fld, extra=[(p, 2 * p), (0, 2 * p)])
    got = to_ints(harness.field_op(fld, MUL_LAZY, to_words(a), to_words(b)))
    want = cios(a, b, p)
    assert (got == want).all(), mismatches(got, want)
    assert (got < 2 * p).all()
    assert ((got - a * b * pow(R, -1, p)) % p == 0).all()


def hi4_edges(p):
    """hi4 values h (the multiplier is h 2^128) up to the largest canonical one, (p - 1) >> 128."""
    top = (p - 1) >> 128
    return [0, 1, 2, top, top - 1, (1 << 125) - 1, 1 << 124, (1 << 64) - 1, 1 << 64]


@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_hi4_products(harness, fld, p):
    """fp_mul_hi4_lazy / fp_mul_hi4 with operands up to 2p - 1 and multipliers up to the largest canonical value whose
    two low limbs are zero: the lazy form is the exact product of montmul(a, h 2^128), below 2p; the reduced one is
    canonical for every a in [0, 2p), which is what bind_pair assumes of fp_mul_hi4(fp_sub_lazy(hi, lo), r)."""
    ae, he = lazy_edges(p), hi4_edges(p)
    top = (p - 1) >> 128
    a = np.concatenate([np.repeat(np.array(ae, dtype=object), len(he)),       # every lazy edge times every hi4 edge
                        rand_range(400 + fld, N_RANDOM, 0, p), rand_range(401 + fld, N_BLOCK, 1 << 253, p),
                        rand_range(402 + fld, 2 * N_BLOCK, p, 2 * p)])
    n = a.size - len(ae) * len(he)
    h = np.concatenate([np.tile(np.array(he, dtype=object), len(ae)),      # uniform hi4, then 125-bit challenges
                        rand_range(410 + fld, n // 2, 0, top + 1), rand_range(411 + fld, n - n // 2, 0, 1 << 125)])
    b = h << 128
    assert (b < p).all()
    da, db = to_words(a), to_words(b)
    lazy = to_ints(harness.field_op(fld, MUL_HI4_LAZY, da, db))
    want = cios(a, h, p, bits=128)
    assert (lazy == want).all(), mismatches(lazy, want)
    assert (want == cios(a, b, p)).all()                     # rows 0..3 of the full product are identities
    assert (lazy < 2 * p).all()
    full = to_ints(harness.field_op(fld, MUL_HI4, da, db))
    reduced = a * b * pow(R, -1, p) % p
    assert (full == reduced).all(), mismatches(full, reduced)


# ---- wide accumulators --------------------------------------------------------------------------------------------

def acc_seeds(n, seed, headroom):
    """n 544-bit seeds below 2^544 - headroom: uniform ones, and ones with words 0..15 all ones so every carry runs
    to word 16."""
    s = rand_range(seed, n, 0, W17 - headroom)
    s[1::4] = (s[1::4] >> 512 << 512) | ((1 << 512) - 1)
    return np.minimum(s, W17 - headroom - 1)


def lazy_pairs(p, n, count, seed, bw=8):
    """(n, count) operand pairs: a in [0, 2p), b in [0, 2^(32 bw)) for bw < 8 and [0, 2p) otherwise; the first rows
    take the extremes, (2p - 1) times the largest multiplier."""
    bmax = 2 * p if bw == 8 else 1 << (32 * bw)
    a = rand_range(seed, n * count, 0, 2 * p)
    b = rand_range(seed + 1, n * count, 0, bmax)
    ext_a = [2 * p - 1, 2 * p - 1, p, p - 1, 0, 1]
    ext_b = [bmax - 1, bmax // 2, bmax - 1, bmax - 1, bmax - 1, bmax - 1]
    a[: len(ext_a) * count] = np.repeat(ext_a, count)
    b[: len(ext_b) * count] = np.repeat(ext_b, count)
    return a.reshape(n, count), b.reshape(n, count)


def wide_inputs(a, b):
    n, count = a.shape
    return (to_words(a.ravel(), 8, 32).reshape(n, count, 8), to_words(b.ravel(), 8, 32).reshape(n, count, 8))


@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_wide_acc_exact(harness, fld, p):
    """mul_wide_acc_reg, mul_wide_acc_smem (at a stride of 64 words) and mul_wide_acc_bw<8> add a sequence of products
    of lazy operands to an arbitrary 17-word seed as exact integers: all three equal seed + sum(a b)."""
    n, count = 2048, 6
    a, b = lazy_pairs(p, n, count, 500 + fld)
    seed = acc_seeds(n, 510 + fld, count * (2 * p) ** 2)
    want = seed + (a * b).sum(axis=1)
    da, db = wide_inputs(a, b)
    for mode in (W_REG, W_SMEM, W_BW8):
        got = to_ints(harness.wide_acc(mode, to_words(seed, 17, 32), da, db), 32)
        assert (got == want).all(), f"mode {mode}: {mismatches(got, want)}"


@pytest.mark.gpu
@pytest.mark.parametrize("bw,mode", [(1, W_BW1), (2, W_BW2), (4, W_BW4)])
def test_wide_acc_narrow_multipliers(harness, bw, mode):
    """mul_wide_acc_bw<1|2|4> (the lincomb and value-source instantiations): a in [0, 2p) times multipliers up to
    2^(32 bw) - 1, added exactly; the words above the multiplier's are ignored, so they carry junk here."""
    p = O.R_MOD
    n, count = 2048, 6
    a, b = lazy_pairs(p, n, count, 600 + bw, bw=bw)
    seed = acc_seeds(n, 610 + bw, count * 2 * p << (32 * bw))
    want = seed + (a * b).sum(axis=1)
    junk = rand_range(620 + bw, n * count, 0, 1 << 256).reshape(n, count) >> (32 * bw) << (32 * bw)
    da, db = wide_inputs(a, b | junk)
    got = to_ints(harness.wide_acc(mode, to_words(seed, 17, 32), da, db), 32)
    assert (got == want).all(), mismatches(got, want)


@pytest.mark.gpu
def test_wide_acc_capacity(harness):
    """The accumulator's whole 544 bits: a seed of 2^544 - 1 - m lands exactly on 2^544 - 1 after adding the largest
    product m once (every form), and after 2^20 worst-case products (2p - 1)^2 on one thread (register and
    shared-memory forms) - "17 words hold > 2^30 such products" has 2^34.8 of room for either modulus."""
    for p in (O.R_MOD, O.Q_MOD):
        assert W17 // (2 * p - 1) ** 2 > 1 << 34
    p = O.Q_MOD
    cases = [(W_REG, 8), (W_SMEM, 8), (W_BW8, 8), (W_BW1, 1), (W_BW2, 2), (W_BW4, 4)]
    for mode, bw in cases:
        m = 2 * p - 1 if bw == 8 else (1 << (32 * bw)) - 1
        seed = to_words([W17 - 1 - (2 * p - 1) * m], 17, 32)
        da, db = wide_inputs(np.array([[2 * p - 1]], dtype=object), np.array([[m]], dtype=object))
        got = to_ints(harness.wide_acc(mode, seed, da, db), 32)
        assert got[0] == W17 - 1, f"mode {mode}: {got[0]:#x}"
    reps = 1 << 20
    worst = (2 * p - 1) ** 2
    seed = to_words([W17 - 1 - reps * worst], 17, 32)
    da, db = wide_inputs(np.array([[2 * p - 1]], dtype=object), np.array([[2 * p - 1]], dtype=object))
    for mode in (W_REG, W_SMEM):
        got = to_ints(harness.wide_acc(mode, seed, da, db, reps=reps), 32)
        assert got[0] == W17 - 1, f"mode {mode}: {got[0]:#x}"


# ---- reduce_wide17 ------------------------------------------------------------------------------------------------

def wide17_values(seed):
    vals = [0, W17 - 1, (1 << 512) - 1, 1 << 512, ((1 << 64) - 1) << 480, (W17 - 1) >> 1, W17 - (1 << 512)]
    rng = random.Random(seed)
    for k in range(17):
        vals += [0xffffffff << (32 * k), rng.getrandbits(32) << (32 * k)]
    vals += [1 << bit for bit in range(544)]
    vals += [rng.getrandbits(544) for _ in range(1 << 16)]
    vals += [rng.getrandbits(64) << 480 | rng.getrandbits(480) for _ in range(1 << 12)]  # straddling word 16
    return np.array(vals, dtype=object)


@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_reduce_wide17(harness, fld, p):
    """reduce_wide17 at 0, 2^544 - 1, every single word and single bit, values straddling word 16 and random 544-bit
    values: canonical and equal to acc R^-1 mod p."""
    acc = wide17_values(700 + fld)
    got = to_ints(harness.reduce_wide17(fld, to_words(acc, 17, 32)))
    want = acc * pow(R, -1, p) % p
    assert (got == want).all(), mismatches(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("fld,p", FIELDS)
def test_reduce_wide17_partial_bound(harness, fld, p):
    """The three lazy products reduce_wide17 adds - montmul(1, lo), montmul(R mod p, hi), montmul(R^2 mod p, top) with
    any 256-bit lo, hi and a 32-bit top - are below p + 1, p + (R mod p) and p + 1 (montmul(c, x) < c x / R + p).
    Their sum is below 3p + (R mod p) + 2 < 4p, tighter than the "5p + 1" its comment states: three of its five
    cond_sub_p calls already reach canonical form, so dropping one or two of them changes no result."""
    one = R % p
    wide = np.concatenate([np.array([R - 1, R - 2, (R - 1) >> 1, p, 2 * p, 5 * p, R - p], dtype=object),
                           rand_range(800 + fld, 4096, 0, R)])
    tops = np.concatenate([np.array([0xffffffff, 0xfffffffe, 1 << 31], dtype=object), rand_range(801 + fld, 4096, 0, 1 << 32)])
    bounds = []
    for c, x in ((1, wide), (one, wide), (R * R % p, tops)):
        got = to_ints(harness.field_op(fld, MUL_LAZY, to_words(np.full(x.size, c, dtype=object)), to_words(x)))
        assert (got == cios(np.full(x.size, c, dtype=object), x, p)).all()
        bounds.append(max(got))
    assert bounds[0] <= p and bounds[1] < p + one and bounds[2] <= p
    assert 3 * p + one + 2 < 4 * p


# ---- lane bins ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_bins_to_fr(harness):
    """bins_to_fr_kernel: lanes of 0, 2^32 - 1, 2^32, 2^64 - 1 (every bin of one value, and random mixes of them) and
    random lanes below 2^64 give sum(lane_w 2^(32 w)) mod p as canonical limbs. Lanes of 2^32 - 1 hold
    lo = 2^256 - 1 > 5p, which needs all five of its cond_sub_p calls."""
    p = O.R_MOD
    edges = np.array([0, (1 << 32) - 1, 1 << 32, (1 << 64) - 1], dtype=np.uint64)
    rng = np.random.default_rng(9)
    lanes = np.concatenate([np.repeat(edges[:, None], 8, axis=1),
                            edges[rng.integers(0, 4, size=(4096, 8))],
                            rng.integers(0, 1 << 64, size=(1 << 16, 8), dtype=np.uint64)])
    v = np.zeros(lanes.shape[0], dtype=object)
    for w in range(8):
        v = v + (lanes[:, w].astype(object) << (32 * w))
    got = to_ints(harness.bins_to_fr(lanes))
    want = v % p
    assert (got == want).all(), mismatches(got, want)
    assert want[1] == ((1 << 256) - 1) % p and ((1 << 256) - 1) >= 5 * p


@pytest.mark.gpu
def test_pf_flush(harness):
    """pf_flush from full warps: all lanes on one key, all keys distinct, keys repeating with periods 2, 3, 4 and 8,
    and emit masks that are full, random, alternating, a single lane and empty; warps share bins, so their atomics
    collide. Value words are mostly 0xffffffff. Every bin lane must be the exact sum of the emitted words."""
    nbins, warps = 48, 768
    rng = np.random.default_rng(17)
    lane = np.arange(32)
    keys, emits = [], []
    for w in range(warps):
        base = int(rng.integers(0, nbins - 32))
        shape = w % 6
        key = [np.full(32, base), base + rng.permutation(32), base + lane % 4, base + lane // 8, base + lane % 3,
               base + lane % 2][shape]
        mask = w // 6 % 5
        emit = [np.ones(32), rng.integers(0, 2, 32), lane % 2, lane == int(rng.integers(0, 32)), np.zeros(32)][mask]
        keys.append(key)
        emits.append(emit)
    key = np.concatenate(keys).astype(np.uint32)
    emit = np.concatenate(emits).astype(np.uint32)
    words = rng.integers(0, 1 << 32, size=(warps * 32, 8), dtype=np.uint64)
    words[rng.random(words.shape) < 0.75] = 0xffffffff
    val = (words[:, 0::2] | (words[:, 1::2] << np.uint64(32))).astype(np.uint64)
    want = np.zeros((nbins, 8), dtype=np.uint64)
    sel = emit != 0
    np.add.at(want, key[sel], words[sel])
    got = harness.pf_flush(emit, key, val, nbins)
    assert (got == want).all(), f"{(got != want).any(axis=1).sum()} bins differ"


# ---- G1 group law -------------------------------------------------------------------------------------------------

Q = O.Q_MOD


def g1_point(k):
    return O.g1_scalar_mul(O.G1_GEN, k)


def xyzz(P, lam):
    """The affine point P (None: the identity) at X = x lam^2, Y = y lam^3, ZZ = lam^2, ZZZ = lam^3."""
    if P is None:
        return (1, 1, 0, 0)                                   # XYZZ::inf()
    x, y = P
    l2, l3 = lam * lam % Q, lam * lam * lam % Q
    return (x * l2 % Q, y * l3 % Q, l2, l3)


def identity_at(rng):
    """An identity with arbitrary X, Y (is_inf looks at ZZ only)."""
    return (rng.randrange(Q), rng.randrange(Q), 0, 0)


def g1_dev(points):
    return C.ints_to_mont([c for pt in points for c in pt], Q).reshape(len(points), 16)


def check_points(out, want, what):
    """Device XYZZ outputs against affine answers: canonical coordinates; ZZ == 0 exactly for the identity;
    otherwise ZZ^3 == ZZZ^2 and (X / ZZ, Y / ZZZ) is the answer."""
    raw = to_ints(out.reshape(-1, 4))
    assert (raw < Q).all(), f"{what}: non-canonical coordinate"
    vals = C.mont_to_ints(out.reshape(-1, 4), Q)
    for i, w in enumerate(want):
        X, Y, ZZ, ZZZ = vals[4 * i: 4 * i + 4]
        if w is None:
            assert raw[4 * i + 2] == 0, f"{what} case {i}: expected the identity"
            continue
        assert ZZ != 0, f"{what} case {i}: identity instead of {w}"
        assert pow(ZZ, 3, Q) == pow(ZZZ, 2, Q), f"{what} case {i}: ZZ^3 != ZZZ^2"
        got = (X * pow(ZZ, -1, Q) % Q, Y * pow(ZZZ, -1, Q) % Q)
        assert got == w, f"{what} case {i}: {got} != {w}"


@pytest.fixture(scope="module")
def g1_cases():
    rng = random.Random(31)
    pts = [g1_point(rng.randrange(1, O.R_MOD)) for _ in range(12)]
    return rng, pts[:6], pts[6:]


def lam(rng):
    return rng.randrange(2, Q)


@pytest.mark.gpu
def test_xyzz_add_affine(harness, g1_cases):
    """xyzz_add_affine with the accumulator the identity (XYZZ::inf and arbitrary X, Y), P, -P, 2P or Q at a non-trivial
    ZZ / ZZZ, plus the affine P, negated or not: the doubling (acc == +-P) and cancellation (acc == -+P) branches are
    reached through projective equality. The affine identity (0, 0) is outside its contract ("never the identity
    here"): msm_accumulate_kernel and msm_select_sum_kernel skip (0, 0) bases before the call (the sorted path drops
    them in msm_digits_kernel), and gen_multiples_kernel adds its non-identity base."""
    rng, ps, qs = g1_cases
    acc, aff, neg, want = [], [], [], []
    for P, Qp in zip(ps, qs):
        for A in (None, "id", P, O.g1_neg(P), O.g1_add(P, P), Qp):
            for negate in (0, 1):
                acc.append(identity_at(rng) if A == "id" else xyzz(A, lam(rng)))
                aff.append((P[0], P[1], 0, 0))
                neg.append(negate)
                want.append(O.g1_add(None if A == "id" else A, O.g1_neg(P) if negate else P))
    out = harness.g1(G_ADD_AFFINE, g1_dev(acc), g1_dev(aff), np.array(neg))
    check_points(out, want, "xyzz_add_affine")


@pytest.mark.gpu
def test_xyzz_add(harness, g1_cases):
    """xyzz_add with either side the identity, a == b, a == -b and general operands, every operand at its own
    non-trivial ZZ / ZZZ, so the doubling and cancellation branches see projectively (not limb-wise) equal points."""
    rng, ps, qs = g1_cases
    a, b, want = [], [], []
    for P, Qp in zip(ps, qs):
        nP, P2 = O.g1_neg(P), O.g1_add(P, P)
        for A, B in ((None, P), (P, None), (None, None), ("id", P), (P, "id"), (P, P), (nP, nP), (P, nP), (nP, P),
                     (P, Qp), (P2, P), (P, P2)):
            a.append(identity_at(rng) if A == "id" else xyzz(A, lam(rng)))
            b.append(identity_at(rng) if B == "id" else xyzz(B, lam(rng)))
            want.append(O.g1_add(None if A == "id" else A, None if B == "id" else B))
    check_points(harness.g1(G_ADD, g1_dev(a), g1_dev(b)), want, "xyzz_add")


@pytest.mark.gpu
def test_xyzz_double(harness, g1_cases):
    """xyzz_double of the identity (both forms) and of general points at non-trivial ZZ / ZZZ."""
    rng, ps, qs = g1_cases
    a, want = [], []
    for P in ps + qs:
        for A in (None, "id", P, O.g1_neg(P)):
            a.append(identity_at(rng) if A == "id" else xyzz(A, lam(rng)))
            want.append(None if A in (None, "id") else O.g1_add(A, A))
    check_points(harness.g1(G_DOUBLE, g1_dev(a), g1_dev(a)), want, "xyzz_double")


@pytest.mark.gpu
def test_fq_inverse(harness):
    """fq_inverse of 1, 2, q - 1, q - 2 and random values: canonical with a a^-1 = 1. Its input 0 has no inverse; the
    exponentiation a^(q - 2) returns 0 for it, and that is pinned here."""
    vals = [1, 2, Q - 1, Q - 2, (1 << 253) + 1] + [v for v in rand_range(41, 2048, 1, Q)]
    a = C.ints_to_mont(vals, Q)
    out = harness.field_op(1, INVERSE, a)
    assert (to_ints(out) < Q).all()
    inv = C.mont_to_ints(out, Q)
    assert all(x * y % Q == 1 for x, y in zip(vals, inv))
    assert (harness.field_op(1, INVERSE, np.zeros((1, 4), dtype=np.uint64)) == 0).all()
