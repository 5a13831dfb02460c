"""One-hot row commitments on the device (jb_msm_g1_one_hot_rows) against the oracle's definition
(tests/one_hot_ref.py: one_hot_row_sets / one_hot_row_commitments), against closed forms over the bases (i + 1) G, and
against the existing device paths that take a materialised matrix (jb_msm_g1_rows) or host-built index sets
(jb_g1_batch_add). Points are compared as affine integers."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import G1Bases, ONE_HOT_NONE, _lib
from jolt_b200 import field as F
from jolt_b200.api import _p
from oracle import bn254 as O
from oracle import coracle as C
import one_hot_ref as ref

pytestmark = pytest.mark.gpu

G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
SRS_LOG = 14
U8, U16 = np.dtype(np.uint8), np.dtype(np.uint16)
LAYOUTS = list(ref.ONE_HOT_LAYOUTS)


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def srs(sess):
    """Random-looking bases beta^i G (scheme.rs:54-73) from the C oracle: affine ints for the oracle, and on the device."""
    xy = C.g1_powers(1 << SRS_LOG, G, C.ints_to_mont([O.random_fr(0x4D534D, 1)[0]])[0])
    pts = [(O.from_mont_limbs(r[:4], O.Q_MOD), O.from_mont_limbs(r[4:], O.Q_MOD)) for r in xy]
    return pts, G1Bases.from_affine(sess, xy)


@pytest.fixture(scope="module")
def multiples(sess):
    """bases[i] = (i + 1) G: a row's commitment is (sum over its columns c of (c + 1)) G."""
    return G1Bases.generate_multiples(sess, G, 1 << 18)


def column(K, T, dtype, seed, none_frac=0.0):
    rng = np.random.Generator(np.random.PCG64(seed))
    top = min(K, ONE_HOT_NONE[np.dtype(dtype)])          # the none value is never an address
    col = rng.integers(0, top, size=T).astype(dtype)
    col[rng.random(T) < none_frac] = ONE_HOT_NONE[np.dtype(dtype)]
    return col


def as_addr(col):
    none = ONE_HOT_NONE[col.dtype]
    return [None if a == none else int(a) for a in col.tolist()]


def to_affine(xyz):
    """(..., 12) Jacobian limbs -> list of affine int pairs / None, converting only the non-identity rows."""
    a = np.ascontiguousarray(xyz, dtype=np.uint64).reshape(-1, 12)
    out = [None] * a.shape[0]
    for i in np.nonzero(a[:, 8:].any(axis=1))[0]:
        out[i] = jolt_b200.g1_jacobian_to_affine(a[i])
    return out


def row_weights(col, K, W, layout):
    """sum of (column + 1) over the hot entries of every row (the closed form's scalar, as a Python int per row)."""
    T = col.shape[0]
    hot = col != ONE_HOT_NONE[col.dtype]
    j = np.nonzero(hot)[0].astype(np.int64)
    k = col[hot].astype(np.int64)
    idx = j * K + k if layout == "cycle_major" else k * T + j
    # float64 sums are exact here: a row's sum is at most W^2 <= 2^36
    sums = np.bincount(idx // W, weights=(idx % W + 1).astype(np.float64), minlength=K * T // W)
    return [int(s) for s in sums]


def closed_form(weights):
    """s_r G for every row through the C oracle; None for s_r == 0."""
    out = []
    for s in weights:
        if s % O.R_MOD == 0:
            out.append(None)
            continue
        xy, inf = C.g1_scalar_mul(G, C.ints_to_mont([s % O.R_MOD])[0])
        out.append(None if inf else (O.from_mont_limbs(xy[:4], O.Q_MOD), O.from_mont_limbs(xy[4:], O.Q_MOD)))
    return out


def widths(K, T):
    return sorted({w for w in (1, K // 2, K, 4 * K, K * T) if 1 <= w <= K * T})


@pytest.mark.parametrize("K", [1, 2, 16, 256])
@pytest.mark.parametrize("T", [1, 2, 16, 1024])
def test_matches_oracle(sess, srs, multiples, K, T):
    """Every valid W of {1, K/2, K, 4K, K T}, both layouts, both kinds; count = 3 (no none entries, 30 % none, all
    none) and count = 1. Bases beta^i G; a row width beyond the 2^14 oracle bases uses (i + 1) G and the closed form."""
    pts, bases = srs
    for dtype in (U8, U16):
        cols = [column(K, T, dtype, 7 * K + T, f) for f in (0.0, 0.3, 1.0)]
        for layout in LAYOUTS:
            for W in widths(K, T):
                wide = W > (1 << SRS_LOG)
                dev = multiples if wide else bases
                got = dev.one_hot_rows(cols, K, W, layout)
                assert got.shape == (3, K * T // W, 12)
                single = dev.one_hot_rows(cols[1], K, W, layout)
                for p, col in enumerate(cols):
                    if wide:
                        want = closed_form(row_weights(col, K, W, layout))
                    else:
                        want = ref.one_hot_row_commitments(pts, as_addr(col), K, T, W, layout)
                    assert to_affine(got[p]) == want, (dtype, layout, W, p)
                assert to_affine(single[0]) == to_affine(got[1])


@pytest.mark.parametrize("layout", LAYOUTS)
def test_skewed_column_is_complete(sess, multiples, layout):
    """Bases (i + 1) G, where partial sums of a row coincide with single bases and with other partial sums (2G + 3G
    meets 5G): a batch_add route gives wrong points here. A column where every cycle hits one address at T = W = 2^16
    makes, in address-major layout, ONE row of 2^16 points (the wide fold runs); with it a uniform column."""
    K, T, W = 16, 1 << 16, 1 << 16
    skew = np.full(T, 5, dtype=np.uint8)
    uni = column(K, T, np.uint8, 99)
    got = multiples.one_hot_rows(np.stack([skew, uni]), K, W, layout)
    for p, col in enumerate((skew, uni)):
        assert to_affine(got[p]) == closed_form(row_weights(col, K, W, layout)), p


@pytest.mark.parametrize("layout", LAYOUTS)
def test_agrees_with_msm_rows_and_batch_add(sess, srs, layout):
    """The materialised u8 0/1 matrix through jb_msm_g1_rows, and host-built row sets through jb_g1_batch_add (bases
    beta^i G keep batch_add's distinct-x precondition), give the same points."""
    _, bases = srs
    K, T, W = 16, 1 << 12, 1 << 8
    col = column(K, T, np.uint16, 4242, 0.2)
    R = K * T // W
    got = to_affine(bases.one_hot_rows(col, K, W, layout)[0])
    M = np.zeros((K, T), dtype=np.uint8)
    hot = col != ONE_HOT_NONE[col.dtype]
    M[col[hot].astype(np.int64), np.nonzero(hot)[0]] = 1
    flat = np.ascontiguousarray(M.T.reshape(-1) if layout == "cycle_major" else M.reshape(-1))
    assert to_affine(bases.msm_rows(flat, R, "u8")) == got
    sets = [np.nonzero(row)[0] for row in flat.reshape(R, W)]
    ba = [None if not r.any() else (F.from_limbs(r[:4], F.Q_MOD), F.from_limbs(r[4:], F.Q_MOD)) for r in bases.batch_add(sets)]
    assert ba == got


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("K,log_t,dtype,none_frac", [(16, 22, np.uint8, 0.0), (256, 24, np.uint16, 0.1)])
def test_dory_shape_at_scale_closed_form(sess, multiples, layout, K, log_t, dtype, none_frac):
    """T = 2^22 (K = 16) and T = 2^24 (K = 256, u16, 10 % none) with the Dory row width W = 2^ceil(log2(K T) / 2):
    every row against its closed form."""
    T = 1 << log_t
    log_kt = K.bit_length() - 1 + log_t
    W = 1 << ((log_kt + 1) // 2)
    col = column(K, T, dtype, log_t, none_frac)
    got = multiples.one_hot_rows(col, K, W, layout)[0]
    assert to_affine(got) == closed_form(row_weights(col, K, W, layout))


def test_internal_split_equals_single_calls(sess, multiples):
    """count = 5 at T = 2^26, K = 2 exceeds one pass's 2^28 hot entries: the call is split over the polynomials and must
    equal five single-polynomial calls (and the closed form, checked for the first)."""
    K, T = 2, 1 << 26
    W = 1 << 14
    cols = np.stack([column(K, T, np.uint8, 500 + p, 0.05 * p) for p in range(5)])
    got = multiples.one_hot_rows(cols, K, W, "address_major")
    assert got.shape == (5, K * T // W, 12)
    for p in range(5):
        assert to_affine(got[p]) == to_affine(multiples.one_hot_rows(cols[p], K, W, "address_major")[0]), p
    assert to_affine(got[0]) == closed_form(row_weights(cols[0], K, W, "address_major"))


def _raw(sess, bases, cols, kind, T, K, W, layout, out_rows=1, null_out=False):
    ptrs = (ctypes.c_void_p * max(len(cols), 1))(*[None if c is None else c.ctypes.data for c in cols])
    out = np.zeros((max(out_rows, 1), 12), dtype=np.uint64)
    return sess.lib.jb_msm_g1_one_hot_rows(sess.h, bases.handle, ptrs, len(cols), kind, T, K, W, layout,
                                           None if null_out else _p(out))


def test_errors_then_a_valid_call(sess, srs):
    pts, bases = srs
    u8, u16 = jolt_b200.SCALAR_KINDS["u8"], jolt_b200.SCALAR_KINDS["u16"]
    INVALID, LENGTH, UNSUPPORTED = _lib.JB_ERR_INVALID, _lib.JB_ERR_LENGTH, _lib.JB_ERR_UNSUPPORTED
    c8 = column(16, 64, np.uint8, 1)
    bad8 = c8.copy()
    bad8[17] = 16                                                     # an address >= K that is not the none value
    assert _raw(sess, bases, [c8, bad8], u8, 64, 16, 16, 0, 128) == INVALID
    bad16 = column(256, 64, np.uint16, 2)
    bad16[3] = 300
    assert _raw(sess, bases, [bad16], u16, 64, 256, 256, 1, 64) == INVALID
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        bases.one_hot_rows(bad8, 16, 16)
    assert e.value.status == INVALID
    assert _raw(sess, bases, [c8], jolt_b200.SCALAR_KINDS["u32"], 64, 16, 16, 0, 64) == INVALID   # unknown kind
    assert _raw(sess, bases, [c8], 99, 64, 16, 16, 0, 64) == INVALID
    assert _raw(sess, bases, [c8], u8, 64, 16, 16, 2, 64) == INVALID                             # unknown layout
    assert _raw(sess, bases, [c8], u8, 64, 12, 16, 0, 64) == INVALID                             # K not a power of two
    assert _raw(sess, bases, [c8[:48]], u8, 48, 16, 16, 0, 64) == INVALID                        # T not a power of two
    assert _raw(sess, bases, [c8], u8, 64, 16, 24, 0, 64) == INVALID                             # W not a power of two
    assert _raw(sess, bases, [c8], u8, 64, 16, 0, 0, 64) == INVALID
    assert _raw(sess, bases, [c8[:4]], u8, 4, 2, 16, 0, 64) == INVALID                           # W > K T
    assert _raw(sess, bases, [None], u8, 64, 16, 16, 0, 64) == INVALID                           # null column
    assert _raw(sess, bases, [c8], u8, 64, 16, 16, 0, 64, null_out=True) == INVALID              # null output
    assert sess.lib.jb_msm_g1_one_hot_rows(sess.h, bases.handle, None, 1, u8, 64, 16, 16, 0,
                                           _p(np.zeros(12, dtype=np.uint64))) == INVALID         # null column list
    big = column(1 << 16, 1 << 15, np.uint16, 3)
    assert _raw(sess, bases, [big], u16, 1 << 15, 1 << 16, 1 << 15, 0, 1) == LENGTH              # W > srs length
    assert _raw(sess, bases, [big, big], u16, 1 << 15, 1 << 16, 1, 0, 1) == UNSUPPORTED          # count R >= 2^32
    assert _raw(sess, bases, [], u8, 64, 16, 16, 0, 1) == _lib.JB_OK                              # count == 0
    with pytest.raises(ValueError):
        bases.one_hot_rows(c8, 16, 16, layout="row_major")
    with pytest.raises(ValueError):
        bases.one_hot_rows(c8.astype(np.uint32), 16, 16)
    import torch
    with pytest.raises(ValueError, match="one_hot_rows"):   # host columns only
        bases.one_hot_rows(torch.from_numpy(c8).cuda(), 16, 16)
    # the same context then commits a valid column correctly
    for layout in LAYOUTS:
        got = bases.one_hot_rows(c8, 16, 16, layout)[0]
        assert to_affine(got) == ref.one_hot_row_commitments(pts, as_addr(c8), 16, 64, 16, layout)
