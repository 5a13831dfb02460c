"""One-hot row commitments without a GPU: the oracle's row sets against the materialised K x T 0/1 matrix laid out and
cut into rows with numpy, its commitments against the naive MSM of every row, and the C entry point's behaviour on a
box without a device."""
import numpy as np
import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import one_hot_ref as ref

SHAPES = [(1, 1), (1, 8), (2, 4), (4, 8), (8, 2), (16, 16)]


def _column(K, T, seed, none_frac):
    rng = np.random.Generator(np.random.PCG64(seed))
    addr = rng.integers(0, K, size=T)
    return [None if rng.random() < none_frac else int(a) for a in addr]


def _widths(K, T):
    return sorted({w for w in (1, K // 2, K, 4 * K, K * T, 2) if 1 <= w <= K * T})


def _numpy_rows(addr, K, T, W, layout):
    M = np.zeros((K, T), dtype=np.uint8)           # M[k, j] = 1 iff cycle j touched address k
    for j, k in enumerate(addr):
        if k is not None:
            M[k, j] = 1
    flat = M.T.reshape(-1) if layout == "cycle_major" else M.reshape(-1)   # j K + k  /  k T + j
    return [list(np.nonzero(row)[0]) for row in flat.reshape(K * T // W, W)]


@pytest.mark.parametrize("K,T", SHAPES)
@pytest.mark.parametrize("layout", ref.ONE_HOT_LAYOUTS)
@pytest.mark.parametrize("none_frac", [0.0, 0.3, 1.0])
def test_row_sets_equal_the_materialised_matrix(K, T, layout, none_frac):
    addr = _column(K, T, 1000 * K + T, none_frac)
    for W in _widths(K, T):
        assert ref.one_hot_row_sets(addr, K, T, W, layout) == _numpy_rows(addr, K, T, W, layout), W


@pytest.mark.parametrize("layout", ref.ONE_HOT_LAYOUTS)
def test_row_commitments_equal_the_naive_msm_of_each_row(layout):
    K, T = 4, 8
    bases = [O.g1_scalar_mul(O.G1_GEN, k) for k in O.random_fr(0x0E07, K * T)]
    bases[3] = bases[5]                                     # a repeated base: doublings inside a row
    addr = _column(K, T, 5, 0.25)
    for W in _widths(K, T):
        got = ref.one_hot_row_commitments(bases, addr, K, T, W, layout)
        rows = _numpy_rows(addr, K, T, W, layout)
        assert len(got) == K * T // W
        for r, cols in enumerate(rows):
            scalars = [1 if c in cols else 0 for c in range(W)]
            assert got[r] == O.g1_msm_naive(bases[:W], scalars), (W, r)


def test_oracle_rejects_an_address_beyond_K():
    with pytest.raises(ValueError):
        ref.one_hot_row_sets([0, 4], 4, 2, 2, "cycle_major")


def test_entry_point_is_exported_and_needs_a_device():
    lib = _lib.load()
    fn = lib.jb_msm_g1_one_hot_rows
    assert "jb_msm_g1_one_hot_rows" in _lib.SIGNATURES
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    assert fn(None, 0, None, 0, 1, 1, 1, 1, 0, None) == _lib.JB_ERR_NO_DEVICE
