"""CPU checks for Dory's vector-matrix product: tests/vmp_ref.py against a brute-force double sum over the terms and
against the materialised one-hot 0/1 matrix; the C entry point's export and no-device status; and the new kernels'
resource budget."""
import ctypes
import pathlib
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import lincomb_ref as LR
import one_hot_ref
import vmp_ref as V
from test_build_artifacts import ptxas_entries
from test_build_artifacts_staged import _loops

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"
VMP_KERNELS = ("vmp_gather_kernel", "vmp_scatter_kernel")


def _addr(rng, T, K, none_frac=0.3):
    return [None if rng.random() < none_frac else int(rng.integers(0, K)) for _ in range(T)]


@pytest.mark.parametrize("W", [1, 2, 4, 8, 16, 32])
def test_reference_is_the_brute_force_double_sum(W):
    rng = np.random.default_rng(W)
    n = 5
    a, b = O.random_fr(1, 1 << n), O.random_fr(2, 1 << (n - 3))
    small = [int(v) for v in rng.integers(-1000, 1000, 1 << (n - 1))]
    addr = _addr(rng, 4, 4)
    c = O.random_fr(3, 4)
    terms = [("table", a, c[0]), ("table", b, c[1]), ("compact", small, c[2]), ("one_hot", addr, 4, "cycle_major", c[3])]
    flat = [0] * 16
    for j, k in enumerate(addr):
        if k is not None:
            flat[j * 4 + k] = 1
    left = O.random_fr(4, (1 << n) // W)
    got = V.vector_matrix_product(terms, 1 << n, W, left)
    for col in range(W):
        want = 0
        for row, l in enumerate(left):
            x = row * W + col
            want += l * c[0] * a[x]
            want += l * c[1] * b[x] if x < len(b) else 0
            want += l * c[2] * small[x] if x < len(small) else 0
            want += l * c[3] * flat[x] if x < len(flat) else 0
        assert got[col] == want % P, col


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
@pytest.mark.parametrize("K,T", [(1, 8), (2, 8), (4, 4), (16, 2)])
def test_one_hot_term_is_the_materialised_matrix(K, T, layout):
    """W below, equal to and above K and T (up to K T), against the 0/1 rows of one_hot_ref"""
    rng = np.random.default_rng(K * 10 + T)
    addr = _addr(rng, T, K)
    c = O.random_fr(K + T, 1)[0]
    W = 1
    while W <= K * T:
        R = K * T // W
        left = O.random_fr(W, R)
        sets = one_hot_ref.one_hot_row_sets(addr, K, T, W, layout)
        want = [c * sum(left[r] for r in range(R) if col in sets[r]) % P for col in range(W)]
        assert V.vector_matrix_product([("one_hot", addr, K, layout, c)], K * T, W, left) == want, W
        W *= 2


def test_reference_of_a_single_row_is_the_linear_combination():
    """W = len: v = left[0] P"""
    terms = [("table", O.random_fr(5, 8), 7), ("compact", [-3, 4], 11)]
    left = O.random_fr(6, 1)
    P_ = LR.linear_combination(terms, 8)
    assert V.vector_matrix_product(terms, 8, 8, left) == [left[0] * v % P for v in P_]


def test_vector_matrix_product_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_lc_vector_matrix_product")
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    out = ctypes.c_uint64()
    terms = (_lib.LcTermC * 1)()
    st = lib.jb_lc_vector_matrix_product(None, ctypes.cast(terms, ctypes.c_void_p), 1, 1, 1, 0, ctypes.byref(out))
    assert st == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


def test_vmp_kernels_within_128_registers_no_spills():
    ents = ptxas_entries(_need(CSRC / "vmp.ptxas.log"))
    for k in VMP_KERNELS:
        mine = {n: v for n, v in ents.items() if k in n}
        assert len(mine) == 1, (k, mine)
        assert all(regs <= 128 and st == 0 and ld == 0 for regs, st, ld in mine.values()), mine


@pytest.mark.parametrize("kernel", VMP_KERNELS)
def test_vmp_kernels_have_no_local_memory(kernel):
    obj = _need(CSRC / "vmp.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    name = next(k for k in ptxas_entries(CSRC / "vmp.ptxas.log") if kernel in k)
    sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, timeout=600).stdout
    assert "LDL" not in sass and "STL" not in sass
    loops = _loops(sass)
    assert loops
    for c in loops:
        assert not any(k.startswith(("LDL", "STL")) for k in c), c
