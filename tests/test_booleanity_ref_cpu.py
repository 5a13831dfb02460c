"""CPU checks for the booleanity member: the member's algorithm (address rounds from the pushforward and its squared
copy, cycle rounds from F[addr]) agrees with the dense sumcheck over the materialised K x T tables on every round
polynomial and final value, in both binding orders; the rounds hold the sumcheck identities; the entry point is
exported, refuses bad arguments without a device, and its kernels use no local memory."""
import ctypes
import pathlib
import shutil
import subprocess

import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import booleanity_ref as B
from test_build_artifacts import ptxas_entries

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def _check(K, T, addrs, seed, order):
    d = len(addrs)
    lk, lt = K.bit_length() - 1, T.bit_length() - 1
    coeffs = O.random_fr(seed, d)
    r_addr, r_cycle = O.random_fr(seed + 1, lk), O.random_fr(seed + 2, lt)
    scale = O.random_fr(seed + 3, 1)[0] if seed % 2 else None
    ch = O.random_fr(seed + 4, lk + lt)
    dense = B.dense_prove(K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order)
    sparse = B.sparse_prove(K, T, addrs, coeffs, r_addr, r_cycle, scale, ch, order)
    assert sparse == dense
    claim = 0  # ra is 0 / 1: the claimed sum is zero
    for s, r in zip(dense[0], ch):
        assert (s[0] + s[1]) % P == claim
        claim = O.uni_evaluate(O.uni_from_evals(s), r)
    e = B.eq_scalar(K, T, r_addr, r_cycle, scale, ch, order)
    assert claim == B.final_claim(dense[1], coeffs, e)


@pytest.mark.parametrize("order", [B.HIGH_TO_LOW, B.LOW_TO_HIGH])
@pytest.mark.parametrize("K", [1, 2, 16])
@pytest.mark.parametrize("T", [2, 8, 64])
@pytest.mark.parametrize("d", [1, 3])
def test_sparse_equals_dense(order, K, T, d):
    _check(K, T, B.random_columns(100 * K + T + d, K, T, d), 7 * K + T + d + order, order)


@pytest.mark.parametrize("order", [B.HIGH_TO_LOW, B.LOW_TO_HIGH])
@pytest.mark.parametrize("K,T", [(2, 8), (16, 8), (16, 2)])
def test_edge_columns_agree(order, K, T):
    all_none = [None] * T
    one_address = [K - 1] * T
    _check(K, T, [all_none], 11 + order, order)
    _check(K, T, [one_address, all_none], 12 + order, order)
    _check(K, T, [[j % K for j in range(T)], one_address], 13 + order, order)


@pytest.mark.parametrize("order", [B.HIGH_TO_LOW, B.LOW_TO_HIGH])
def test_single_cycle_agrees(order):
    _check(8, 1, B.random_columns(3, 8, 1, 2, none_frac=0.0), 21 + order, order)


def test_entry_point_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_booleanity")
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = ctypes.c_void_p()
    assert lib.jb_member_create_booleanity(None, None, 0, 1, 0, 2, 1, None, None, None, None, 1,
                                           ctypes.byref(h)) == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


BOOL_KERNELS = ("bool_addr_kernel", "bool_cycle_kernel", "bool_final_kernel")


def test_bool_kernels_no_spills():
    ents = ptxas_entries(_need(CSRC / "booleanity.ptxas.log"))
    for k in BOOL_KERNELS:
        assert any(k in name for name in ents), k
    for name, (regs, st, ld) in ents.items():
        if "bool_" in name:
            assert st == 0 and ld == 0, name


@pytest.mark.parametrize("kernel", BOOL_KERNELS)
def test_bool_kernels_have_no_local_memory(kernel):
    obj = _need(CSRC / "booleanity.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    names = [k for k in ptxas_entries(CSRC / "booleanity.ptxas.log") if kernel in k]
    assert names
    for name in names:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True,
                              timeout=600).stdout
        assert "EXIT" in sass and "LDL" not in sass and "STL" not in sass, name
