"""CPU checks for the read-write checking member: the dense reference and the restatement of the sparse entry
algorithm agree on every round polynomial and every final value over small register- and RAM-shaped workloads; the
rounds hold the sumcheck identities; the entry point is exported and reports no device; the new kernels use no local
memory."""
import ctypes
import pathlib
import shutil
import subprocess

import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import rw_ref as R
from test_build_artifacts import ptxas_entries

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def _check(K, T, A, shape, seed, **kw):
    wl = R.workload(seed, K, T, A, shape, **kw)
    t = T.bit_length() - 1
    w = O.random_fr(seed + 1, t)
    scale = O.random_fr(seed + 2, 1)[0] if seed % 2 else None
    ch = O.random_fr(seed + 3, t + K.bit_length() - 1)
    dense = R.dense_prove(*wl, w, scale, ch)
    sparse = R.sparse_prove(*wl, w, scale, ch)
    assert sparse == dense
    claim = R.claimed_sum(T, wl[2], wl[4], w, scale)
    for s, r in zip(dense[0], ch):
        assert (s[0] + s[1]) % P == claim
        claim = O.uni_evaluate(O.uni_from_evals(s), r)
    ra_val_inc = dense[1]
    fin = sum(c * ra_val_inc[a] * (ra_val_inc[-2] + d * ra_val_inc[-1]) for a, (_x, _v, c, d) in enumerate(wl[2]))
    e = O.evaluate(O.eq_evals(w, scale), ch[:t][::-1])
    assert claim == e * fin % P


@pytest.mark.parametrize("K", [1, 2, 8, 128])
@pytest.mark.parametrize("T", [2, 4, 64])
def test_references_agree_registers(K, T):
    for A in (1, 2, 3, 4):
        _check(K, T, A, "registers", 100 * K + T + A)


@pytest.mark.parametrize("K", [1, 2, 8, 128])
@pytest.mark.parametrize("T", [2, 4, 64])
def test_references_agree_ram(K, T):
    _check(K, T, 2, "ram", 7 * K + T, none_frac=0.05)


@pytest.mark.parametrize("K,A,shape", [(8, 3, "registers"), (128, 2, "ram")])
def test_references_agree_at_1024_cycles(K, A, shape):
    _check(K, 1024, A, shape, 5 + K, local=True)


def test_edge_patterns_agree():
    # all none; one key for everything; rs1 = rs2 = rd
    K, T = 4, 8
    for addr in ([None] * T, [2] * T, [j % K for j in range(T)]):
        accesses_addr = [addr, addr, addr]
        inc = [0 if a is None else 5 + j for j, a in enumerate(addr)]
        init = [10, 20, 30, 40]
        val = R.val_table(K, T, [(a, None, 0, 0) for a in accesses_addr], 2, inc, init)
        acc = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], c, d)
               for a, c, d in zip(accesses_addr, [3, 4, 5], [0, 0, 1])]
        w, ch = O.random_fr(1, 3), O.random_fr(2, 5)
        assert R.sparse_prove(K, T, acc, 2, inc, init, w, None, ch) == R.dense_prove(K, T, acc, 2, inc, init, w, None, ch)


def test_entry_point_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_read_write")
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = ctypes.c_void_p()
    assert lib.jb_member_create_read_write(None, None, 0, 0, 1, 0, 2, 1, None, None, None, 0, None, 1,
                                           ctypes.byref(h)) == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


RW_KERNELS = ("rw_eval_kernel", "rw_bind_kernel", "rw_flag_kernel", "rw_rows_kernel", "rw_count_kernel",
              "rw_fill_kernel", "rw_load_kernel", "rw_tables_kernel", "rw_scatter_kernel")


def test_rw_kernels_no_spills():
    ents = ptxas_entries(_need(CSRC / "read_write.ptxas.log"))
    for k in RW_KERNELS:
        assert any(k in name for name in ents), k
    for name, (regs, st, ld) in ents.items():
        if "rw_" in name:
            assert st == 0 and ld == 0, name


@pytest.mark.parametrize("kernel", RW_KERNELS)
def test_rw_kernels_have_no_local_memory(kernel):
    obj = _need(CSRC / "read_write.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    names = [k for k in ptxas_entries(CSRC / "read_write.ptxas.log") if kernel in k]
    assert names
    for name in names:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True,
                              timeout=600).stdout
        assert "EXIT" in sass and "LDL" not in sass and "STL" not in sass, name
