"""CPU checks for the read-write checking member with its address rounds after p cycle rounds: the dense reference in
the mixed layout and the restatement of the member's three phases agree on every round polynomial and every final value
for every p, over small register- and RAM-shaped workloads and the device tests' access patterns; p = t is rw_ref's
order; the rounds hold the sumcheck identities; the entry point is exported and reports no device; the new kernels use
no local memory."""
import ctypes
import pathlib

import numpy as np
import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import rw_ref as R
import rw_phases_ref as RP
from test_build_artifacts import ptxas_entries

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def _check(wl, seed, ps=None):
    K, T, accesses, write, inc, init = wl
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    w = O.random_fr(seed + 1, t)
    scale = O.random_fr(seed + 2, 1)[0] if seed % 2 else None
    ch = O.random_fr(seed + 3, t + kappa)
    for p in range(t + 1) if ps is None else ps:
        dense = RP.dense_prove(*wl, w, scale, ch, p)
        sparse = RP.sparse_prove(*wl, w, scale, ch, p)
        assert sparse == dense, p
        claim = R.claimed_sum(T, accesses, inc, w, scale)
        for s, r in zip(dense[0], ch):
            assert (s[0] + s[1]) % P == claim, p
            claim = O.uni_evaluate(O.uni_from_evals(s), r)
        fin = dense[1]
        r_addr, r_cycle = RP.point(K, T, p, ch)
        e = O.evaluate(O.eq_evals(w, scale), r_cycle)
        assert claim == e * sum(c * fin[a] * (fin[-2] + d * fin[-1]) for a, (_x, _v, c, d) in enumerate(accesses)) % P
        assert fin[-1] == O.evaluate([x % P for x in inc], r_cycle)


@pytest.mark.parametrize("K,T", [(1, 2), (1, 8), (2, 2), (2, 4), (4, 8), (8, 16), (16, 32), (16, 8)])
@pytest.mark.parametrize("A", [1, 2, 3, 4])
def test_references_agree_registers(K, T, A):
    _check(R.workload(100 * K + T + A, K, T, A, "registers"), 10 * K + T + A)


@pytest.mark.parametrize("K,T", [(1, 4), (2, 2), (8, 16), (16, 32), (16, 8)])
def test_references_agree_ram(K, T):
    _check(R.workload(7 * K + T, K, T, 2, "ram", none_frac=0.05), 3 * K + T)


@pytest.mark.parametrize("pattern", ["all_none", "one_key", "distinct", "rs1_rs2_rd", "write_only"])
def test_access_patterns(pattern):
    # the patterns of the device test, at a size the dense reference can take
    K, T = 16, 16
    rng = np.random.default_rng(7)
    if pattern == "all_none":
        cols = [[None] * T] * 3
    elif pattern == "one_key":
        cols = [[5] * T] * 3
    elif pattern == "distinct":
        cols = [[(j + 5 * a) % K for j in range(T)] for a in range(3)]
    elif pattern == "rs1_rs2_rd":
        c = [int(x) for x in rng.integers(0, K, T)]
        cols = [c, c, c]
    else:  # writes to keys never read
        cols = [[int(x) for x in rng.integers(0, 4, T)]] * 2 + [[int(x) for x in rng.integers(8, K, T)]]
    inc = [0 if cols[2][j] is None else int(rng.integers(0, 1 << 40)) for j in range(T)]
    init = [int(x) for x in rng.integers(0, 1 << 60, K)]
    val = R.val_table(K, T, [(a, None, 0, 0) for a in cols], 2, inc, init)
    acc = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], c, d)
           for a, c, d in zip(cols, O.random_fr(9, 3), [0, 0, 1])]
    _check((K, T, acc, 2, inc, init), 11)


@pytest.mark.parametrize("K,T,A,shape", [(1, 64, 3, "registers"), (8, 64, 3, "registers"), (128, 64, 2, "ram"),
                                         (128, 1024, 3, "registers")])
def test_p_t_is_rw_ref(K, T, A, shape):
    wl = R.workload(K + T, K, T, A, shape)
    t = T.bit_length() - 1
    w, ch = O.random_fr(1, t), O.random_fr(2, t + K.bit_length() - 1)
    assert RP.sparse_prove(*wl, w, 5, ch, t) == R.sparse_prove(*wl, w, 5, ch)


def test_sparse_at_1024_cycles_every_split_point():
    # the sparse restatement alone at a size the dense one cannot take: the final claim from the final values
    K, T = 128, 1024
    wl = R.workload(77, K, T, 2, "ram", local=True)
    t, kappa = 10, 7
    w, ch = O.random_fr(78, t), O.random_fr(79, t + kappa)
    for p in (0, 3, 9):
        rounds, fin = RP.sparse_prove(*wl, w, None, ch, p)
        claim = R.claimed_sum(T, wl[2], wl[4], w)
        for s, r in zip(rounds, ch):
            assert (s[0] + s[1]) % P == claim, p
            claim = O.uni_evaluate(O.uni_from_evals(s), r)
        e = O.evaluate(O.eq_evals(w), RP.point(K, T, p, ch)[1])
        assert claim == e * sum(c * fin[a] * (fin[-2] + d * fin[-1]) for a, (_x, _v, c, d) in enumerate(wl[2])) % P


def test_entry_point_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_read_write_phases")
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = ctypes.c_void_p()
    assert lib.jb_member_create_read_write_phases(None, None, 0, 0, 1, 0, 2, 1, None, None, None, 0, None, 0, 1,
                                                  ctypes.byref(h)) == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


PHASE_KERNELS = ("rw_key_eval_kernel", "rw_iota_kernel", "rw_gather_kernel", "rw_key_offsets_kernel", "rw_dense_kernel")


@pytest.mark.parametrize("kernel", PHASE_KERNELS)
def test_phase_kernels_built_without_spills(kernel):
    ents = ptxas_entries(_need(CSRC / "read_write.ptxas.log"))
    names = [name for name in ents if kernel in name]
    assert names
    for name in names:
        _regs, st, ld = ents[name]
        assert st == 0 and ld == 0, name
