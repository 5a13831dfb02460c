"""CPU checks for expression members over sources: the promotion and gather of tests/source_ref.py against Python ints
and the evaluation references, the reference member's final evaluations against the evaluation entry points'
references, the C entry point's export and no-device status, and the source kernels' resource budget in the build."""
import ctypes
import pathlib
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import SCALAR_KINDS, _lib, small_scalars
from oracle import bn254 as O
import expr_ref as E
import mle_eval_ref as M
import source_ref as SR
from test_build_artifacts import ptxas_entries
from test_build_artifacts_staged import _loops

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"
U64, U128 = (1 << 64) - 1, (1 << 128) - 1
I64_MIN, I128_MIN = -(1 << 63), -(1 << 127)

# kind -> (values, their field values)
EXTREMES = {
    "u8": (np.array([0, 1, 255], dtype=np.uint8), [0, 1, 255]),
    "u16": (np.array([0, 65535], dtype=np.uint16), [0, 65535]),
    "u32": (np.array([0, (1 << 32) - 1], dtype=np.uint32), [0, (1 << 32) - 1]),
    "u64": (np.array([0, U64], dtype=np.uint64), [0, U64]),
    "i64": (np.array([0, -1, I64_MIN, (1 << 63) - 1], dtype=np.int64), [0, P - 1, P - (1 << 63), (1 << 63) - 1]),
    "u128": ([0, U128, 1 << 127], [0, U128, 1 << 127]),
    "i128": ([0, -1, I128_MIN, (1 << 127) - 1], [0, P - 1, P - (1 << 127), (1 << 127) - 1]),
    "s64": ([(0, True), (0, False), (U64, True), (U64, False)], [0, 0, U64, P - U64]),
    "s128": ([(0, True), (0, False), (U128, True), (U128, False)], [0, 0, U128, P - U128]),
}


@pytest.mark.parametrize("kind", sorted(EXTREMES))
def test_promotion_of_encoded_extremes(kind):
    values, want = EXTREMES[kind]
    a, k, n = small_scalars(values, kind if kind in ("u128", "i128", "s64", "s128") else None)
    assert k == SCALAR_KINDS[kind]
    assert SR.promote_column(SR.decode_column(a, kind)) == want
    assert SR.source_table(("compact", SR.decode_column(a, kind))) == want


@pytest.mark.parametrize("K", [1, 2, 16, 256])
def test_gather_matches_one_hot_evaluation(K):
    T = 32
    rng = np.random.default_rng(K)
    addr = [None if rng.random() < 0.2 else int(rng.integers(0, K)) for _ in range(T)]
    lk, lt = K.bit_length() - 1, T.bit_length() - 1
    point = O.random_fr(0x500 + K, lt + lk)
    r_cycle, r_addr = point[:lt], point[lt:]
    ra = SR.gather_one_hot(addr, K, r_addr)
    eq_a = O.eq_evals(list(r_addr)) if lk else [1]
    assert ra == [0 if a is None else eq_a[a] for a in addr]
    want = M.one_hot_evaluate_direct(addr, K, T, point, "cycle_major")
    assert M.evaluate(ra, r_cycle) == want
    if K <= 16:
        assert M.one_hot_evaluate(addr, K, T, point, "cycle_major") == want


def test_addresses_none_value():
    assert SR.addresses(np.array([0, 254, 255], dtype=np.uint8)) == [0, 254, None]
    assert SR.addresses(np.array([0, 65534, 65535], dtype=np.uint16)) == [0, 65534, None]


@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
def test_member_final_evals_are_the_evaluations(order):
    """read checking eq * (ra val + g wa val + g^2 wa inc) over one-hot ra / wa, a field val and an i64 inc: the final
    evaluations are the sources' values at the challenge point and the final claim eq(w, r) * the expression"""
    n, K, g = 4, 4, 0x1234567890ABCDEF
    T = 1 << n
    rng = np.random.default_rng(7)
    ra = [None if j % 5 == 0 else int(rng.integers(0, K)) for j in range(T)]
    wa = [int(rng.integers(0, K)) for _ in range(T)]
    val = O.random_fr(11, T)
    inc = [int(v) for v in rng.integers(-(1 << 63), (1 << 63) - 1, T)]
    r_ra, r_wa = O.random_fr(12, 2), O.random_fr(13, 2)
    mons = [(1, [0, 2]), (g, [1, 2]), (g * g % P, [1, 3])]
    w = O.random_fr(14, n)
    ref = SR.SourcesMember([("one_hot", ra, K, r_ra), ("one_hot", wa, K, r_wa), ("table", val), ("compact", inc)],
                           mons, order, w)
    claim = ref.claim()
    bound, bind = [], None
    for rnd in range(n):
        ev = ref.round_evals(bind)
        assert (ev[0] + ev[1]) % P == claim
        bind = O.random_fr(0x60 + rnd, 1)[0]
        claim = O.uni_from_evals(ev)
        claim = sum(c * pow(bind, i, P) for i, c in enumerate(claim)) % P
        bound.append(bind)
    ref.finish_rounds(bind)
    r = bound if order == O.HIGH_TO_LOW else list(reversed(bound))
    fin = ref.final_evals()
    assert fin[0] == M.one_hot_evaluate_direct(ra, K, T, list(r) + list(r_ra), "cycle_major")
    assert fin[1] == M.one_hot_evaluate_direct(wa, K, T, list(r) + list(r_wa), "cycle_major")
    assert fin[2] == M.evaluate(val, r)
    assert fin[3] == M.evaluate_small(inc, r)
    assert claim == ref.eq_scalar() * E.expr_value(fin, mons) % P


def test_create_expr_sources_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_expr_sources")
    assert ctypes.sizeof(_lib.SourceC) == 48   # 3 ints, padding, table, values, K, r_addr
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    out = ctypes.c_void_p()
    src = (_lib.SourceC * 1)()
    mons = (_lib.MonomialC * 1)()
    st = lib.jb_member_create_expr_sources(None, ctypes.cast(src, ctypes.c_void_p), 1, 2, ctypes.cast(mons, ctypes.c_void_p),
                                           1, None, 0, None, 0, ctypes.byref(out))
    assert st == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


def _entries(name):
    return {k: v for k, v in ptxas_entries(_need(CSRC / "sources.ptxas.log")).items() if name in k}


def test_source_kernels_within_128_registers_no_spills():
    ents = _entries("source_round_kernel")
    assert len(ents) == 12, ents      # 2 orders x (eval-only, bind, 125-bit bind) x (plain, split-eq weighted)
    assert all(regs <= 128 and st == 0 and ld == 0 for regs, st, ld in ents.values()), ents
    for name in ("source_bind_kernel", "check_addresses_kernel"):
        ents = _entries(name)
        assert len(ents) == 2 and all(st == 0 and ld == 0 for _, st, ld in ents.values()), ents


def test_source_kernel_loops_have_no_local_memory():
    obj = _need(CSRC / "sources.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    names = [k for k in ptxas_entries(CSRC / "sources.ptxas.log") if "source_round_kernel" in k]
    for name in names:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, timeout=600).stdout
        assert "LDS" in sass, name   # the pairs are staged in shared-memory columns
        assert "LDL" not in sass and "STL" not in sass, name
        loops = _loops(sass)
        assert loops, name
        for c in loops:
            assert not any(k.startswith(("LDL", "STL")) for k in c), (name, c)
