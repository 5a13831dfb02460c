"""CPU checks for expression members: the reference in tests/expr_ref.py against brute force over the hypercube (the
round polynomial evaluated from the multilinear extensions at (bound challenges, t, free variables)), the C entry
point's export and its no-device status, and the expression kernel's resource budget in the build."""
import ctypes
import itertools
import math
import pathlib
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import _lib, field as F
from oracle import bn254 as O
import expr_ref as E
import sumcheck_ref as S
from test_build_artifacts import ptxas_entries
from test_build_artifacts_staged import _loops

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def _eq(w, x):
    return math.prod((wi * xi + (1 - wi) * (1 - xi)) % P for wi, xi in zip(w, x)) % P


def brute_round(tables, monomials, order, bound, t, eq_point=None, eq_scale=1):
    """s(t) of the round after binding `bound` (challenges in round order), from the multilinear extensions."""
    n = len(tables[0]).bit_length() - 1
    k = len(bound)
    total = 0
    for rest in itertools.product([0, 1], repeat=n - k - 1):
        if order == O.HIGH_TO_LOW:   # round k binds variable k (the MSB first)
            pt = list(bound) + [t] + list(rest)
        else:                        # round k binds variable n-1-k
            pt = list(rest) + [t] + list(reversed(bound))
        v = E.expr_value([O.evaluate(tab, pt) for tab in tables], monomials)
        if eq_point is not None:
            v = v * eq_scale * _eq(eq_point, pt)
        total += v
    return total % P


def _to_ints(limbs):
    return F.limbs_to_ints(np.ascontiguousarray(limbs, dtype=np.uint64))


GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
SHAPES = {
    "booleanity": (1, [(1, [0, 0]), (-1, [0])]),
    "ab_minus_c": (3, [(1, [0, 1]), (-1, [2])]),
    "rw_shared": (4, [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA, [1, 3])]),
    "square_in_product": (2, [(5, [0, 0, 1])]),
    "degree6": (4, [(GAMMA, [0, 1, 2, 3, 0, 1])]),
    "degree1": (1, [(7, [0])]),
    "zero_coeff": (3, [(0, [0, 1]), (1, [1, 2]), (3, [2])]),
    "extreme_coeffs": (3, [(P - 1, [0, 1]), ((1 << 256) % P, [1, 2]), (S.C_SIGN, [2, 0, 0])]),
}


@pytest.mark.parametrize("eq", [False, True])
@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_reference_matches_brute_force_every_round(shape, order, eq):
    T, monomials = SHAPES[shape]
    n = 3
    if shape == "degree6" and eq:
        n = 2
    tables = [_to_ints(S.rand_limbs_full(0x51 + j, 1 << n)) for j in range(T)]
    if shape == "extreme_coeffs":   # limb-extreme entries
        tables = [_to_ints(np.stack([S.extreme_limbs[(3 * j + i) % len(S.extreme_limbs)] for i in range(1 << n)]))
                  for j in range(T)]
    w = O.random_fr(0xE0 + n, n) if eq else None
    scale = 11 if eq else None
    ref = E.ExpressionMember(tables, monomials, order, w, scale)
    deg = E.expr_degree(monomials, eq)
    assert ref.degree == deg
    first = E.expr_round_evals(tables, monomials, order, w, scale)
    bound = []
    bind = None
    for rnd in range(n):
        ev = ref.round_evals(bind)
        if rnd == 0:
            assert ev == first
        want = [brute_round(tables, monomials, order, bound, t, w, scale or 1) for t in range(deg + 1)]
        assert ev == want, f"round {rnd}"
        bind = O.random_fr(0x900 + rnd, 1)[0] if rnd % 2 else F.from_limbs(S.extreme_challenge(rnd + 1))
        bound.append(bind)
    ref.finish_rounds(bind)
    pt = bound if order == O.HIGH_TO_LOW else list(reversed(bound))
    assert ref.final_evals() == [O.evaluate(t, pt) for t in tables]
    if eq:
        assert ref.eq_scalar() == scale * _eq(w, pt) % P


def test_reference_prove_batch_round_checks():
    """the oracle engine accepts the member: its claims chain through every round"""
    n = 4
    tabs = [O.random_fr(70 + j, 1 << n) for j in range(3)]
    mons = [(1, [0, 1]), (-1, [2]), (GAMMA, [0, 0, 2])]
    ref = E.ExpressionMember(tabs, mons, O.LOW_TO_HIGH, O.random_fr(3, n))
    claim = ref.claim()
    res = O.prove_batch([dict(input_claim=claim, coefficient=1, rounds=n, offset=0)], [ref], n, ref.degree, claim,
                        lambda r, c: (sum(c) * 7 + r + 3) % P)
    fin = ref.final_evals()
    assert res["final_claim"] == ref.eq_scalar() * E.expr_value(fin, [(c % P, t) for c, t in mons]) % P


def test_create_expr_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_expr")
    assert ctypes.sizeof(_lib.MonomialC) == 64   # 32 + 4 + 4 * JB_EXPR_MAX_DEGREE, padded to the 8-byte alignment
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    out = ctypes.c_void_p()
    mons = (_lib.MonomialC * 1)()
    handles = np.zeros(1, dtype=np.uint64)
    st = lib.jb_member_create_expr(None, handles.ctypes.data_as(_lib.c_u64p), 1, ctypes.cast(mons, ctypes.c_void_p), 1,
                                   None, 0, None, 0, ctypes.byref(out))
    assert st == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


def test_expr_kernels_within_128_registers_no_spills():
    ents = {k: v for k, v in ptxas_entries(_need(CSRC / "member.ptxas.log")).items() if "expr_round_kernel" in k}
    assert len(ents) == 12, ents      # 2 orders x (eval-only, bind, 125-bit bind) x (plain, split-eq weighted)
    assert all(regs <= 128 and st == 0 and ld == 0 for regs, st, ld in ents.values()), ents


def test_expr_kernel_loops_have_no_local_memory():
    obj = _need(CSRC / "member.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    names = [k for k in ptxas_entries(CSRC / "member.ptxas.log") if "expr_round_kernel" in k]
    for name in names:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, timeout=600).stdout
        assert "LDS" in sass, name   # the bound pairs are staged in shared-memory columns
        assert "LDL" not in sass and "STL" not in sass, name
        loops = _loops(sass)
        assert loops, name
        for c in loops:
            assert not any(k.startswith(("LDL", "STL")) for k in c), (name, c)
