"""Multilinear evaluation without a GPU: the references of tests/mle_eval_ref.py against bind sequences (both orders)
and brute force over the hypercube, the pushforward against binding the materialised one-hot polynomial, the entry
points' behaviour on a box without a device, and the static resource budget of the evaluation kernels."""
import pathlib
import re
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import mle_eval_ref as ref
from test_build_artifacts import ptxas_entries

CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"
R = O.R_MOD


def _column(K, T, seed, none_frac):
    rng = np.random.Generator(np.random.PCG64(seed))
    addr = rng.integers(0, K, size=T)
    return [None if rng.random() < none_frac else int(a) for a in addr]


def _brute(evals, point):
    n = len(point)
    total = 0
    for x, f in enumerate(evals):
        w = 1
        for i, r in enumerate(point):
            bit = (x >> (n - 1 - i)) & 1
            w = w * (r if bit else 1 - r) % R
        total += f * w
    return total % R


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5])
def test_evaluate_equals_binds_in_both_orders_and_brute_force(n):
    evals = O.random_fr(100 + n, 1 << n)
    point = O.random_fr(200 + n, n)
    v = ref.evaluate(evals, point)
    hi = list(evals)
    for r in point:
        hi = O.bind(hi, r, O.HIGH_TO_LOW)
    lo = list(evals)
    for r in reversed(point):
        lo = O.bind(lo, r, O.LOW_TO_HIGH)
    assert [v] == hi == lo
    assert v == _brute(evals, point)


def test_compact_promotion():
    assert ref.promote(-1) == R - 1 and ref.promote(-(1 << 127)) == R - (1 << 127)
    assert ref.promote((0, False)) == 0 and ref.promote((5, False)) == R - 5 and ref.promote((5, True)) == 5
    vals = [3, -(1 << 63), (1 << 64) - 1, -7]
    pt = O.random_fr(7, 2)
    assert ref.evaluate_small(vals, pt) == ref.evaluate([v % R for v in vals], pt)


@pytest.mark.parametrize("K,T", [(1, 1), (1, 8), (2, 4), (4, 8), (8, 2), (16, 16)])
@pytest.mark.parametrize("none_frac", [0.0, 0.3, 1.0])
def test_pushforward_equals_the_bound_cycle_major_polynomial(K, T, none_frac):
    addr = _column(K, T, 31 * K + T, none_frac)
    lt, lk = T.bit_length() - 1, K.bit_length() - 1
    r_cycle, r_addr = O.random_fr(K + T, lt), O.random_fr(K * T, lk)
    G = ref.pushforward(addr, K, r_cycle)
    bound = ref.one_hot_flat(addr, K, T, "cycle_major")
    for r in r_cycle:
        bound = O.bind(bound, r, O.HIGH_TO_LOW)
    assert G == bound
    eq_addr = O.eq_evals(r_addr)
    dot = sum(a * b for a, b in zip(eq_addr, G)) % R
    assert dot == ref.one_hot_evaluate(addr, K, T, r_cycle + r_addr, "cycle_major")
    # address-major: the same polynomial with the two halves of the point swapped
    assert dot == ref.one_hot_evaluate(addr, K, T, r_addr + r_cycle, "address_major")
    # and the direct definition sum_j eq(r_cycle, j) eq(r_addr, addr_j)
    eq_cyc = O.eq_evals(r_cycle)
    assert dot == sum(eq_cyc[j] * eq_addr[a] for j, a in enumerate(addr) if a is not None) % R
    for layout in ("cycle_major", "address_major"):
        pt = r_cycle + r_addr if layout == "cycle_major" else r_addr + r_cycle
        assert ref.one_hot_evaluate_direct(addr, K, T, pt, layout) == dot


def test_entry_points_are_exported_and_need_a_device():
    lib = _lib.load()
    names = ["jb_table_evaluate_batch", "jb_small_evaluate_batch", "jb_one_hot_evaluate", "jb_one_hot_pushforward"]
    for n in names:
        assert n in _lib.SIGNATURES
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    assert lib.jb_table_evaluate_batch(None, None, 0, None, 0, None) == _lib.JB_ERR_NO_DEVICE
    assert lib.jb_small_evaluate_batch(None, None, 0, None, 1, 0, None, 0, None) == _lib.JB_ERR_NO_DEVICE
    assert lib.jb_one_hot_evaluate(None, None, 0, 1, 1, 1, 0, 0, None, None) == _lib.JB_ERR_NO_DEVICE
    assert lib.jb_one_hot_pushforward(None, None, 0, 1, 1, 1, 0, None, None) == _lib.JB_ERR_NO_DEVICE


def test_evaluation_kernels_fit_two_blocks_per_sm_without_local_memory():
    log = CSRC / "mle_eval.ptxas.log"
    if not log.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    ents = {k: v for k, v in ptxas_entries(log).items() if "mle_eval_kernel" in k or "pushforward_kernel" in k}
    assert len(ents) == 18      # field + 9 compact kinds + 4 one-hot gathers; 4 pushforward shapes
    for name, (regs, st, ld) in ents.items():
        assert regs <= 128 and (st, ld) == (0, 0), (name, regs, st, ld)
    obj, cuobjdump = CSRC / "mle_eval.o", shutil.which("cuobjdump")
    if not obj.exists() or cuobjdump is None:
        pytest.skip("mle_eval.o or cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], capture_output=True, text=True, timeout=300).stdout
    assert "IMAD.WIDE.U32" in sass
    assert not re.search(r"\b(LDL|STL)\b", sass)
