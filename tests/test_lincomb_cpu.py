"""CPU checks for random linear combinations: tests/lincomb_ref.py against brute-force sums, the prefix-evaluation
identity and the materialised one-hot 0/1 matrix; the C restatement (tests/lincomb_cref.py) against the big-int
reference; the C entry point's export, struct layout and no-device status; and the kernel's resource budget."""
import ctypes
import pathlib
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import _lib, small_scalars
from jolt_b200 import field as F
from oracle import bn254 as O
import lincomb_cref as CR
import lincomb_ref as LR
import mle_eval_ref as M
import one_hot_ref
import source_ref as SR
from test_build_artifacts import ptxas_entries
from test_build_artifacts_staged import _loops

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def _addr(rng, T, K, none_frac=0.3):
    return [None if rng.random() < none_frac else int(rng.integers(0, K)) for _ in range(T)]


def test_reference_is_the_brute_force_sum():
    rng = np.random.default_rng(1)
    n = 4
    a, b = O.random_fr(1, 1 << n), O.random_fr(2, 1 << (n - 2))
    small = [int(v) for v in rng.integers(-1000, 1000, 1 << (n - 1))]
    addr = _addr(rng, 4, 4)
    c = O.random_fr(3, 4)
    got = LR.linear_combination([("table", a, c[0]), ("table", b, c[1]), ("compact", small, c[2]),
                                 ("one_hot", addr, 4, "address_major", c[3])], 1 << n)
    flat = M.one_hot_flat(addr, 4, 4, "address_major")
    for x in range(1 << n):
        want = c[0] * a[x]
        want += c[1] * b[x] if x < len(b) else 0
        want += c[2] * (small[x] % P) if x < len(small) else 0
        want += c[3] * flat[x]
        assert got[x] == want % P


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
@pytest.mark.parametrize("K", [1, 2, 16])
def test_one_hot_term_is_the_materialised_matrix(K, layout):
    T = 8
    rng = np.random.default_rng(K)
    addr = _addr(rng, T, K)
    c = O.random_fr(K, 1)[0]
    sets = one_hot_ref.one_hot_row_sets(addr, K, T, K * T, layout)[0]
    want = [c if x in sets else 0 for x in range(K * T)]
    assert LR.linear_combination([("one_hot", addr, K, layout, c)], K * T) == want


@pytest.mark.parametrize("n", [0, 1, 3, 6])
def test_prefix_evaluation_identity(n):
    """P(point) = sum_i c_i prod_{k < n - n_i} (1 - point[k]) p_i(point[n - n_i:])"""
    rng = np.random.default_rng(n)
    point = O.random_fr(40 + n, n)
    terms, claims = [], []
    for i, n_i in enumerate(sorted({0, n // 2, n})):
        vals = O.random_fr(50 + i, 1 << n_i)
        c = O.random_fr(60 + i, 1)[0]
        terms.append(("table", vals, c))
        claims.append((c, n_i, M.evaluate(vals, point[n - n_i:])))
    if n >= 1:
        lt = n - 1
        addr = _addr(rng, 1 << lt, 2)
        c = O.random_fr(70, 1)[0]
        terms.append(("one_hot", addr, 2, "cycle_major", c))
        claims.append((c, n, M.one_hot_evaluate_direct(addr, 2, 1 << lt, point, "cycle_major")))
    got = LR.linear_combination(terms, 1 << n)
    assert M.evaluate(got, point) == LR.combined_claim(claims, point)


def test_c_restatement_matches_reference():
    rng = np.random.default_rng(9)
    n = 7
    terms_py, terms_c = [], []
    tab = O.random_fr(90, 1 << n)
    terms_py.append(("table", tab, P - 1))
    terms_c.append(("table", F.ints_to_limbs(tab), P - 1))
    for kind in ("u8", "u16", "u32", "u64", "i64"):
        dt = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i64": np.int64}[kind]
        info = np.iinfo(dt)
        vals = rng.integers(info.min, info.max, 1 << (n - 1), dtype=dt, endpoint=True)
        a, k, m = small_scalars(vals)
        c = O.random_fr(91 + k, 1)[0]
        terms_py.append(("compact", SR.decode_column(a, kind), c))
        terms_c.append(("compact", a, k, m, c))
    for kind in ("u128", "i128", "s64", "s128"):
        lim = 64 if kind == "s64" else 127
        raw = [int(rng.integers(0, 1 << 62)) << (lim - 62) for _ in range(1 << n)]
        vals = {"u128": [v << 1 for v in raw], "i128": [v if i % 2 else -v for i, v in enumerate(raw)],
                "s64": [(v & ((1 << 64) - 1), i % 3 != 0) for i, v in enumerate(raw)],
                "s128": [(v, i % 2 == 0) for i, v in enumerate(raw)]}[kind]
        vals[0] = {"u128": (1 << 128) - 1, "i128": -(1 << 127), "s64": (0, False), "s128": (0, False)}[kind]
        a, k, m = small_scalars(vals, kind)
        c = O.random_fr(95 + k, 1)[0]
        terms_py.append(("compact", SR.decode_column(a, kind), c))
        terms_c.append(("compact", a, k, m, c))
    for K, layout, dt in ((4, "cycle_major", np.uint8), (8, "address_major", np.uint16)):
        col = rng.integers(0, K, 1 << (n - 3)).astype(dt)
        col[::3] = np.iinfo(dt).max
        c = (1 << 125) - 7
        terms_py.append(("one_hot", SR.addresses(col), K, layout, c))
        terms_c.append(("one_hot", col, K, 0 if layout == "cycle_major" else 1, c))
    want = LR.linear_combination(terms_py, 1 << n)
    assert F.limbs_to_ints(CR.linear_combination(terms_c, 1 << n)) == want


def test_linear_combination_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_table_linear_combination")
    assert ctypes.sizeof(_lib.LcTermC) == 80   # 4 ints, table, values, len, K, coeff
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    out = ctypes.c_uint64()
    terms = (_lib.LcTermC * 1)()
    st = lib.jb_table_linear_combination(None, ctypes.cast(terms, ctypes.c_void_p), 1, 1, ctypes.byref(out))
    assert st == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


def test_lincomb_kernel_within_128_registers_no_spills():
    ents = {k: v for k, v in ptxas_entries(_need(CSRC / "lincomb.ptxas.log")).items() if "lincomb_kernel" in k}
    assert len(ents) == 1, ents
    assert all(regs <= 128 and st == 0 and ld == 0 for regs, st, ld in ents.values()), ents


def test_lincomb_kernel_has_no_local_memory():
    obj = _need(CSRC / "lincomb.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    name = next(k for k in ptxas_entries(CSRC / "lincomb.ptxas.log") if "lincomb_kernel" in k)
    sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, timeout=600).stdout
    assert "LDS" in sass   # the descriptors are staged in shared memory
    assert "LDL" not in sass and "STL" not in sass
    loops = _loops(sass)
    assert loops
    for c in loops:
        assert not any(k.startswith(("LDL", "STL")) for k in c), c
