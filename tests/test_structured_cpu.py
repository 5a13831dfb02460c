"""CPU checks for the LT and eq+1 tables: the definitions, the split forms the kernels compute, the closed forms of
jolt_b200.LtPolynomial / EqPlusOnePolynomial and the threaded C build agree for n = 0..10 at random and extreme
points; the C entry points are exported and report no device; the new kernels use no local memory."""
import ctypes
import pathlib
import shutil
import subprocess

import numpy as np
import pytest

from jolt_b200 import EqPlusOnePolynomial, LtPolynomial, _lib
from jolt_b200 import field as F
from oracle import bn254 as O
import structured_ref as S
from test_build_artifacts import ptxas_entries

P = O.R_MOD
CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"
MAX125 = F.from_limbs(np.array([0, 0, (1 << 64) - 1, (1 << 61) - 1], dtype=np.uint64))  # largest [0,0,lo,hi]


def _points(n: int):
    """(name, coordinates, scale): random full and 125-bit points and every extreme coordinate."""
    rng = np.random.default_rng(n)
    full = O.random_fr(100 + n, n)
    short = [F.from_limbs(O.challenge_to_mont_limbs(int(rng.integers(0, 1 << 63)), int(rng.integers(0, 1 << 61))))
             for _ in range(n)]
    out = [("full", full, None), ("short", short, O.random_fr(7 + n, 1)[0])]
    for name, v in (("zero", 0), ("one", 1), ("p-1", P - 1), ("max125", MAX125)):
        out.append((name, [v] * n, None))
    out.append(("mixed", [[0, 1, P - 1, MAX125][i % 4] if i % 2 else full[i] for i in range(n)], P - 1))
    return out


@pytest.mark.parametrize("n", range(11))
def test_tables_definitions_and_split_forms_agree(n):
    for name, r, scale in _points(n):
        lt = S.lt_table(r, scale)
        assert S.lt_doubling(r, scale) == lt, name
        for s in range(1, n + 1):
            assert S.lt_split(r, scale, s) == lt, (name, s)
        assert S.lt_stream(r, scale, block=4, reg=2) == lt, name
        assert S.lt_stream(r, scale, block=5, reg=3) == lt, name
        e1 = S.eq_plus_one_table(r, scale)
        for s in range(n + 1):
            assert S.eq_plus_one_split(r, scale, s) == e1, (name, s)


def test_nvars_zero_is_zero():
    assert S.lt_table([], 5) == [0] and S.eq_plus_one_table([], 5) == [0]
    assert LtPolynomial.evaluate([], []) == 0 and EqPlusOnePolynomial.evaluate([], []) == 0


@pytest.mark.parametrize("n", range(11))
def test_closed_forms_are_the_tables(n):
    for name, r, scale in _points(n):
        sc = 1 if scale is None else scale
        lt, e1 = S.lt_table(r, scale), S.eq_plus_one_table(r, scale)
        for j in range(1 << n):
            x = S.bits(j, n)
            assert lt[j] == sc * LtPolynomial.evaluate(x, r) % P, (name, j)
            assert e1[j] == sc * EqPlusOnePolynomial.evaluate(r, x) % P, (name, j)
        # the closed forms are the tables' multilinear extensions
        rho = O.random_fr(300 + n, n)
        assert O.evaluate(lt, rho) == sc * LtPolynomial.evaluate(rho, r) % P, name
        assert O.evaluate(e1, rho) == sc * EqPlusOnePolynomial.evaluate(r, rho) % P, name
        # the sums the GPU tests check
        assert sum(lt) % P == sc * sum(ri << (n - 1 - i) for i, ri in enumerate(r)) % P, name
        prod = 1
        for ri in r:
            prod = prod * ri % P
        assert sum(e1) % P == sc * (1 - prod) % P, name


@pytest.mark.parametrize("n", range(5))
def test_closed_forms_on_the_cube(n):
    for a in range(1 << n):
        for b in range(1 << n):
            x, y = S.bits(a, n), S.bits(b, n)
            assert LtPolynomial.evaluate(x, y) == int(a < b)
            assert EqPlusOnePolynomial.evaluate(x, y) == int(b == a + 1)


def test_closed_forms_refuse_points_of_different_lengths():
    with pytest.raises(ValueError):
        LtPolynomial.evaluate([1, 2], [3])
    with pytest.raises(ValueError):
        EqPlusOnePolynomial.evaluate([1], [])


@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("n", [0, 1, 2, 5, 10, 13])
def test_c_build_matches_python(n, threads):
    for name, r, scale in _points(n)[:3] + _points(n)[-1:]:
        rl = F.ints_to_limbs(r).reshape(-1, 4)
        sl = None if scale is None else F.to_limbs(scale)
        lt = F.limbs_to_ints(S.lt_evals_c(rl, sl, threads))
        e1 = F.limbs_to_ints(S.eq_plus_one_evals_c(rl, sl, threads))
        if n <= 10:
            assert lt == S.lt_table(r, scale), name
        else:
            assert lt == S.lt_split(r, scale, 6), name
        assert e1 == S.eq_plus_one_table(r, scale), name


def test_entry_points_exported_and_no_device():
    lib = _lib.load()
    so = ctypes.CDLL(str(_lib.LIB_PATH))
    for fn in ("jb_lt_evals", "jb_eq_plus_one_evals"):
        assert hasattr(so, fn)
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    r = F.ints_to_limbs([3, 4])
    h = ctypes.c_uint64()
    for fn in (lib.jb_lt_evals, lib.jb_eq_plus_one_evals):
        assert fn(None, r.ctypes.data_as(_lib.c_u64p), 2, None, ctypes.byref(h)) == _lib.JB_ERR_NO_DEVICE


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


STRUCTURED_KERNELS = ("lt_expand_kernel", "lt_stream_kernel")


def test_structured_kernels_no_spills():
    ents = ptxas_entries(_need(CSRC / "structured.ptxas.log"))
    assert sum("lt_expand_kernel" in k for k in ents) == 1
    assert sum("lt_stream_kernel" in k for k in ents) == 4
    for name, (regs, st, ld) in ents.items():
        assert st == 0 and ld == 0, name


@pytest.mark.parametrize("kernel", STRUCTURED_KERNELS)
def test_structured_kernels_have_no_local_memory(kernel):
    obj = _need(CSRC / "structured.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    names = [k for k in ptxas_entries(CSRC / "structured.ptxas.log") if kernel in k]
    assert names
    for name in names:
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True,
                              timeout=600).stdout
        assert "EXIT" in sass and "LDL" not in sass and "STL" not in sass, name
