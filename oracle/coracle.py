"""ORACLE (test infrastructure, NOT product code): ctypes binding to oracle/liboracle.so
(the C restatement in oracle/oracle.c). numpy arrays of uint64 limbs in, limbs out."""
from __future__ import annotations

import ctypes
import pathlib
import subprocess

import numpy as np

_HERE = pathlib.Path(__file__).resolve().parent
_LIB = None
u64p = ctypes.POINTER(ctypes.c_uint64)


def build(force: bool = False) -> pathlib.Path:
    so = _HERE / "liboracle.so"
    src = _HERE / "oracle.c"
    if force or not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.check_call(["make", "-C", str(_HERE), "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(str(build()))
        _LIB.orc_max_threads.restype = ctypes.c_int
    return _LIB


def _p(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u64p)


def max_threads() -> int:
    return lib().orc_max_threads()


def ints_to_mont(vals, p=None) -> np.ndarray:
    """list of canonical Python ints -> (n,4) uint64 Montgomery limbs (via Python big-int)."""
    from . import bn254 as O
    p = O.R_MOD if p is None else p
    out = np.empty((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        out[i] = O.to_mont_limbs(v, p)
    return out


def mont_to_ints(arr: np.ndarray, p=None) -> list[int]:
    from . import bn254 as O
    p = O.R_MOD if p is None else p
    rinv = pow(1 << 256, -1, p)
    a = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4)
    return [(sum(int(a[i, k]) << (64 * k) for k in range(4)) * rinv) % p for i in range(a.shape[0])]


def f_vec(sel: int, op: int, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    b = np.ascontiguousarray(b, dtype=np.uint64)
    o = np.empty_like(a)
    lib().orc_f_vec(sel, op, _p(o), _p(a), _p(b), ctypes.c_size_t(a.size // 4))
    return o


def to_mont(sel: int, canon: np.ndarray) -> np.ndarray:
    canon = np.ascontiguousarray(canon, dtype=np.uint64).reshape(-1, 4)
    o = np.empty_like(canon)
    for i in range(canon.shape[0]):
        lib().orc_f_to_mont(sel, _p(o[i]), _p(canon[i]))
    return o


def bind(table: np.ndarray, s: np.ndarray, order: int, threads: int = 1) -> np.ndarray:
    table = np.ascontiguousarray(table, dtype=np.uint64).reshape(-1, 4)
    n = table.shape[0]
    out = np.empty((n // 2, 4), dtype=np.uint64)
    s = np.ascontiguousarray(s, dtype=np.uint64)
    lib().orc_bind(_p(out), _p(table), ctypes.c_size_t(n), _p(s), order, threads)
    return out


def eq_evals(r: np.ndarray, scale: np.ndarray | None = None, threads: int = 1) -> np.ndarray:
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    n = r.shape[0]
    out = np.empty((1 << n, 4), dtype=np.uint64)
    sc = None if scale is None else _p(np.ascontiguousarray(scale, dtype=np.uint64))
    rp = _p(r) if n else None
    if threads > 1:
        lib().orc_eq_evals_par(_p(out), rp, n, sc, threads)
    else:
        lib().orc_eq_evals(_p(out), rp, n, sc)
    return out


def product_round_evals(tables: list[np.ndarray], degree: int, order: int, threads: int = 1) -> np.ndarray:
    tabs = [np.ascontiguousarray(t, dtype=np.uint64).reshape(-1, 4) for t in tables]
    m = len(tabs)
    n = tabs[0].shape[0]
    arr = (u64p * m)(*[_p(t) for t in tabs])
    out = np.empty((degree + 1, 4), dtype=np.uint64)
    lib().orc_product_round_evals(_p(out), arr, m, ctypes.c_size_t(n), degree, order, threads)
    return out


def g1_scalar_mul(base_xy: np.ndarray, scalar_mont: np.ndarray):
    out = np.zeros(8, dtype=np.uint64)
    inf = lib().orc_g1_scalar_mul(_p(out), _p(np.ascontiguousarray(base_xy, dtype=np.uint64)),
                                  _p(np.ascontiguousarray(scalar_mont, dtype=np.uint64)))
    return out, bool(inf)


def g1_add(a_xy: np.ndarray, b_xy: np.ndarray):
    out = np.zeros(8, dtype=np.uint64)
    inf = lib().orc_g1_add(_p(out), _p(np.ascontiguousarray(a_xy, dtype=np.uint64)),
                           _p(np.ascontiguousarray(b_xy, dtype=np.uint64)))
    return out, bool(inf)


def g1_on_curve(xy: np.ndarray) -> bool:
    return bool(lib().orc_g1_on_curve(_p(np.ascontiguousarray(xy, dtype=np.uint64))))


def g1_powers(n: int, g_xy: np.ndarray, beta_mont: np.ndarray) -> np.ndarray:
    out = np.empty((n, 8), dtype=np.uint64)
    lib().orc_g1_powers(_p(out), ctypes.c_size_t(n), _p(np.ascontiguousarray(g_xy, dtype=np.uint64)),
                        _p(np.ascontiguousarray(beta_mont, dtype=np.uint64)))
    return out


def g1_powers_fast(n: int, g_xy: np.ndarray, tau_mont: np.ndarray, threads: int | None = None) -> np.ndarray:
    """The same affine powers tau^i * g as g1_powers, from a fixed-base table of g on all host threads."""
    out = np.empty((n, 8), dtype=np.uint64)
    lib().orc_g1_powers_fast(_p(out), ctypes.c_size_t(n), _p(np.ascontiguousarray(g_xy, dtype=np.uint64)),
                             _p(np.ascontiguousarray(tau_mont, dtype=np.uint64)),
                             max_threads() if threads is None else threads)
    return out


def g1_msm_naive(bases_xy: np.ndarray, scalars_mont: np.ndarray):
    bases_xy = np.ascontiguousarray(bases_xy, dtype=np.uint64).reshape(-1, 8)
    scalars_mont = np.ascontiguousarray(scalars_mont, dtype=np.uint64).reshape(-1, 4)
    assert bases_xy.shape[0] == scalars_mont.shape[0], "msm: bases/scalars length mismatch"
    out = np.zeros(8, dtype=np.uint64)
    inf = lib().orc_g1_msm_naive(_p(out), _p(bases_xy), _p(scalars_mont), ctypes.c_size_t(bases_xy.shape[0]))
    return out, bool(inf)


def g1_msm_pippenger(bases_xy: np.ndarray, scalars_mont: np.ndarray, c: int = 0, threads: int = 1):
    bases_xy = np.ascontiguousarray(bases_xy, dtype=np.uint64).reshape(-1, 8)
    scalars_mont = np.ascontiguousarray(scalars_mont, dtype=np.uint64).reshape(-1, 4)
    assert bases_xy.shape[0] == scalars_mont.shape[0], "msm: bases/scalars length mismatch"
    out = np.zeros(8, dtype=np.uint64)
    inf = lib().orc_g1_msm_pippenger(_p(out), _p(bases_xy), _p(scalars_mont),
                                     ctypes.c_size_t(bases_xy.shape[0]), c, threads)
    return out, bool(inf)


def witness_polynomial(f: np.ndarray, u: np.ndarray) -> np.ndarray:
    f = np.ascontiguousarray(f, dtype=np.uint64).reshape(-1, 4)
    d = f.shape[0]
    h = np.zeros((max(d - 1, 0), 4), dtype=np.uint64)
    if d > 1:
        lib().orc_witness_polynomial(_p(h), _p(f), ctypes.c_size_t(d), _p(np.ascontiguousarray(u, dtype=np.uint64)))
    return h


def eval_univariate(coeffs: np.ndarray, u: np.ndarray) -> np.ndarray:
    coeffs = np.ascontiguousarray(coeffs, dtype=np.uint64).reshape(-1, 4)
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_eval_univariate(_p(out), _p(coeffs), ctypes.c_size_t(coeffs.shape[0]),
                              _p(np.ascontiguousarray(u, dtype=np.uint64)))
    return out


# ---- synthetic inputs shared by the parity tests and bench.py's CPU leg -------------------------
def rand_limbs(seed: int, n: int) -> np.ndarray:
    """n canonical Montgomery elements from numpy's PCG64: draw 256 bits and clear the top 3, so the
    raw value < 2^253 < p - every such limb pattern is a valid canonical Montgomery representative."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = rng.integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64(((1 << 64) - 1) >> 3)
    return a


def rand_challenge(seed: int) -> np.ndarray:
    """125-bit challenge as raw Montgomery limbs [0,0,lo,hi] (jolt-field/src/bn254/mod.rs:172-184)."""
    from . import bn254 as O
    st, lo = O.splitmix64(seed)
    st, hi = O.splitmix64(st)
    return np.array(O.challenge_to_mont_limbs(lo, hi), dtype=np.uint64)
