"""ORACLE (test infrastructure, NOT product code) for the LT and eq+1 tables (jb_lt_evals, jb_eq_plus_one_evals).

Big-int tables straight from the definitions, with E = scale eq(r, .) (r[0] <-> MSB):
    LT[j] = sum_{t > j} E[t]        E1[j] = E[j - 1], E1[0] = 0
the split forms the device uses, and a ctypes binding to tests/native/structured_ref.c, the threaded C build on the C
oracle's arithmetic for 2^22+ tables (compiled on first use into the temporary directory, so the tree can stay
read-only). The closed forms LT(x, y) / EqPlusOne(x, y) are jolt_b200.LtPolynomial / EqPlusOnePolynomial.evaluate;
the tests pin them against these tables."""
from __future__ import annotations

import ctypes
import hashlib
import os
import pathlib
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import bn254 as O

P = O.R_MOD
SRC = pathlib.Path(__file__).resolve().parent / "native" / "structured_ref.c"
ORACLE_C = pathlib.Path(__file__).resolve().parents[1] / "oracle" / "oracle.c"
_LIB = None


def lt_table(r: list[int], scale: int | None = None) -> list[int]:
    """The definition, term by term: O(4^n)."""
    e = O.eq_evals(r, scale)
    return [sum(e[j + 1:]) % P for j in range(len(e))]


def eq_plus_one_table(r: list[int], scale: int | None = None) -> list[int]:
    e = O.eq_evals(r, scale)
    return [0] + e[:-1]


def lt_doubling(r: list[int], scale: int | None = None) -> list[int]:
    """One variable at a time, as the single-block kernel: E'[2i+1] = E[i] r, E'[2i] = E[i] - E'[2i+1],
    LT'[2i+1] = LT[i], LT'[2i] = LT[i] + E'[2i+1]."""
    e, lt = [1 if scale is None else scale % P], [0]
    for rj in r:
        e2, lt2 = [0] * (2 * len(e)), [0] * (2 * len(e))
        for i, (v, l) in enumerate(zip(e, lt)):
            hi = v * rj % P
            e2[2 * i], e2[2 * i + 1] = (v - hi) % P, hi
            lt2[2 * i], lt2[2 * i + 1] = (l + hi) % P, l
        e, lt = e2, lt2
    return lt


def lt_split(r: list[int], scale: int | None, s: int) -> list[int]:
    """j = h 2^s + l: LT[j] = LT_hi[h] + E_hi[h] LT_lo[l], with the scale in the leading tables and LT_hi built by
    the same split, recursively."""
    n = len(r)
    if n <= s:
        return lt_doubling(r, scale)
    hv = n - s
    e_hi, lt_hi, lt_lo = O.eq_evals(r[:hv], scale), lt_split(r[:hv], scale, s), lt_doubling(r[hv:])
    return [(lt_hi[h] + e_hi[h] * lt_lo[l]) % P for h in range(1 << hv) for l in range(1 << s)]


def lt_stream(r: list[int], scale: int | None = None, block: int = 11, reg: int = 3) -> list[int]:
    """The streaming kernel's form for n > block: j = (h, k, t) over n - block, reg and block - reg variables,
    LT[j] = LT_H[h] + E_H[h] LT_reg[k] + E_H[h] eq_reg[k] LT_t[t]."""
    n = len(r)
    if n <= block:
        return lt_doubling(r, scale)
    hv = n - block
    e_h, lt_h = O.eq_evals(r[:hv], scale), lt_stream(r[:hv], scale, block, reg)
    eq_k, lt_k, lt_t = O.eq_evals(r[hv:hv + reg]), lt_doubling(r[hv:hv + reg]), lt_doubling(r[hv + reg:])
    nt = 1 << (block - reg)
    return [(lt_h[h] + e_h[h] * lt_k[k] + e_h[h] * eq_k[k] * lt_t[t]) % P
            for h in range(1 << hv) for k in range(1 << reg) for t in range(nt)]


def eq_plus_one_split(r: list[int], scale: int | None, s: int) -> list[int]:
    """E1[j] = E_hi[y_h] E_lo[y_l] with y = j - 1 = y_h 2^s + y_l."""
    n = len(r)
    hv = max(n - s, 0)
    e_hi, e_lo = O.eq_evals(r[:hv], scale), O.eq_evals(r[hv:])
    lo_bits = n - hv
    return [0] + [e_hi[y >> lo_bits] * e_lo[y & ((1 << lo_bits) - 1)] % P for y in range((1 << n) - 1)]


def bits(j: int, n: int) -> list[int]:
    """MSB first."""
    return [(j >> (n - 1 - i)) & 1 for i in range(n)]


# ---- the C build -------------------------------------------------------------------------------------------------
def lib():
    global _LIB
    if _LIB is None:
        digest = hashlib.sha256(SRC.read_bytes() + ORACLE_C.read_bytes()).hexdigest()[:16]
        so = pathlib.Path(tempfile.gettempdir()) / f"jolt_b200_structured_ref_{os.getuid()}_{digest}.so"
        if not so.exists():
            cc = shutil.which("gcc") or "cc"
            tmp = so.with_suffix(f".{os.getpid()}.tmp")
            flags = ["-O3", "-march=x86-64-v2", "-fPIC", "-std=gnu11", "-shared", "-o", str(tmp), str(SRC), "-lm"]
            if subprocess.run([cc, "-fopenmp", *flags], capture_output=True).returncode != 0:
                subprocess.check_call([cc, "-Wno-unknown-pragmas", *flags])
            os.replace(tmp, so)
        _LIB = ctypes.CDLL(str(so))
        u64p = ctypes.POINTER(ctypes.c_uint64)
        for fn in (_LIB.orc_lt_evals, _LIB.orc_eq_plus_one_evals):
            fn.argtypes = [u64p, u64p, ctypes.c_int, u64p, ctypes.c_int]
            fn.restype = None
        _LIB.orc_max_threads.restype = ctypes.c_int
    return _LIB


def _c_table(fn, r_limbs, scale_limbs, threads):
    r = np.ascontiguousarray(r_limbs, dtype=np.uint64).reshape(-1, 4)
    n = r.shape[0]
    out = np.empty((1 << n, 4), dtype=np.uint64)
    u64p = ctypes.POINTER(ctypes.c_uint64)
    sc = None if scale_limbs is None else np.ascontiguousarray(scale_limbs, dtype=np.uint64).reshape(4)
    fn(out.ctypes.data_as(u64p), r.ctypes.data_as(u64p) if n else None, n,
       sc.ctypes.data_as(u64p) if sc is not None else None, threads or lib().orc_max_threads())
    return out


def lt_evals_c(r_limbs, scale_limbs=None, threads: int = 0) -> np.ndarray:
    """(2^n, 4) Montgomery limbs of the LT table; threads = 0: all the C oracle's threads."""
    return _c_table(lib().orc_lt_evals, r_limbs, scale_limbs, threads)


def eq_plus_one_evals_c(r_limbs, scale_limbs=None, threads: int = 0) -> np.ndarray:
    return _c_table(lib().orc_eq_plus_one_evals, r_limbs, scale_limbs, threads)
