"""ORACLE (test infrastructure, NOT product code): ctypes binding to tests/native/lincomb_ref.c, the threaded C
restatement of jb_table_linear_combination. The library is compiled on first use into the temporary directory, so the
tree can stay read-only. Terms:
    ("table", limbs (n, 4) uint64 Montgomery, coeff)
    ("compact", raw array as small_scalars returns it, kind code, n, coeff)
    ("one_hot", address array (uint8 / uint16), K, layout code, coeff)
coeff: a Python int (taken mod r) or 4 Montgomery limbs."""
from __future__ import annotations

import ctypes
import hashlib
import os
import pathlib
import shutil
import subprocess
import tempfile

import numpy as np

from jolt_b200 import _lib
from jolt_b200 import field as F

SRC = pathlib.Path(__file__).resolve().parent / "native" / "lincomb_ref.c"
ORACLE_C = pathlib.Path(__file__).resolve().parents[1] / "oracle" / "oracle.c"
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        digest = hashlib.sha256(SRC.read_bytes() + ORACLE_C.read_bytes()).hexdigest()[:16]
        so = pathlib.Path(tempfile.gettempdir()) / f"jolt_b200_lincomb_ref_{os.getuid()}_{digest}.so"
        if not so.exists():
            cc = shutil.which("gcc") or "cc"
            tmp = so.with_suffix(f".{os.getpid()}.tmp")
            flags = ["-O3", "-march=x86-64-v2", "-fPIC", "-std=gnu11", "-shared", "-o", str(tmp), str(SRC), "-lm"]
            if subprocess.run([cc, "-fopenmp", *flags], capture_output=True).returncode != 0:
                subprocess.check_call([cc, "-Wno-unknown-pragmas", *flags])
            os.replace(tmp, so)
        _LIB = ctypes.CDLL(str(so))
        _LIB.lc_linear_combination.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p, ctypes.c_size_t,
                                               ctypes.c_size_t]
        _LIB.lc_linear_combination.restype = None
    return _LIB


def _coeff(c) -> np.ndarray:
    if isinstance(c, (int, np.integer)):
        return F.to_limbs(int(c) % F.R_MOD)
    return np.ascontiguousarray(c, dtype=np.uint64).reshape(4)


def linear_combination(terms, length: int) -> np.ndarray:
    """(length, 4) Montgomery limbs of sum_i c_i p_i."""
    arr = (_lib.LcTermC * len(terms))()
    keep = []
    for i, t in enumerate(terms):
        c = arr[i]
        if t[0] == "table":
            a = np.ascontiguousarray(t[1], dtype=np.uint64).reshape(-1, 4)
            c.type, c.len = _lib.JB_LC_TABLE, a.shape[0]
        elif t[0] == "compact":
            a = np.ascontiguousarray(t[1])
            c.type, c.kind, c.len = _lib.JB_LC_COMPACT, t[2], t[3]
        else:
            a = np.ascontiguousarray(t[1])
            c.type, c.kind, c.len, c.K, c.layout = _lib.JB_LC_ONE_HOT, 1 if a.dtype == np.uint8 else 2, a.shape[0], t[2], t[3]
        keep.append(a)
        c.values = a.ctypes.data
        c.coeff[:] = [int(x) for x in _coeff(t[-1])]
    out = np.empty((length, 4), dtype=np.uint64)
    lib().lc_linear_combination(out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), ctypes.cast(arr, ctypes.c_void_p),
                                len(terms), length)
    return out
