"""Big-int reference for expression members over sources (jb_member_create_expr_sources): a compact source is its
promoted table F::from(v), a one-hot source the gathered table ra(r_addr, j) = eq(r_addr, addr[j]) (0 where the cycle
touched no address), and the member is tests/expr_ref.py's ExpressionMember over those tables. Pinned by
tests/test_source_ref_cpu.py; tests/test_gpu_expr_sources.py runs the device in lockstep with it."""
import numpy as np

from oracle import bn254 as O
import expr_ref as E
import mle_eval_ref as M

P = O.R_MOD


def decode_column(a: np.ndarray, kind: str) -> list:
    """The entries of a column as small_scalars encodes it: ints, or (magnitude, is_positive) for s64 / s128."""
    if kind in ("s64", "s128"):
        limbs = 1 if kind == "s64" else 2
        return [(sum(int(r[j]) << (64 * j) for j in range(limbs)), bool(int(r[limbs]) & 0xFF)) for r in a]
    if kind in ("u128", "i128"):
        vals = [int(r[0]) | (int(r[1]) << 64) for r in a]
        return [v - (1 << 128) if kind == "i128" and v >> 127 else v for v in vals]
    return [int(v) for v in a]


def promote_column(values) -> list[int]:
    """F::from(v) of every entry (ints, or sign-magnitude records)."""
    return [M.promote(v) for v in values]


def gather_one_hot(addr, K: int, r_addr) -> list[int]:
    """ra(r_addr, j) = eq(r_addr, addr[j]); addr[j] None = the cycle touched no address."""
    eq = O.eq_evals(list(r_addr)) if len(r_addr) else [1]
    assert len(eq) == K
    return [0 if a is None else eq[a] for a in addr]


def addresses(col: np.ndarray) -> list:
    """An address column as the device reads it: the all-ones value of its width is None."""
    none = 0xFF if col.dtype == np.uint8 else 0xFFFF
    return [None if int(a) == none else int(a) for a in col]


def source_table(src) -> list[int]:
    """("table", ints) | ("compact", values) | ("one_hot", addr, K, r_addr) -> the field table it stands for."""
    if src[0] == "table":
        return [v % P for v in src[1]]
    if src[0] == "compact":
        return promote_column(src[1])
    _, addr, K, r_addr = src
    return gather_one_hot(addr, K, r_addr)


class SourcesMember(E.ExpressionMember):
    def __init__(self, sources, monomials, order=O.HIGH_TO_LOW, eq_point=None, eq_scale=None):
        super().__init__([source_table(s) for s in sources], monomials, order, eq_point, eq_scale)
