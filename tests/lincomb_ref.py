"""Big-int reference for random linear combinations (jb_table_linear_combination): P[x] = sum_i c_i p_i[x] for
x < len_i, each term contributing 0 beyond its length. Terms:
    ("table", values, c)                  field values
    ("compact", values, c)                compact entries as source_ref.decode_column returns them: F::from(v)
    ("one_hot", addr, K, layout, c)       addr[j] None = no address; the K T one-hot polynomial of one_hot_ref
Pinned by tests/test_lincomb_cpu.py; tests/test_gpu_lincomb.py compares the device against it."""
from oracle import bn254 as O
import mle_eval_ref as M

P = O.R_MOD


def term_values(term) -> list[int]:
    """The field values of one term, of its own length."""
    if term[0] == "table":
        return [v % P for v in term[1]]
    if term[0] == "compact":
        return [M.promote(v) for v in term[1]]
    _, addr, K, layout, _c = term
    return M.one_hot_flat(addr, K, len(addr), layout)


def term_coeff(term) -> int:
    return term[-1] % P


def linear_combination(terms, length: int) -> list[int]:
    out = [0] * length
    for term in terms:
        vals, c = term_values(term), term_coeff(term)
        assert len(vals) <= length
        for x, v in enumerate(vals):
            out[x] = (out[x] + c * v) % P
    return out


def prefix_factor(point, n_i: int) -> int:
    """prod_{k < n - n_i} (1 - point[k]): the value at `point` of a term embedded as the prefix of the index range,
    relative to its own value at point[n - n_i:]."""
    f = 1
    for r in point[: len(point) - n_i]:
        f = f * (1 - r) % P
    return f


def combined_claim(claims, point) -> int:
    """sum_i c_i prod(1 - point_hi) v_i for (c_i, n_i, v_i) with v_i = p_i(point[n - n_i:]): P(point) of the
    combination (the claim a batched opening proves)."""
    return sum(c * prefix_factor(point, n_i) * v for c, n_i, v in claims) % P
