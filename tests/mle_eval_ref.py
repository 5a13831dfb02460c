"""Big-integer references for multilinear evaluation at a point (include/jolt_b200.h: jb_table_evaluate_batch,
jb_small_evaluate_batch, jb_one_hot_evaluate, jb_one_hot_pushforward). Pinned by tests/test_mle_eval_cpu.py against
bind sequences and brute force over the hypercube; tests/test_gpu_mle_eval.py compares the device against them."""
from oracle import bn254 as O
import one_hot_ref

R = O.R_MOD


def evaluate(evals, point) -> int:
    """Polynomial::evaluate (dense.rs:339-360): sum_x f(x) eq(point, x), point[0] <-> the most significant bit."""
    assert len(evals) == 1 << len(point)
    return O.evaluate([v % R for v in evals], list(point))


def promote(v) -> int:
    """F::from(v) for a compact entry: an int (signed kinds: negatives -> r - |v|) or a sign-magnitude record
    (magnitude, is_positive) - a zero magnitude with either sign is 0."""
    if isinstance(v, (tuple, list)):
        mag, pos = int(v[0]), bool(v[1])
        return mag % R if pos else (-mag) % R
    return int(v) % R


def evaluate_small(values, point) -> int:
    return evaluate([promote(v) for v in values], point)


def one_hot_flat(addr, K: int, T: int, layout: str) -> list[int]:
    """The one-hot polynomial materialised as K T field values at one_hot_ref's flat index (j K + k cycle-major,
    k T + j address-major); addr[j] None = the cycle touched no address."""
    flat = [0] * (K * T)
    for row, cols in enumerate(one_hot_ref.one_hot_row_sets(addr, K, T, K * T, layout)):
        for c in cols:
            flat[row * K * T + c] = 1
    return flat


def split_point(point, K: int, T: int, layout: str):
    """(r_cycle, r_addr) of a one-hot evaluation point."""
    lt, lk = T.bit_length() - 1, K.bit_length() - 1
    assert len(point) == lt + lk
    return (point[:lt], point[lt:]) if layout == "cycle_major" else (point[lk:], point[:lk])


def one_hot_evaluate(addr, K: int, T: int, point, layout: str) -> int:
    return evaluate(one_hot_flat(addr, K, T, layout), point)


def one_hot_evaluate_direct(addr, K: int, T: int, point, layout: str) -> int:
    """The same value from its definition sum_j eq(r_cycle, j) eq(r_addr, addr_j), without the K T table."""
    r_cycle, r_addr = split_point(point, K, T, layout)
    eq_c, eq_a = O.eq_evals(list(r_cycle)), O.eq_evals(list(r_addr))
    return sum(eq_c[j] * eq_a[a] for j, a in enumerate(addr) if a is not None) % R


def pushforward(addr, K: int, r_cycle) -> list[int]:
    """G[k] = sum_{j: addr_j = k} eq(r_cycle, j), as a direct sum."""
    eq = O.eq_evals(list(r_cycle))
    G = [0] * K
    for j, a in enumerate(addr):
        if a is not None:
            G[a] = (G[a] + eq[j]) % R
    return G
