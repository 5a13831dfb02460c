"""ORACLE (test infrastructure, NOT product code) for u32 address columns (K up to 2^24), where the flat K T one-hot
polynomial and the K-entry eq table are too large for the big-integer references of tests/mle_eval_ref.py:
  * eq(r, x) of one index, the one-hot evaluation and the pushforward one cycle at a time;
  * read-write workloads with u32 address columns (tests/rw_ref.py's builders with a wider address type), and a
    small RAM workload that touches addresses 0 and K - 1.
Pinned against the flat references by tests/test_one_hot_u32_cpu.py."""
import numpy as np

from oracle import bn254 as O
import rw_ref as R

P = O.R_MOD
NONE32 = 0xFFFFFFFF


def eq_at(r, x: int) -> int:
    """eq(r, x) for one index x (r[0] <-> its most significant bit), without the 2^len(r) table."""
    n, v = len(r), 1
    for i, ri in enumerate(r):
        v = v * (ri if (x >> (n - 1 - i)) & 1 else 1 - ri) % P
    return v


def one_hot_evaluate_sparse(addr, r_cycle, r_addr) -> int:
    """sum_j eq(r_cycle, j) eq(r_addr, addr_j) over the cycles that touched an address (addr_j None: none)."""
    return sum(eq_at(r_cycle, j) * eq_at(r_addr, a) for j, a in enumerate(addr) if a is not None) % P


def pushforward_sparse(addr, r_cycle) -> dict:
    """{k: G[k]} over the addresses the column touches (G is 0 everywhere else)."""
    G = {}
    for j, a in enumerate(addr):
        if a is not None:
            G[a] = (G.get(a, 0) + eq_at(r_cycle, j)) % P
    return G


def ram_workload_with_edges(seed, K, T, none_frac=0.1):
    """A RAM workload of rw_ref's list form (one column read and written, values by the precondition) whose column
    touches address 0 at cycle 0 and K - 1 at cycle 1."""
    rng = np.random.default_rng(seed)
    ad = [None if rng.random() < none_frac else int(x) for x in rng.integers(0, K, T)]
    ad[0], ad[1] = 0, K - 1
    addrs = [ad, ad]
    write = 1
    inc = [0 if ad[j] is None else (int.from_bytes(rng.bytes(8), "little") - (1 << 63)) % P for j in range(T)]
    init = [int(x) for x in rng.integers(0, 1 << 62, K)]
    val = R.val_table(K, T, [(a, None, 0, 0) for a in addrs], write, inc, init)
    coeffs = O.random_fr(seed + 11, 2)
    accesses = [(a, [0 if a[j] is None else val[a[j]][j] for j in range(T)], coeffs[i], 1 if i == write else 0)
                for i, a in enumerate(addrs)]
    return K, T, accesses, write, inc, init


def ram_columns_workload_u32(seed, K, T, none_frac=0.05, local=False):
    """rw_ref.columns_workload's RAM shape with a u32 address column (none = 0xFFFFFFFF): u64 values
    v(j) = Val(addr(j), j) (0 at none), a u64 inc (0 at none) and u64 init. local: the addresses are a random walk
    (steps -2 .. 2, modulo K) instead of uniform."""
    rng = np.random.default_rng(seed)
    a = (np.cumsum(rng.integers(-2, 3, T)) % K if local else rng.integers(0, K, T)).astype(np.uint32)
    a[rng.random(T) < none_frac] = NONE32
    wv = a != NONE32
    inc = np.where(wv, rng.integers(0, 1 << 32, T), 0).astype(np.uint64)
    init = rng.integers(0, 1 << 40, K).astype(np.uint64)
    # Val(k, j) = init(k) + the increments of the earlier writes to k: prefix sums over the writes sorted by (k, j)
    j_all = np.arange(T, dtype=np.int64)
    k = a.astype(np.int64)
    wkey = k[wv] * T + j_all[wv]
    order = np.argsort(wkey, kind="stable")
    wkey = wkey[order]
    cum = np.concatenate([[0], np.cumsum(inc[wv][order])]).astype(np.uint64)
    s = cum[np.searchsorted(wkey, k * T + j_all, "left")] - cum[np.searchsorted(wkey, k * T, "left")]
    values = np.where(wv, init[np.minimum(k, K - 1)] + s, 0).astype(np.uint64)
    coeffs = O.random_fr(seed + 1, 2)
    return dict(K=K, T=T, addrs=[a, a], values=[values, values], coeffs=coeffs, ds=[0, 1], write=1, inc=inc,
                init=init, none=NONE32)
