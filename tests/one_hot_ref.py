"""Reference for the one-hot row commitments (jb_msm_g1_one_hot_rows), restated from the definition in
include/jolt_b200.h on top of the oracle's G1 addition. Pinned by tests/test_one_hot_cpu.py against the materialised
0/1 matrix and the oracle's naive MSM; tests/test_gpu_one_hot.py compares the device against it."""
from oracle import bn254 as O

ONE_HOT_LAYOUTS = ("cycle_major", "address_major")


def one_hot_row_sets(addr, K: int, T: int, W: int, layout: str):
    """Dory tier-1 rows of a one-hot polynomial from its address column: addr[j] is the address cycle j touched, or None
    if it touched none; coefficient (k, j) is 1 iff addr[j] == k. The flat coefficient index is j K + k under
    JB_ONE_HOT_CYCLE_MAJOR ("cycle_major") and k T + j under JB_ONE_HOT_ADDRESS_MAJOR ("address_major"); the matrix has
    R = K T / W rows of width W, and row r holds the coefficients idx with idx // W == r at column idx % W. Returns, per
    row, the sorted columns of its 1 coefficients. An address >= K raises ValueError."""
    assert layout in ONE_HOT_LAYOUTS and len(addr) == T
    assert K > 0 and T > 0 and W > 0 and (K * T) % W == 0
    sets = [[] for _ in range(K * T // W)]
    for j, k in enumerate(addr):
        if k is None:
            continue
        if not 0 <= k < K:
            raise ValueError(f"one-hot address {k} at cycle {j} is not below K = {K}")
        idx = j * K + k if layout == "cycle_major" else k * T + j
        sets[idx // W].append(idx % W)
    return [sorted(s) for s in sets]


def one_hot_row_commitments(bases, addr, K: int, T: int, W: int, layout: str):
    """C_r = the group sum of bases[c] over the columns c of row r (one_hot_row_sets), added one by one with the oracle's
    g1_add (complete: repeated and opposite points included); an empty row is the identity (None)."""
    out = []
    for cols in one_hot_row_sets(addr, K, T, W, layout):
        acc = None
        for c in cols:
            acc = O.g1_add(acc, bases[c])
        out.append(acc)
    return out
