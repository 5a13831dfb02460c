"""Product members over sources without a GPU: a Python model of product_round_kernel's evaluation scheme (the binary
counter of merges, the backward difference tables, the k! L constants) equals the direct evaluation of
prod_i (lo_i + t D_i) at every published point; the reference member equals brute-force round sums for 7 .. 16 factors;
the kernel's register / local-memory budget; the exported symbol."""
import ctypes
import math
import random
import shutil
import subprocess

import pytest

from jolt_b200 import _lib
from oracle import bn254 as O
import source_ref as SR
from test_build_artifacts import ptxas_entries
from test_source_ref_cpu import CSRC, _need

P = O.R_MOD
INF = -1


def program(d):
    """product.cu's build_program: [("leaf", j, base) | ("merge", base, a, b)] and the column slots it needs"""
    steps, stk, slots = [], [], 0

    def merge_top():
        nonlocal slots
        (ba, a, la), (_, b, lb) = stk[-2], stk[-1]
        steps.append(("merge", ba, a, b))
        slots = max(slots, ba + 2 * (a + b) + 4)
        del stk[-2:]
        stk.append((ba, a + b, la + lb))

    for j in range(d):
        base = stk[-1][0] + stk[-1][1] + 1 if stk else 0
        steps.append(("leaf", j, base))
        slots = max(slots, base + 2)
        stk.append((base, 1, 1))
        while len(stk) >= 2 and stk[-1][2] == stk[-2][2]:
            merge_top()
    while len(stk) >= 2:
        merge_top()
    return steps, slots


class Counts:
    def __init__(self):
        self.mul = self.small = self.add = 0


def run_model(pairs, points, weight=None, cnt=None):
    """the kernel's per-pair evaluation on one column of slots: returns the values at `points` (INF = infinity)"""
    cnt = cnt or Counts()
    d = len(pairs)
    steps, slots = program(d)
    col = [None] * slots

    def mul(x, y):
        cnt.mul += 1
        return x * y % P

    def add(x, y):
        cnt.add += 1
        return (x + y) % P

    def sub(x, y):
        cnt.add += 1
        return (x - y) % P

    def table(S_, k, T):
        for j in range(k - 1):
            col[T + j] = sub(col[S_ + j + 1], col[S_ + j])
        col[T + k - 1] = col[S_ + k - 1]
        for l in range(2, k):
            for j in range(k - l):
                col[T + j] = sub(col[T + j + 1], col[T + j])
        if k > 1:
            cnt.small += 1
        col[T + k] = math.factorial(k) * col[S_ + k] % P   # double-and-add on the device

    def step(T, k):
        v = add(col[T], col[T + k])
        col[T] = v
        for j in range(1, k):
            v = add(col[T + j], v)
            col[T + j] = v
        return v

    skip1 = 1 not in points
    for si, st in enumerate(steps):
        if st[0] == "leaf":
            _, j, base = st
            lo, hi = pairs[j]
            dl = sub(hi, lo)
            if weight is not None and si == 0:
                lo, dl = mul(lo, weight), mul(dl, weight)
            col[base], col[base + 1] = lo, dl
        else:
            _, SA, a, b = st
            SB, c = SA + a + 1, a + b
            TA, TB = SB + b + 1, SB + b + 1 + a + 1
            table(SA, a, TA)
            table(SB, b, TB)
            lc = mul(col[SA + a], col[SB + b])
            for t in range(c):
                x = col[SA + t] if t < a else step(TA, a)
                z = col[SB + t] if t < b else step(TB, b)
                if skip1 and t == 1 and si == len(steps) - 1:
                    continue
                col[SA + t] = mul(x, z)
            col[SA + c] = lc
    if d == 1:
        col[1] = add(col[0], col[1])
    return [col[d if t == INF else t] for t in points]


def kernel_points(d, skip1):
    pts = [0] + ([] if skip1 else [1]) + list(range(2, d))
    return pts + ([INF] if d >= 2 else [])


def direct(pairs, t, weight=1):
    if t == INF:
        return weight * math.prod(hi - lo for lo, hi in pairs) % P
    return weight * math.prod(lo + t * (hi - lo) for lo, hi in pairs) % P


# limb extremes: 0, 1, p - 1, p - 2, (p - 1) / 2, powers of two at limb boundaries
EXTREMES = [0, 1, 2, P - 1, P - 2, (P - 1) // 2, (1 << 64) % P, (1 << 128) - 1, (1 << 192) % P, (1 << 253) % P]


@pytest.mark.parametrize("skip1", [False, True])
@pytest.mark.parametrize("d", range(1, 17))
def test_model_equals_direct_evaluation(d, skip1):
    rng = random.Random(0x51 + d)
    pts = kernel_points(d, skip1)
    for trial in range(6):
        pick = (lambda: rng.choice(EXTREMES)) if trial % 2 else (lambda: rng.randrange(P))
        pairs = [(pick(), pick()) for _ in range(d)]
        w = pick() if trial >= 3 else None
        got = run_model(pairs, pts, w)
        assert got == [direct(pairs, t, 1 if w is None else w) for t in pts], (d, trial)


def test_program_shapes():
    for d in range(1, 17):
        steps, slots = program(d)
        assert sum(s[0] == "leaf" for s in steps) == d and sum(s[0] == "merge" for s in steps) == d - 1
        assert all(s[2] <= 8 and s[3] <= 8 for s in steps if s[0] == "merge")   # children <= 8 (fact table)
        assert slots <= 36
    assert program(16)[1] == 36


def product_counts(d, eq):
    """per pair: (full Montgomery products of the tree, k! L multiples, additions / subtractions besides those multiples,
    full products of the per-point loop: (d - 1) per point plus one weighting per point with eq)"""
    cnt = Counts()
    pts = kernel_points(d, eq)
    run_model([(3, 5)] * d, pts, 7 if eq else None, cnt)
    tree = cnt.mul + (1 if eq else 0)          # + the weight e_out * e_in
    naive = len(pts) * (d - 1) + (len(pts) if eq else 0)
    return tree, cnt.small, cnt.add, naive


# (d, eq) -> full Montgomery products, k! L multiples, additions / subtractions per pair (the figures of DESIGN section 4)
COUNTS = {(8, False): (31, 6, 80, 63), (8, True): (33, 6, 80, 64), (9, True): (43, 7, 125, 81),
          (16, False): (79, 14, 344, 255), (16, True): (81, 14, 344, 256)}


@pytest.mark.parametrize("d,eq", sorted(COUNTS))
def test_product_counts(d, eq):
    assert product_counts(d, eq) == COUNTS[(d, eq)]
    tree, _, _, naive = COUNTS[(d, eq)]
    if d == 16:
        assert 2 * tree <= naive


@pytest.mark.parametrize("order", [O.HIGH_TO_LOW, O.LOW_TO_HIGH])
@pytest.mark.parametrize("d", [7, 9, 12, 16])
def test_reference_member_equals_brute_force(d, order):
    n = 3
    rng = random.Random(0x61 + d)
    tabs = [[rng.randrange(P) for _ in range(1 << n)] for _ in range(d)]
    ref = SR.SourcesMember([("table", t) for t in tabs], [(1, list(range(d)))], order)
    assert ref.degree == d
    for rnd in range(n):
        ev = ref.round_evals(None if rnd == 0 else rng.randrange(P))
        cur = ref.tables
        half = len(cur[0]) // 2
        for t in range(d + 1):
            want = 0
            for y in range(half):
                ps = [O.pair(tb, y, order) for tb in cur]
                want += math.prod(lo + t * (hi - lo) for lo, hi in ps)
            assert ev[t] == want % P, (rnd, t)


def test_create_product_sources_exported_and_no_device():
    lib = _lib.load()
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "jb_member_create_product_sources")
    assert _lib.JB_PRODUCT_MAX_FACTORS == 16
    if lib.jb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    out = ctypes.c_void_p()
    src = (_lib.SourceC * 1)()
    st = lib.jb_member_create_product_sources(None, ctypes.cast(src, ctypes.c_void_p), 1, 2, None, 0, None, 0,
                                              ctypes.byref(out))
    assert st == _lib.JB_ERR_NO_DEVICE


def _entries(name):
    return {k: v for k, v in ptxas_entries(_need(CSRC / "product.ptxas.log")).items() if name in k}


def test_product_kernels_no_spills_no_stack():
    ents = _entries("product_round_kernel")
    # 2 orders x (source read, source bind, 125-bit source bind, table bind, 125-bit table bind) x (plain, weighted)
    assert len(ents) == 20, ents
    assert all(regs <= 255 and st == 0 and ld == 0 for regs, st, ld in ents.values()), ents
    ents = _entries("source_bind_kernel")   # the terminal bind shared with sources.cu, over ProductParams
    assert len(ents) == 2 and all(st == 0 and ld == 0 for _, st, ld in ents.values()), ents
    log = (CSRC / "product.ptxas.log").read_text()
    assert "bytes stack frame" in log
    assert all(" 0 bytes stack frame" in line for line in log.splitlines() if "bytes stack frame" in line)


def test_product_kernels_have_no_local_memory():
    obj = _need(CSRC / "product.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    for name in _entries("product_round_kernel"):
        sass = subprocess.run([cuobjdump, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, timeout=600).stdout
        assert "LDS" in sass, name
        assert "LDL" not in sass and "STL" not in sass, name
