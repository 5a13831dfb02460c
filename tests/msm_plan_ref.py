"""Restatement of the G1 MSM planner (jolt_b200/csrc/msm.cu: plan_with, plan_for, shared_window_for and the plan
choices of msm_device) and exact closed forms for MSMs over the synthetic bases (i + 1) * G.

Over G1Bases.generate_multiples bases, an MSM of any scalar column v is ONE scalar multiplication,
    msm(v) = (sum_i v_i (i + 1) mod r) * G,
and G1 has prime order r, so comparing the device result with that point is exact. weighted_sum computes the scalar for
every column kind the device takes, in numpy over 32-bit limb halves (a 2^25-term column takes seconds).

The case tables of tests/test_gpu_msm_plans.py live here too, so that tests/test_msm_plan_ref_cpu.py can check, without a
device, that they still reach every width the planner picks."""
from __future__ import annotations

import numpy as np

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
RINV = pow(1 << 256, -1, R_MOD)  # Montgomery R^-1 mod r

KIND_BITS = {"u8": 8, "u16": 16, "u32": 32, "u64": 64, "i64": 64, "s64": 64,
             "u128": 128, "i128": 128, "s128": 128, "fr": 254}
SIGNED_KINDS = {64: ("i64", "s64"), 128: ("i128", "s128")}
UNSIGNED_OF = {8: "u8", 16: "u16", 32: "u32", 64: "u64", 128: "u128"}

SMALL_MAX = 4096             # largest MSM the 8-bit small table serves
SMALL_TABLE_DEFAULT = 1 << 15  # bases the small table covers after precompute (or the SRS length, if shorter)
MAX_CHUNKS, MAX_CHUNKS_SMALL, CHUNK = 64, 16384, 64


# ---- the planner ---------------------------------------------------------------------------------------------------
def small_kind_bits(kind: str) -> int:
    return KIND_BITS[kind]


def seg_size(buckets: int) -> int:
    return 64 if buckets >= 1 << 21 else 16


def plan_with(c: int, bits: int = 254) -> tuple[int, int, int, int]:
    """(c, W, B, T): window bits, windows, buckets per window, segments per window."""
    W = (bits + c - 1) // c
    if bits - (W - 1) * c > c - 1:
        W += 1  # top window: data < 2^(c-1), so data + carry <= 2^(c-1) = B
    B = 1 << (c - 1)
    T = (B + seg_size(B) - 1) // seg_size(B)
    return c, W, B, T


def shared_window_for(srs_len: int) -> int:
    lg = srs_len.bit_length() - 1
    if lg >= 24:
        return 22
    if lg >= 20:
        return 20
    if lg >= 18:
        return 17
    if lg >= 16:
        return 16
    return 15


def plan_for(n: int, bits: int = 254) -> tuple[int, int, int, int]:
    lg = n.bit_length() - 1 if n > 0 else 0
    c0 = lg - 4
    small = bits < 254
    best, best_c = 0.0, 0
    for c in range(4 if small else c0 - 2, (16 if small else c0 + 2) + 1):
        if c < 4 or c > 16:
            continue
        _, W, B, _ = plan_with(c, bits)
        top_bits = max(bits - (W - 1) * c, 1)
        cnt_top = n / (1 << (top_bits - 1))
        chunk = 64.0 if cnt_top / 64.0 < 64.0 else cnt_top / 64.0
        if small and n / B / 64.0 > chunk:
            chunk = n / B / 64.0
        cost = W * n + 2.8 * W * B + 750.0 * chunk
        if best_c == 0 or cost < best:
            best, best_c = cost, c
    if best_c == 0:
        best_c = 4 if c0 < 4 else 16
    return plan_with(best_c, bits)


def path_for(n: int, offset: int = 0, srs_n: int | None = None, pre_c: int = 0, small_len: int = 0,
             bits: int = 254, rows: int = 1) -> tuple[str, int, int]:
    """(path, c, W) of one msm_device call: "rows" (row-batched, 8-bit table), "small" (8-bit table), "shared"
    (precomputed table of width pre_c) or "per_window". pre_c = 0: no precomputed table; small_len = 0: no small
    table. For a row pass, n is the pass's terms (rows x width)."""
    assert srs_n is None or offset + (n if rows == 1 else n // rows) <= srs_n
    if rows > 1:
        return ("rows",) + plan_with(8, bits)[:2]
    if small_len and n <= SMALL_MAX and offset + n <= small_len:
        return ("small",) + plan_with(8, bits)[:2]
    if pre_c and n >= 1 << (pre_c - 4):
        return ("shared",) + plan_with(pre_c, bits)[:2]
    return ("per_window",) + plan_for(n, bits)[:2]


def small_table_len(srs_n: int, want: int = 0) -> int:
    """Bases the 8-bit table covers after build_small_table(want) on an SRS of srs_n bases (0 before)."""
    return min(max(min(srs_n, SMALL_TABLE_DEFAULT), want), srs_n)


def scatter_mode(n: int, c: int, W: int, shared: bool, rows: int = 1) -> int:
    """0: every window per thread; 1: one grid row per window; 2: one grid row per quarter of the shared buckets."""
    if rows > 1 or W * n < 1 << 25:
        return 0
    if not shared:
        return 1
    return 2 if c - 1 >= 6 else 0


def chunk_plan(n: int, bits: int = 254, rows: int = 1) -> tuple[int, int]:
    """(smallest chunk, chunk cap) of the accumulation's task plan."""
    if bits == 254 or rows > 1:
        return (128 if bits == 254 and rows == 1 and n >= 1 << 18 else CHUNK), MAX_CHUNKS
    return CHUNK, MAX_CHUNKS_SMALL


def row_pass_rows(row_w: int, bits: int) -> int:
    """Rows per pass of jb_msm_g1_rows."""
    W = plan_with(8, bits)[1]
    return max(2, min((1 << 28) // (W * row_w), 32768))


def width_ranges(bits: int, lg_max: int = 25) -> list[tuple[int, int, int]]:
    """[(c, first n, last n)]: the per-window planner's width over n in [1, 2^lg_max], as maximal runs. The cost model
    reads n itself, so widths change inside a power-of-two range too: every such range is sampled and each change
    between neighbouring samples is located exactly by bisection."""
    def width(n):
        return plan_for(n, bits)[0]

    runs: list[list[int]] = []

    def extend(n_lo, n_hi):  # [n_lo, n_hi]: width(n_lo) is known to start or continue the last run
        c_hi = width(n_hi)
        if c_hi == runs[-1][0]:
            runs[-1][2] = n_hi
            return
        lo, hi = n_lo, n_hi  # width(lo) == runs[-1][0] != width(hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if width(mid) == runs[-1][0]:
                lo = mid
            else:
                hi = mid
        runs[-1][2] = lo
        runs.append([width(hi), hi, hi])
        extend(hi, n_hi)

    runs.append([width(1), 1, 1])
    for lg in range(lg_max + 1):
        a, b = 1 << lg, min((1 << (lg + 1)) - 1, 1 << lg_max)
        pts = sorted({a, b} | {a + (b - a) * k // 256 for k in range(257)})
        prev = runs[-1][2]
        for x in pts:
            if x > prev:
                extend(prev, x)
                prev = x
    return [tuple(r) for r in runs]


def widths_picked(bits: int, lg_max: int = 25) -> dict[int, tuple[int, int]]:
    """{c: (smallest n, largest n <= 2^lg_max)} over n in [1, 2^lg_max] for the per-window planner."""
    out: dict[int, tuple[int, int]] = {}
    for c, lo, hi in width_ranges(bits, lg_max):
        out[c] = (min(lo, out.get(c, (lo, hi))[0]), max(hi, out.get(c, (lo, hi))[1]))
    return out


# ---- closed forms ----------------------------------------------------------------------------------------------------
def _halves(values: np.ndarray, kind: str) -> tuple[list[tuple[int, np.ndarray]], np.ndarray | None]:
    """[(bit shift, 32-bit part as uint64)], negative mask (None: no sign) of a column in its device layout.
    `values` may carry a leading rows axis."""
    M32 = np.uint64(0xFFFFFFFF)
    v = np.asarray(values)
    words: list[np.ndarray]
    neg = None
    if kind == "fr":
        words = [v[..., k].astype(np.uint64) for k in range(4)]
    elif kind in ("u8", "u16", "u32", "u64"):
        words = [v.astype(np.uint64)]
    elif kind == "i64":
        u = v.view(np.uint64)
        neg = (u >> np.uint64(63)) != 0
        words = [np.where(neg, np.uint64(0) - u, u)]
    elif kind in ("u128", "i128"):
        lo, hi = v[..., 0].astype(np.uint64), v[..., 1].astype(np.uint64)
        if kind == "i128":
            neg = (hi >> np.uint64(63)) != 0
            nlo = np.uint64(0) - lo  # two's-complement negate over 128 bits
            nhi = ~hi + (lo == 0).astype(np.uint64)
            lo, hi = np.where(neg, nlo, lo), np.where(neg, nhi, hi)
        words = [lo, hi]
    elif kind in ("s64", "s128"):
        limbs = 1 if kind == "s64" else 2
        words = [v[..., j].astype(np.uint64) for j in range(limbs)]
        nonzero = np.zeros(words[0].shape, dtype=bool)
        for w in words:
            nonzero |= w != 0
        neg = ((v[..., limbs] & np.uint64(0xFF)) == 0) & nonzero  # is_positive == false; -0 is 0
    else:
        raise ValueError(kind)
    parts = []
    for k, w in enumerate(words):
        parts.append((64 * k, w & M32))
        parts.append((64 * k + 32, w >> np.uint64(32)))
    return parts, neg


def _weighted_part_sums(part: np.ndarray, mask: np.ndarray | None, offset: int) -> list[int]:
    """Per row: sum_i part[i] (offset + i + 1) [mask[i]] as Python ints. part < 2^32 and offset + i + 1 <= 2^26, so
    32-term chunks of products stay below 2^63; the chunk sums are split into 32-bit halves and summed again in uint64."""
    p2 = part.reshape(-1, part.shape[-1])
    m2 = None if mask is None else mask.reshape(-1, part.shape[-1])
    rows, n = p2.shape
    assert offset + n <= 1 << 26
    lo_tot = np.zeros(rows, dtype=np.uint64)
    hi_tot = np.zeros(rows, dtype=np.uint64)
    step = 1 << 21  # column block: bounds the temporaries
    for s in range(0, n, step):
        e = min(n, s + step)
        prod = p2[:, s:e] * np.arange(offset + s + 1, offset + e + 1, dtype=np.uint64)
        if m2 is not None:
            prod = np.where(m2[:, s:e], prod, np.uint64(0))
        pad = (-(e - s)) % 32
        if pad:
            prod = np.concatenate([prod, np.zeros((rows, pad), dtype=np.uint64)], axis=1)
        chunks = prod.reshape(rows, -1, 32).sum(axis=2, dtype=np.uint64)
        lo_tot += (chunks & np.uint64(0xFFFFFFFF)).sum(axis=1, dtype=np.uint64)
        hi_tot += (chunks >> np.uint64(32)).sum(axis=1, dtype=np.uint64)
    return [int(a) + (int(b) << 32) for a, b in zip(lo_tot, hi_tot)]


def weighted_sums(values: np.ndarray, kind: str, offset: int = 0) -> list[int]:
    """sum_i v_i (offset + i + 1) mod r for every row of `values` (device layout with a leading rows axis): the
    closed-form scalar of each row's MSM over bases[offset ..] of (i + 1) * G. fr rows are Montgomery limbs, decoded
    once at the end."""
    parts, neg = _halves(values, kind)
    rows = parts[0][1].reshape(-1, parts[0][1].shape[-1]).shape[0]
    total = [0] * rows
    for shift, part in parts:
        if neg is None:
            for r, s in enumerate(_weighted_part_sums(part, None, offset)):
                total[r] += s << shift
        else:
            pos_s = _weighted_part_sums(part, ~neg, offset)
            neg_s = _weighted_part_sums(part, neg, offset)
            for r in range(rows):
                total[r] += (pos_s[r] - neg_s[r]) << shift
    if kind == "fr":
        return [t * RINV % R_MOD for t in total]
    return [t % R_MOD for t in total]


def weighted_sum(values: np.ndarray, kind: str, offset: int = 0) -> int:
    """sum_i v_i (offset + i + 1) mod r of one column in its device layout (see weighted_sums)."""
    v = np.asarray(values)
    if v.shape[0] == 0:
        return 0
    return weighted_sums(v[None, ...], kind, offset)[0]


# ---- device records (the layouts jb_msm_g1_small reads; small_scalars builds them element by element) -----------------
def wide_records(lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """u128 / i128 column (i128 in two's complement): (n, 2) uint64 lo, hi."""
    return np.ascontiguousarray(np.stack([lo.astype(np.uint64), hi.astype(np.uint64)], axis=-1))


def s64_records(mag: np.ndarray, positive: np.ndarray) -> np.ndarray:
    """jb_s64: one magnitude word, then the is_positive byte (padded to a word)."""
    return np.ascontiguousarray(np.stack([mag.astype(np.uint64), positive.astype(np.uint64)], axis=-1))


def s128_records(lo: np.ndarray, hi: np.ndarray, positive: np.ndarray) -> np.ndarray:
    """jb_s128: two magnitude words, then the is_positive byte (padded to a word)."""
    return np.ascontiguousarray(np.stack([lo.astype(np.uint64), hi.astype(np.uint64), positive.astype(np.uint64)],
                                         axis=-1))


_U64_MAX = (1 << 64) - 1


def _extremes(kind: str) -> list:
    """Each kind's extreme values (Python ints; sign-magnitude kinds as (magnitude, is_positive), (0, False) = -0)."""
    bits = KIND_BITS[kind]
    if kind.startswith("u"):
        top = (1 << bits) - 1
        return [top, 0, 1, top - 1, 1 << (bits - 1), (1 << (bits - 1)) - 1, 2]
    if kind in ("i64", "i128"):
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        return [lo, hi, -1, 0, 1, lo + 1, 2]
    top = (1 << bits) - 1
    return [(top, True), (top, False), (0, False), (0, True), (1, False), (1 << (bits - 1), False), (2, True)]


def records_from_ints(kind: str, vals: list) -> np.ndarray:
    """A short column from Python ints (sign-magnitude kinds: (magnitude, is_positive) pairs) in device layout."""
    if kind in ("u8", "u16", "u32", "u64"):
        return np.array(vals, dtype={"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64}[kind])
    if kind == "i64":
        return np.array(vals, dtype=np.int64)
    if kind in ("u128", "i128"):
        w = [v & ((1 << 128) - 1) for v in vals]
        return wide_records(np.array([x & _U64_MAX for x in w], dtype=np.uint64), np.array([x >> 64 for x in w], dtype=np.uint64))
    mags = [m for m, _ in vals]
    pos = np.array([p for _, p in vals], dtype=bool)
    if kind == "s64":
        return s64_records(np.array(mags, dtype=np.uint64), pos)
    return s128_records(np.array([m & _U64_MAX for m in mags], dtype=np.uint64), np.array([m >> 64 for m in mags], dtype=np.uint64), pos)


def ints_of(kind: str, rec: np.ndarray) -> list[int]:
    """The signed integer values of a column in device layout (slow; for short columns and the CPU tests)."""
    if kind in ("u8", "u16", "u32", "u64", "i64"):
        return [int(x) for x in rec]
    if kind in ("u128", "i128"):
        out = [int(a) | (int(b) << 64) for a, b in rec]
        return [x - (1 << 128) if kind == "i128" and x >> 127 else x for x in out]
    limbs = 1 if kind == "s64" else 2
    out = []
    for r in rec:
        mag = sum(int(r[j]) << (64 * j) for j in range(limbs))
        out.append(mag if int(r[limbs]) & 0xFF else -mag)
    return out


def random_column(kind: str, n: int, seed: int, extremes: bool = True) -> np.ndarray:
    """n uniformly random values of `kind` over its whole range in device layout, the kind's extremes (and -0 for the
    sign-magnitude kinds) spread over the column."""
    rng = np.random.Generator(np.random.PCG64(seed))
    bits = KIND_BITS[kind]
    if kind in ("u8", "u16", "u32", "u64"):
        dt = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64}[kind]
        col = np.frombuffer(rng.bytes(n * (bits // 8)), dtype=dt).copy()
    elif kind == "i64":
        col = np.frombuffer(rng.bytes(n * 8), dtype=np.int64).copy()
    elif kind in ("u128", "i128"):
        col = np.frombuffer(rng.bytes(n * 16), dtype=np.uint64).reshape(n, 2).copy()
    else:
        limbs = 1 if kind == "s64" else 2
        mag = np.frombuffer(rng.bytes(n * 8 * limbs), dtype=np.uint64).reshape(n, limbs)
        pos = rng.integers(0, 2, size=n, dtype=np.uint64)
        col = np.ascontiguousarray(np.concatenate([mag, pos[:, None]], axis=1))
    if extremes and n:
        ex = records_from_ints(kind, _extremes(kind))
        at = np.linspace(0, n - 1, num=min(len(ex), n)).astype(np.int64)
        col[at] = ex[: len(at)]
    return col


def constant_column(kind: str, n: int, value) -> np.ndarray:
    rec = records_from_ints(kind, [value])
    return np.ascontiguousarray(np.repeat(rec, n, axis=0))


# ---- the case tables of tests/test_gpu_msm_plans.py -------------------------------------------------------------------
# A. per-window path, field scalars: every width at the smallest and largest n that pick it, plus one odd n; the
#    64- / 128-point chunk edge (2^18 - 1, 2^18) and the scatter mode 0 / 1 edge (2^21 - 1, 2^21).
FIELD_PER_WINDOW_N = [1, 65, 127, 128, 191, 255, 256, 383, 511, 512, 767, 1023, 1024, 2065, 3106, 3107, 4301, 5495,
                      5496, 19131, 32767, 32768, 108135, 183500, 183501, 262143, 262144, 435815, 688128, 688129,
                      1392641, 2097151, 2097152]

# B. per-window path, small kinds: (bits class, n) for every width the class picks (the largest n that picks it; the
#    smallest for the open-ended top width), run for the unsigned and the signed kinds of that width; then scatter
#    mode 1 at its power-of-two threshold per class.
SMALL_PER_WINDOW = [(8, 22), (8, 627), (8, 628),
                    (16, 67), (16, 89), (16, 1164), (16, 1165),
                    (32, 56), (32, 224), (32, 358), (32, 1971), (32, 5734), (32, 5735),
                    (64, 50), (64, 201), (64, 806), (64, 1433), (64, 2508), (64, 4112), (64, 7168), (64, 40140),
                    (64, 40141),
                    (128, 60), (128, 201), (128, 477), (128, 1344), (128, 2329), (128, 3942), (128, 15769),
                    (128, 28672), (128, 51609), (128, 298188), (128, 298189)]
SMALL_MODE1 = [("u128", 1 << 22), ("u64", 1 << 23), ("i64", 1 << 23), ("u16", 1 << 24), ("u32", 1 << 24),
               ("u8", 1 << 25)]

# C. shared-bucket path: every table width 8..23 at the smallest n on the shared path (and one below it, which leaves
#    it); c = 23 at 2^19 and 2^20; field scatter mode 2 on both sides of its threshold; each bits class at c = 9, 16, 22.
SHARED_WIDTHS = list(range(8, 24))
SHARED_C23_N = [1 << 19, 1 << 20]
SHARED_MODE2 = [(16, -(-(1 << 25) // 16) - 1), (16, -(-(1 << 25) // 16)), (20, -(-(1 << 25) // 13) - 1),
                (20, -(-(1 << 25) // 13))]
SHARED_SMALL = [(kind, c) for kind in ("u8", "u16", "u32", "i64", "s128") for c in (9, 16, 22)]
SHARED_MODE2_SMALL = ("u128", 22, -(-(1 << 25) // 6))  # W = 6 for 128-bit magnitudes at c = 22


def shared_srs_len(c: int) -> int:
    """Bases for the c-sweep: one more than the shared path's smallest n, so both n and n - 1 fit."""
    return (1 << max(c - 4, 13)) + 1


def shared_edge_n(c: int) -> tuple[int, int]:
    """(smallest n on the shared path, the n just below the shared threshold)."""
    return max(1 << (c - 4), SMALL_MAX + 1), (1 << (c - 4)) - 1
