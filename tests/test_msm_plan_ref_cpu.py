"""The MSM planner restatement and closed forms of tests/msm_plan_ref.py, without a device: weighted_sum against plain
Python integers for every scalar kind, and the case tables of tests/test_gpu_msm_plans.py against every width the
planner can pick (a retuned planner makes this test name the widths that lost their case)."""
import numpy as np
import pytest

import msm_plan_ref as P
from oracle import bn254 as O

KINDS = ["u8", "u16", "u32", "u64", "i64", "s64", "u128", "i128", "s128"]


def _plain(vals, offset=0):
    return sum(v * (offset + i + 1) for i, v in enumerate(vals)) % O.R_MOD


@pytest.mark.parametrize("kind", KINDS)
def test_weighted_sum_matches_python_ints(kind):
    for n, seed in ((1, 3), (7, 4), (1000, 5), (4099, 6)):
        col = P.random_column(kind, n, seed)
        vals = P.ints_of(kind, col)
        assert P.weighted_sum(col, kind) == _plain(vals)
        assert P.weighted_sum(col, kind, offset=12345) == _plain(vals, 12345)
    # the kind's extremes (and -0) on their own
    ex = P.records_from_ints(kind, P._extremes(kind))
    assert P.weighted_sum(ex, kind) == _plain(P.ints_of(kind, ex))


@pytest.mark.parametrize("kind", ["i64", "s64", "i128", "s128"])
def test_weighted_sum_all_negative_and_negative_zero(kind):
    bits = P.KIND_BITS[kind]
    if kind.startswith("i"):
        vals = [-(1 << (bits - 1)), -1, -2, -((1 << (bits - 1)) - 1)] * 9
    else:
        vals = [((1 << bits) - 1, False), (1, False), (1 << (bits - 1), False), (0, False)] * 9
    col = P.records_from_ints(kind, vals)
    ints = P.ints_of(kind, col)
    assert all(v <= 0 for v in ints)
    assert P.weighted_sum(col, kind) == _plain(ints)
    if kind.startswith("s"):
        zeros = P.records_from_ints(kind, [(0, False)] * 5)  # -0 contributes nothing
        assert P.weighted_sum(zeros, kind) == 0


def test_weighted_sum_field_limbs_and_rows():
    rng = np.random.Generator(np.random.PCG64(11))
    limbs = rng.integers(0, 1 << 64, size=(3, 513, 4), dtype=np.uint64)
    limbs[..., 3] &= np.uint64(((1 << 64) - 1) >> 3)
    rinv = pow(1 << 256, -1, O.R_MOD)
    for r, got in enumerate(P.weighted_sums(limbs, "fr")):
        vals = [sum(int(x) << (64 * k) for k, x in enumerate(row)) * rinv % O.R_MOD for row in limbs[r]]
        assert got == _plain(vals)
    u8 = rng.integers(0, 256, size=(5, 64), dtype=np.uint8)
    assert P.weighted_sums(u8, "u8") == [_plain([int(x) for x in row]) for row in u8]


def test_weighted_sum_large_column_stays_exact():
    """2^22 terms of the largest magnitudes: the uint64 chunk sums must not wrap."""
    n = 1 << 22
    col = P.constant_column("u64", n, (1 << 64) - 1)
    assert P.weighted_sum(col, "u64") == ((1 << 64) - 1) * (n * (n + 1) // 2) % O.R_MOD
    alt = np.where(np.arange(n) % 2 == 0, np.int64(2**63 - 1), np.int64(-(2**63 - 1)))
    assert P.weighted_sum(alt, "i64") == (2**63 - 1) * (-(n // 2)) % O.R_MOD


def test_planner_restatement_known_points():
    assert P.plan_with(16) == (16, 16, 1 << 15, 2048)
    assert P.plan_with(8, 8) == (8, 2, 128, 8)            # top-window increment: 8 bits in an 8-bit window
    assert P.plan_with(23) == (23, 12, 1 << 22, 1 << 16)  # 64-bucket segments
    assert [P.plan_for(1 << lg)[0] for lg in (6, 7, 8, 9, 10, 12, 13, 15, 18, 20)] == [4, 5, 6, 7, 8, 9, 10, 13, 15, 16]
    assert P.shared_window_for(1 << 24) == 22 and P.shared_window_for((1 << 16) + 1) == 16
    assert P.chunk_plan((1 << 18) - 1) == (64, 64) and P.chunk_plan(1 << 18) == (128, 64)
    assert P.chunk_plan(1 << 20, 64) == (64, 16384) and P.chunk_plan(1 << 20, 254, rows=2) == (64, 64)
    assert P.scatter_mode((1 << 21) - 1, 16, 16, False) == 0 and P.scatter_mode(1 << 21, 16, 16, False) == 1
    assert P.row_pass_rows(64, 8) == 32768 and P.row_pass_rows(1 << 13, 254) == 1024


def _field_cases():
    return {P.path_for(n)[1] for n in P.FIELD_PER_WINDOW_N}


def test_field_cases_cover_every_width_at_both_ends():
    picked = P.widths_picked(254, 25)
    assert sorted(picked) == [4, 5, 6, 7, 8, 9, 10, 13, 15, 16]
    ns = set(P.FIELD_PER_WINDOW_N)
    for c, (lo, hi) in picked.items():
        assert lo in ns, f"field width {c}: no case at its smallest n {lo}"
        if c != 16:
            assert hi in ns, f"field width {c}: no case at its largest n {hi}"
        assert any(lo < n < hi and n % 2 for n in ns), f"field width {c}: no odd n inside its range"
    assert _field_cases() == set(picked)
    # the chunk switch and the scatter mode switch, on both sides
    assert {P.chunk_plan(n)[0] for n in ((1 << 18) - 1, 1 << 18)} == {64, 128} and {(1 << 18) - 1, 1 << 18} <= ns
    modes = {P.scatter_mode(n, *P.path_for(n)[1:], False) for n in ((1 << 21) - 1, 1 << 21)}
    assert modes == {0, 1} and {(1 << 21) - 1, 1 << 21} <= ns


@pytest.mark.parametrize("bits", [8, 16, 32, 64, 128])
def test_small_cases_cover_every_width(bits):
    picked = set(P.widths_picked(bits, 25))
    have = {P.path_for(n, bits=bits)[1] for b, n in P.SMALL_PER_WINDOW if b == bits}
    assert have == picked, f"{bits}-bit kinds: widths without a case: {sorted(picked - have)}"
    # scatter mode 1 of the aggregated scatter at the class's power-of-two threshold
    mode1 = [(k, n) for k, n in P.SMALL_MODE1 if P.KIND_BITS[k] == bits]
    assert mode1
    for k, n in mode1:
        _, c, W = P.path_for(n, bits=bits)
        assert P.scatter_mode(n, c, W, False) == 1 and P.scatter_mode(n // 2, *P.path_for(n // 2, bits=bits)[1:], False) == 0


def test_shared_cases_cover_every_table_width():
    assert P.SHARED_WIDTHS == list(range(8, 24))
    for c in P.SHARED_WIDTHS:
        srs = P.shared_srs_len(c)
        small = P.small_table_len(srs)
        on, below = P.shared_edge_n(c)
        assert P.path_for(on, srs_n=srs, pre_c=c, small_len=small)[:2] == ("shared", c)
        path_below = P.path_for(below, srs_n=srs, pre_c=c, small_len=small)[0]
        assert path_below == ("small" if c <= 16 else "per_window")
    # c = 23: the 4 Mi-bucket scan, 64-bucket segments and more than 2048 segments (a two-level tree)
    c, W, B, T = P.plan_with(23)
    assert B == 1 << 22 and P.seg_size(B) == 64 and T > 2048
    for n in P.SHARED_C23_N:
        assert P.path_for(n, srs_n=1 << 20, pre_c=23, small_len=1 << 15)[:2] == ("shared", 23)
    # field mode 2 on both sides of its threshold
    for c in (16, 20):
        got = sorted(P.scatter_mode(n, c, P.plan_with(c)[1], True) for cc, n in P.SHARED_MODE2 if cc == c)
        assert got == [0, 2]
    kind, c, n = P.SHARED_MODE2_SMALL
    W = P.plan_with(c, P.KIND_BITS[kind])[1]
    assert P.scatter_mode(n, c, W, True) == 2 and P.scatter_mode(n - 1, c, W, True) == 0
    assert {P.KIND_BITS[k] for k, _ in P.SHARED_SMALL} == {8, 16, 32, 64, 128}
