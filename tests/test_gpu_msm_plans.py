"""Every G1 MSM plan against its closed form.

msm_device (jolt_b200/csrc/msm.cu) picks a plan from its input: the path (per-window buckets, the shared bucket set
over a precomputed table, the 8-bit small table, row passes, msm_binary), the window width, the scatter mode, the
chunk plan, the segment size and the depth of the segment tree. tests/msm_plan_ref.py restates the planner; the cases
here reach every width it picks for field scalars and for each class of small-scalar kinds, every precomputed width
8..23, both sides of each switch, skewed columns whose buckets split into up to 16384 chunks, and row passes.

Every MSM runs over the synthetic bases (i + 1) * G, so its value is (sum_i v_i (i + 1) mod r) * G, exactly. Every
call's msm_accumulate timing record must carry the terms of the call and the width the restated planner predicts, so a
case the planner no longer routes where its name says fails instead of testing something else. Each test frees its
bases: the largest tables here take several GiB."""
import ctypes

import numpy as np
import pytest

import jolt_b200
import msm_plan_ref as P
from jolt_b200 import G1Bases, _lib, g1_jacobian_to_affine
from oracle import bn254 as O
from oracle import coracle as C
from gpu_util import rand_limbs

pytestmark = pytest.mark.gpu

G_LIMBS = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
G_AFF = (1, 2)
HITS = set()  # (path, kind class, width, scatter mode) of every checked call


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    s.timing_enable(True)
    yield s
    s.timing_enable(False)
    s.close()
    print("\nMSM plans reached (path, kind class, width, scatter mode):")
    for h in sorted(HITS, key=str):
        print("  ", h)


def expect_point(scalar: int):
    return O.g1_scalar_mul(G_AFF, scalar) if scalar % O.R_MOD else None


def field_column(n: int, seed: int) -> np.ndarray:
    """n canonical Montgomery scalars, starting with 0, 1, 2 and r - 1."""
    col = rand_limbs(seed, n)
    edge = C.ints_to_mont([0, 1, 2, O.R_MOD - 1])
    col[: min(n, 4)] = edge[: min(n, 4)]
    return col


def msm_column(sess, bases: G1Bases, col: np.ndarray, kind: str, offset: int = 0) -> np.ndarray:
    """One MSM of a column in its device layout: jb_msm_g1 for field limbs, jb_msm_g1_small otherwise (numpy-built
    records, without small_scalars' per-element loop)."""
    if kind == "fr":
        return bases.msm(col, offset=offset)
    a = np.ascontiguousarray(col)
    out = np.zeros(12, dtype=np.uint64)
    sess.check(sess.lib.jb_msm_g1_small(sess.h, bases.handle, offset, a.ctypes.data_as(ctypes.c_void_p), a.shape[0],
                                        jolt_b200.SCALAR_KINDS[kind], out.ctypes.data_as(_lib.c_u64p)))
    return out


def accumulate_records(sess) -> list[tuple[int, int]]:
    return [(t["items"], t["m"]) for t in sess.timing_collect() if t["kind"] == "msm_accumulate"]


def kind_class(kind: str) -> str:
    return "fr" if kind == "fr" else f"{P.KIND_BITS[kind]}-bit"


def check(sess, bases, col, kind, plan, offset=0):
    """MSM of `col` over bases[offset ..] == closed form, and the call took `plan` = (path, c, W) of path_for (or
    ("binary", 1, 1): msm_binary's record carries window 1)."""
    n = col.shape[0]
    path, c, W = plan
    sess.timing_collect()
    out = msm_column(sess, bases, col, kind, offset)
    recs = accumulate_records(sess)
    assert recs == [(n, c)], f"{kind} n={n} offset={offset}: the planner predicts {plan}; the call recorded {recs}"
    assert g1_jacobian_to_affine(out) == expect_point(P.weighted_sum(col, kind, offset)), f"{kind} n={n} {plan}"
    mode = P.scatter_mode(n, c, W, path in ("shared", "small")) if path != "binary" else 0
    HITS.add((path, kind_class(kind), c, mode))


# ---- A. per-window path, field scalars -------------------------------------------------------------------------------
@pytest.mark.parametrize("n", P.FIELD_PER_WINDOW_N)
def test_field_per_window_widths(sess, n):
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n)
    try:
        check(sess, bases, field_column(n, 0xA000 + n), "fr", P.path_for(n, srs_n=n))
    finally:
        bases.free()


# ---- B. per-window path, small kinds ---------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,n", P.SMALL_PER_WINDOW)
def test_small_kinds_per_window_widths(sess, bits, n):
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n)
    try:
        for kind in (P.UNSIGNED_OF[bits],) + P.SIGNED_KINDS.get(bits, ()):
            check(sess, bases, P.random_column(kind, n, 0xB000 + n + bits), kind, P.path_for(n, srs_n=n, bits=bits))
    finally:
        bases.free()


@pytest.mark.parametrize("kind,n", P.SMALL_MODE1)
def test_small_kinds_scatter_mode1(sess, kind, n):
    """The aggregated scatter (equal slots of a warp share one atomic) with one grid row per window."""
    plan = P.path_for(n, srs_n=n, bits=P.KIND_BITS[kind])
    assert P.scatter_mode(n, plan[1], plan[2], False) == 1
    col = P.random_column(kind, n, 0xB100 + n)
    if kind == "u8":
        assert int(col.max()) >= 2  # not the msm_binary arm
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n)
    try:
        check(sess, bases, col, kind, plan)
    finally:
        bases.free()


# ---- C. shared-bucket path -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", P.SHARED_WIDTHS)
def test_shared_width_and_its_threshold(sess, c):
    """precompute(c): the smallest n on the shared path, and n = 2^(c-4) - 1, which leaves it (for the 8-bit small table
    while n <= 4096, for the per-window path above)."""
    srs = P.shared_srs_len(c)
    small = P.small_table_len(srs)
    on, below = P.shared_edge_n(c)
    bases = G1Bases.generate_multiples(sess, G_LIMBS, srs).precompute(c)
    try:
        plan_on = P.path_for(on, srs_n=srs, pre_c=c, small_len=small)
        plan_below = P.path_for(below, srs_n=srs, pre_c=c, small_len=small)
        assert plan_on[:2] == ("shared", c) and plan_below[0] != "shared"
        check(sess, bases, field_column(on, 0xC000 + c), "fr", plan_on)
        check(sess, bases, field_column(below, 0xC100 + c), "fr", plan_below)
    finally:
        bases.free()


@pytest.mark.parametrize("c", [16, 20])
def test_shared_field_scatter_mode2_threshold(sess, c):
    """W n = 2^25 switches the shared scatter to one grid row per quarter of the buckets."""
    ns = sorted(n for cc, n in P.SHARED_MODE2 if cc == c)
    bases = G1Bases.generate_multiples(sess, G_LIMBS, ns[-1]).precompute(c)
    try:
        modes = set()
        for n in ns:
            plan = P.path_for(n, srs_n=ns[-1], pre_c=c, small_len=P.SMALL_TABLE_DEFAULT)
            assert plan[:2] == ("shared", c)
            modes.add(P.scatter_mode(n, c, plan[2], True))
            check(sess, bases, field_column(n, 0xC200 + n), "fr", plan)
        assert modes == {0, 2}
    finally:
        bases.free()


@pytest.mark.parametrize("c", [9, 16, 22])
def test_shared_small_kinds(sess, c):
    n = P.shared_edge_n(c)[0]
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n).precompute(c)
    try:
        for kind, cc in P.SHARED_SMALL:
            if cc == c:
                plan = P.path_for(n, srs_n=n, pre_c=c, small_len=P.small_table_len(n), bits=P.KIND_BITS[kind])
                assert plan[:2] == ("shared", c)
                check(sess, bases, P.random_column(kind, n, 0xC300 + c), kind, plan)
    finally:
        bases.free()


def test_shared_128bit_kind_scatter_mode2(sess):
    kind, c, n = P.SHARED_MODE2_SMALL
    plan = P.path_for(n, srs_n=n, pre_c=c, small_len=P.SMALL_TABLE_DEFAULT, bits=P.KIND_BITS[kind])
    assert plan[:2] == ("shared", c) and P.scatter_mode(n, c, plan[2], True) == 2
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n).precompute(c)
    try:
        check(sess, bases, P.random_column(kind, n, 0xC400), kind, plan)
    finally:
        bases.free()


# ---- D. path edges on one handle -------------------------------------------------------------------------------------
def test_path_edges_on_one_precomputed_handle(sess):
    srs = 1 << 16
    c = P.shared_window_for(srs)
    small = P.small_table_len(srs)
    assert (c, small) == (16, 1 << 15)
    bases = G1Bases.generate_multiples(sess, G_LIMBS, srs).precompute()

    def run(col, kind, offset=0, want=None):
        plan = P.path_for(col.shape[0], offset, srs, c, small, P.KIND_BITS[kind])
        if want:
            assert plan[0] == want
        check(sess, bases, col, kind, plan, offset)

    try:
        # the small table's size limit: 4096 terms against 4097
        run(field_column(4096, 0xD0), "fr", want="small")
        run(field_column(4097, 0xD1), "fr", want="shared")
        # the small table's end: offset + n at its length, and one past it
        run(field_column(1000, 0xD2), "fr", small - 1000, "small")
        run(field_column(1000, 0xD3), "fr", small - 999, "per_window")
        run(field_column(4096, 0xD4), "fr", small - 4096, "small")
        run(field_column(4096, 0xD5), "fr", small - 4095, "shared")
        # 0/1 u8 columns on both sides of the max scan: the general path below 2^14 terms, msm_binary from 2^14
        flags = (np.arange(1 << 14) % 3 == 1).astype(np.uint8)
        run(flags[: (1 << 14) - 1], "u8", want="shared")
        check(sess, bases, flags, "u8", ("binary", 1, 1))
        # a row pass with rows wider than 2^15 grows the small table; a small MSM then reaches past 2^15
        w = (1 << 15) + (1 << 14)
        vals = P.random_column("u8", 2 * w, 0xD6)
        sess.timing_collect()
        got = bases.msm_rows(vals, 2, kind="u8")
        assert accumulate_records(sess) == [(2 * w, 8)]
        want = P.weighted_sums(vals.reshape(2, w), "u8")
        assert [g1_jacobian_to_affine(r) for r in got] == [expect_point(s) for s in want]
        HITS.add(("rows", "8-bit", 8, 0))
        small = P.small_table_len(srs, w)
        run(field_column(1000, 0xD7), "fr", 40000, "small")
    finally:
        bases.free()


# ---- E. skewed small columns at scale --------------------------------------------------------------------------------
def skewed_columns(n: int):
    i = np.arange(n)
    yield "u16", P.constant_column("u16", n, 0xBEEF)                          # one bucket per window holds every term
    yield "i64", P.constant_column("i64", n, -(1 << 62) - 12345)
    yield "u64", (i % 4 == 0).astype(np.uint64)                               # one-hot: K = 4, one hot entry per cycle
    yield "i64", np.where(i % 2 == 0, np.int64(2**63 - 1), np.int64(-(2**63 - 1)))


@pytest.mark.parametrize("precomputed", [False, True], ids=["per_window", "shared"])
def test_skewed_columns_at_scale(sess, precomputed):
    """Buckets holding 2^20 .. 2^24 terms: more than 64 chunks, up to the 16384-chunk cap with chunks longer than 64
    points, folded by msm_combine_wide_kernel."""
    srs = 1 << 24
    c = 22 if precomputed else 0
    bases = G1Bases.generate_multiples(sess, G_LIMBS, srs)
    if precomputed:
        bases.precompute(c)
    try:
        for n in (1 << 22, 1 << 24):
            for kind, col in skewed_columns(n):
                plan = P.path_for(n, srs_n=srs, pre_c=c, small_len=P.small_table_len(srs) if c else 0,
                                  bits=P.KIND_BITS[kind])
                assert plan[0] == ("shared" if precomputed else "per_window")
                check(sess, bases, col, kind, plan)
    finally:
        bases.free()


# ---- F. row-batched MSMs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,rows,width", [("u8", 32769, 64), ("fr", 1025, 1 << 13)])
def test_rows_full_pass_then_lone_row(sess, kind, rows, width):
    """A full pass (32768 u8 rows of 64: 4 Mi bucket counters; 1024 field rows of 2^13), then the lone last row on the
    single-MSM path. Each row's closed form is one scalar multiplication of the C oracle."""
    bits = P.KIND_BITS[kind]
    per = P.row_pass_rows(width, bits)
    assert rows == per + 1
    if kind == "fr":
        vals = rand_limbs(0xF000 + width, rows * width)
        mat = vals.reshape(rows, width, 4)
    else:
        vals = P.random_column(kind, rows * width, 0xF000 + width)
        mat = vals.reshape(rows, width)
    bases = G1Bases.generate_multiples(sess, G_LIMBS, width)
    try:
        sess.timing_collect()
        got = bases.msm_rows(vals, rows, kind=kind)
        lone = P.path_for(width, srs_n=width, small_len=P.small_table_len(width, width), bits=bits)
        assert accumulate_records(sess) == [(per * width, 8), (width, lone[1])]
        HITS.add(("rows", kind_class(kind), 8, 0))
        HITS.add((lone[0], kind_class(kind), lone[1], 0))
        want = P.weighted_sums(mat, kind)
        mont = C.ints_to_mont(want)
        for r in range(rows):
            xy, inf = C.g1_scalar_mul(G_LIMBS, mont[r])
            exp = None if inf else (O.from_mont_limbs(xy[:4], O.Q_MOD), O.from_mont_limbs(xy[4:], O.Q_MOD))
            assert g1_jacobian_to_affine(got[r]) == exp, f"row {r}"
    finally:
        bases.free()


# ---- G. refusals -----------------------------------------------------------------------------------------------------
def test_precompute_refuses_windows_outside_8_to_23(sess):
    """c = 24 would need 2^23 bucket counters, twice what the bucket scan holds; c = 7 is below the table's range. The
    refused handle keeps the per-window path; precompute(23) then builds the widest table: a 4 Mi-counter scan,
    64-bucket segments and a two-level segment tree."""
    n = 1 << 20
    bases = G1Bases.generate_multiples(sess, G_LIMBS, n)
    try:
        for bad in (24, 7):
            with pytest.raises(jolt_b200.JoltB200Error, match=r"window bits must be in 8\.\.23") as e:
                bases.precompute(bad)
            assert e.value.status == _lib.JB_ERR_INVALID
        check(sess, bases, field_column(n, 0x6000), "fr", P.path_for(n, srs_n=n))
        bases.precompute(23)
        for m in P.SHARED_C23_N:
            plan = P.path_for(m, srs_n=n, pre_c=23, small_len=P.small_table_len(n))
            assert plan[:2] == ("shared", 23)
            check(sess, bases, field_column(m, 0x6100 + m), "fr", plan)
    finally:
        bases.free()
