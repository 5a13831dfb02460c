"""One-hot row commitments on one GPU: jb_msm_g1_one_hot_rows against the route callers had before it - numpy index sets
per Dory row built on the host, then jb_g1_batch_add - over the same polynomials, after checking that both give the
same points for every row. Workloads: T in {2^20, 2^22, 2^24}, K in {16 (u8), 256 (u16)}, both layouts, count in
{1, 8}, uniform columns and columns where 90 % of the cycles hit one address; Dory row width W = 2^ceil(log2(K T) / 2).

Reports per workload the new call's wall time (ends in a synchronise; median of 10 after a warm-up), its accumulation
kernel time (CUDA events), the batch_add route's time (median of 3: index sets + upload + levels), and the new call
against the accumulation bound: one mixed XYZZ addition (~10 Fq products) per hot entry at ~60 G Fq products/s.
The bases are random-looking points (random Fr combinations of (i + 1) G), so batch_add's distinct-x precondition holds.
Reads the card's name and power limit in the same run. Output: one JSON line per workload on stdout, and in FILE with --out.

usage: python tools/one_hot_bench.py [--log-t 20 22 24] [--K 16 256] [--out FILE]"""
import argparse
import ctypes
import json
import pathlib
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import jolt_b200  # noqa: E402
from jolt_b200 import G1Bases, ONE_HOT_NONE  # noqa: E402
from jolt_b200.api import _p  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from oracle import coracle as C  # noqa: E402

FQ_PRODUCTS_PER_S = 60e9      # measured Montgomery-product rate of the integer pipes (DESIGN.md section 6)
PRODUCTS_PER_ADD = 10         # mixed XYZZ addition: 8M + 2S


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return f"unknown ({e})", "unknown"


def make_column(K, T, dtype, seed, skewed):
    rng = np.random.Generator(np.random.PCG64(seed))
    col = rng.integers(0, K, size=T).astype(dtype)
    if skewed:
        col[rng.random(T) < 0.9] = 3
    return col


def host_sets(cols, K, W, layout):
    """The previous route's host work: flat indices, rows, and the columns of every row in row order (counting sort)."""
    T = cols[0].shape[0]
    R = K * T // W
    lw = W.bit_length() - 1
    flats, counts = [], []
    for col in cols:
        hot = col != ONE_HOT_NONE[col.dtype]
        j = np.nonzero(hot)[0].astype(np.int64)
        k = col[hot].astype(np.int64)
        idx = j * K + k if layout == "cycle_major" else k * T + j
        rows = idx >> lw
        order = np.argsort(rows.astype(np.uint32 if R > (1 << 16) else np.uint16), kind="stable")
        flats.append((idx[order] & (W - 1)).astype(np.uint32))
        counts.append(np.bincount(rows, minlength=R))
    offs = np.zeros(len(cols) * R + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(np.concatenate(counts))
    return offs, np.ascontiguousarray(np.concatenate(flats))


def batch_add_route(sess, bases, cols, K, W, layout):
    offs, flat = host_sets(cols, K, W, layout)
    nsets = offs.shape[0] - 1
    out = np.zeros((nsets, 8), dtype=np.uint64)
    sess.check(sess.lib.jb_g1_batch_add(sess.h, bases.handle, _p(offs), flat.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)),
                                        nsets, _p(out)))
    return out


def random_bases(sess, n):
    """n random-looking affine points: row r of a row-batched MSM of random Fr scalars against (i + 1) G."""
    G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
    gen = G1Bases.generate_multiples(sess, G, 16)
    xyz = gen.msm_rows(C.rand_limbs(0x0E07, n * 16), n, "fr")
    gen.free()
    return G1Bases.from_jacobian(sess, xyz)


def main():
    ap = argparse.ArgumentParser(description="one-hot row commitments vs host index sets + batch_add")
    ap.add_argument("--log-t", type=int, nargs="+", default=[20, 22, 24], help="log2 of the cycle counts T")
    ap.add_argument("--K", type=int, nargs="+", default=[16, 256], choices=[16, 256], help="address counts")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    name, power = card()
    sess = jolt_b200.Session(0)
    bases = random_bases(sess, 1 << 16)
    out = []
    for log_t in args.log_t:
        T = 1 << log_t
        for K, dtype in ((k, np.uint8 if k < 256 else np.uint16) for k in args.K):
            log_kt = K.bit_length() - 1 + log_t
            W = 1 << ((log_kt + 1) // 2)
            for skewed in (False, True):
                cols8 = [make_column(K, T, dtype, 100 * log_t + 10 * p + skewed, skewed) for p in range(8)]
                for count in (1, 8):
                    cols = cols8[:count]
                    hot = int(sum(int((c != ONE_HOT_NONE[c.dtype]).sum()) for c in cols))
                    for layout in ("cycle_major", "address_major"):
                        got = bases.one_hot_rows(cols, K, W, layout)             # warm-up
                        ref = batch_add_route(sess, bases, cols, K, W, layout)
                        norm = G1Bases.from_jacobian(sess, got.reshape(-1, 12))  # device normalisation to affine
                        equal = bool((norm.affine() == ref).all())
                        norm.free()
                        ts = []
                        sess.timing_enable(True, 0)
                        sess.timing_collect()
                        for _ in range(10):
                            t0 = time.perf_counter()
                            bases.one_hot_rows(cols, K, W, layout)
                            ts.append(time.perf_counter() - t0)
                        acc = [t["ms"] for t in sess.timing_collect() if t["kind"] == "msm_accumulate"]
                        sess.timing_enable(False)
                        tb = []
                        for _ in range(3):
                            t0 = time.perf_counter()
                            batch_add_route(sess, bases, cols, K, W, layout)
                            tb.append(time.perf_counter() - t0)
                        ms = statistics.median(ts) * 1e3
                        bound_ms = hot * PRODUCTS_PER_ADD / FQ_PRODUCTS_PER_S * 1e3
                        rec = dict(log_t=log_t, K=K, W=W, layout=layout, count=count,
                                   column="90% one address" if skewed else "uniform", hot_entries=hot, equal_points=equal,
                                   one_hot_ms=round(ms, 3), one_hot_spread_ms=round((max(ts) - min(ts)) * 1e3, 3),
                                   accumulate_ms=round(sum(acc) / 10, 3) if acc else None,
                                   batch_add_route_ms=round(statistics.median(tb) * 1e3, 1),
                                   speedup=round(statistics.median(tb) * 1e3 / ms, 1),
                                   accumulation_bound_ms=round(bound_ms, 3), fraction_of_bound=round(bound_ms / ms, 3),
                                   gpu=name, power_limit=power)
                        print(json.dumps(rec), flush=True)
                        out.append(rec)
    sess.close()
    if args.out:
        with open(args.out, "w") as f:
            for r in out:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
