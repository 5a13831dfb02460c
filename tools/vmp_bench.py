"""Dory's vector-matrix product on one GPU: jb_lc_vector_matrix_product against the materialise-and-bind route a caller
had before it (jb_table_linear_combination, jb_table_clone, then log R HighToLow binds by the row coordinates), after
checking that both give the same table, wherever P fits in device memory.

Workloads: 8 field tables at 2^24; the tools/lincomb_bench.py mixes (8 mixed terms, the Jolt-shaped mix with K = 16,
4 compact device columns) at 2^22 and 2^24; the Jolt shape at T = 2^24 (one-hot K = 256 u8 columns in both layouts,
2^32 coefficients each, a compact u64 and an i128 column and a field table as prefixes; W = R = 2^16; no route); and
one-hot terms alone, K = 16 / 256 (T = 2^20, u8) and K = 2^16 (T = 2^20, u16), uniform and skewed (90 % of the cycles
at one address), in both layouts. L is eq(r_row) and W = 2^ceil(n / 2).
Reports per workload the call's device time (CUDA events on the session's stream around the whole call, host columns'
copies included; median of 7 after 2 warm-ups), the route's device time the same way, and the call against its
bound: the larger of its bytes (each term read once in its own format, L read once, the bins and the output written
once) over the data-sheet 3.35 TB/s HBM and its integer work over the Montgomery-product rate measured in the same run
(jb_diag_mul_throughput; a 256 x 256 unreduced product counts 64/136 of a Montgomery product, a 256 x 32w one 8w/136,
one-hot entries count none). Reads the card's name and power limit in the same run.
Output: one JSON line per workload on stdout, and in FILE with --out.

usage: python tools/vmp_bench.py [--out FILE] [--quick]"""
import argparse
import ctypes
import json
import pathlib
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import jolt_b200  # noqa: E402
from jolt_b200 import EqPolynomial, LinearTerm, Polynomial  # noqa: E402
from jolt_b200 import field as F  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from lincomb_bench import HBM_BYTES_PER_S, Workload, card, device_ms  # noqa: E402

FREE_BYTES_MARGIN = 4 << 30


def terms(s, n, seed):
    """lincomb_bench's term builder with nothing counted yet: this call writes W entries, not 2^n."""
    w = Workload(s, n, seed)
    w.bytes, w.mont = 0, 0
    return w


class OneHot(Workload):
    """One one-hot term alone: its address column read once (no integer work counted)."""

    def __init__(self, s, K, lt, layout, skewed, seed):
        super().__init__(s, (K << lt).bit_length() - 1, seed)
        self.bytes, self.mont = 0, 0
        dt = np.uint8 if K <= 256 else np.uint16
        none = np.iinfo(dt).max
        col = self.rng.integers(0, min(K, none), 1 << lt).astype(dt)
        if skewed:
            col[self.rng.random(1 << lt) < 0.9] = K // 2
        col[self.rng.random(1 << lt) < 0.05] = none
        t = torch.from_numpy(col if dt == np.uint8 else col.view(np.int16)).cuda()
        self.keep.append(t)
        self.dev.append(LinearTerm.one_hot(t, K, self.coeff(), layout))
        self.bytes += col.nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small sizes only (a rehearsal of the script)")
    a = ap.parse_args()
    name, power = card()
    s = jolt_b200.Session(0, cuda_stream=torch.cuda.current_stream().cuda_stream)
    gops = ctypes.c_double()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    s.check(s.lib.jb_diag_mul_throughput(s.h, 0, 0, 4096, sm * 8, ctypes.byref(gops)))
    mont_per_s = gops.value * 1e9
    lines = []

    def run(label, w, lw=None, route=True):
        n = w.n
        lw = (n + 1) // 2 if lw is None else lw
        W, R = 1 << lw, 1 << (n - lw)
        r_row = O.random_fr(w.seed + 7, n - lw)
        L = EqPolynomial.evals(s, F.ints_to_limbs(r_row))

        def call():
            return Polynomial.vector_matrix_product(s, w.dev, L, W, length=1 << n)

        def bind_route():
            P = Polynomial.linear_combination(s, w.dev, 1 << n)
            Q = P.clone()
            P.free()
            for r in r_row:
                Q.bind(r)
            return Q

        v = call()
        got = v.evals()
        v.free()
        fits = route and (64 << n) + FREE_BYTES_MARGIN < torch.cuda.mem_get_info()[0]
        if fits:
            Q = bind_route()
            assert np.array_equal(got, Q.evals()), label
            Q.free()
        else:   # no independent route at this size: check determinism at least
            v = call()
            assert np.array_equal(got, v.evals()), label
            v.free()
        ms = device_ms(lambda: call().free())
        route_ms = device_ms(lambda: bind_route().free()) if fits else None
        nbytes, mont = w.bytes + 32 * R + 96 * W, w.mont   # + L, the bins (written, read) and the output
        hbm, alu = nbytes / HBM_BYTES_PER_S, mont / mont_per_s
        bound = max(hbm, alu) * 1e3
        rec = dict(workload=label, log_n=n, log_w=lw, terms=len(w.dev), card=name, power_limit=power, ms=round(ms, 4),
                   bytes=int(nbytes), mont_products=int(mont), bound_ms=round(bound, 4),
                   bound_by="hbm" if hbm >= alu else "integer", fraction_of_bound=round(bound / ms, 3),
                   mont_products_per_s=round(mont_per_s / 1e9, 1),
                   route_ms=None if route_ms is None else round(route_ms, 3),
                   speedup_vs_route=None if route_ms is None else round(route_ms / ms, 1))
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
        L.free()

    sizes = [12, 14] if a.quick else [22, 24]
    w = terms(s, sizes[-1], 1)
    for _ in range(8):
        w.table()
    run("8_field_tables", w)
    del w
    for n in sizes:
        w = terms(s, n, 2)
        for kind in ("u8", "u64", "i128"):
            w.compact(kind)
        for _ in range(5):
            w.table()
        run("8_mixed", w)
        del w
        w = terms(s, n, 3)
        for _ in range(4):
            w.one_hot(16)
        for kind in ("u8", "u64", "i64", "i128"):
            w.compact(kind)
        for _ in range(2):
            w.table()
        run("jolt_shaped_k16", w)
        del w
        w = terms(s, n, 4)
        for kind in ("u8", "u64", "i64", "i128"):
            w.compact(kind)
        run("compact_device", w)
        del w
        torch.cuda.empty_cache()
    # the Jolt shape beyond what can be materialised
    lt = 12 if a.quick else 24
    w = terms(s, lt, 5)
    w.compact("u64")
    w.compact("i128")
    w.table()
    for layout in ("cycle_major", "address_major"):
        oh = OneHot(s, 256, lt, layout, False, 6 + len(w.dev))
        w.dev += oh.dev
        w.keep += oh.keep
        w.bytes += oh.bytes
    w.n = lt + 8
    run("jolt_shape_k256", w, lw=w.n // 2, route=False)
    del w
    torch.cuda.empty_cache()
    lt = 10 if a.quick else 20
    for K in (16, 256, 1 << 16):
        for layout in ("cycle_major", "address_major"):
            for skewed in (False, True):
                w = OneHot(s, K, lt, layout, skewed, 7)
                run(f"one_hot_k{K}_{layout}_{'skewed' if skewed else 'uniform'}", w)
                del w
                torch.cuda.empty_cache()
    if a.out:
        pathlib.Path(a.out).write_text("\n".join(lines) + "\n")
    s.close()


if __name__ == "__main__":
    main()
