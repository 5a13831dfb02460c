"""Random linear combinations on one GPU: jb_table_linear_combination against the host route a caller had before it -
the threaded C combination (tests/lincomb_cref.py, every host thread) plus jb_table_upload of the result - after
checking that both give the same table.

Workloads at 2^22 and 2^24 entries: 8 field tables; 8 mixed terms (u8, u64 and i128 device columns plus 5 field
tables); a Jolt-shaped mix (4 one-hot K = 16 u8 address columns, 4 compact device columns, 2 field tables); 4 compact
columns (u8, u64, i64, i128) from device memory and the same from host memory.
Reports per workload the call's device time (CUDA events on the session's stream around the whole call, host columns'
copies included; median of 7 after 2 warm-ups), the host route's wall time (median of 3), and the call against its
bound: the larger of its bytes (each term read once in its own format, the output written once) over the data-sheet
3.35 TB/s HBM and its integer work over the Montgomery-product rate measured in the same run (jb_diag_mul_throughput;
a 256 x 256 unreduced product counts 64/136 of a Montgomery product, a 256 x 32w one 8w/136, the reduction 3). Reads
the card's name and power limit in the same run.
Output: one JSON line per workload on stdout, and in FILE with --out.

usage: python tools/lincomb_bench.py [--out FILE] [--quick]"""
import argparse
import ctypes
import json
import os
import pathlib
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import jolt_b200  # noqa: E402
from jolt_b200 import SCALAR_KINDS, LinearTerm, Polynomial  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from oracle.coracle import rand_limbs  # noqa: E402
import lincomb_cref as CR  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
WORDS = {"u8": 1, "u16": 1, "u32": 1, "u64": 2, "i64": 2, "u128": 4, "i128": 4}
BYTES = {"u8": 1, "u16": 2, "u32": 4, "u64": 8, "i64": 8, "u128": 16, "i128": 16}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return f"unknown ({e})", "unknown"


def device_ms(fn, reps=7, warm=2):
    """Median device time of fn() (CUDA events on the current torch stream, which the session enqueues on)."""
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


class Workload:
    """Terms in the device's and the C oracle's forms, with the bytes and integer work of one device call."""

    def __init__(self, s, n, seed):
        self.s, self.n, self.rng, self.seed = s, n, np.random.default_rng(seed), seed
        self.dev, self.cref, self.keep = [], [], []
        self.bytes, self.mont = 32 << n, 3 << n   # the output written once, one reduction per output

    def coeff(self):
        return O.random_fr(self.seed * 131 + len(self.dev), 1)[0]

    def table(self):
        c = self.coeff()
        limbs = rand_limbs(self.seed * 17 + len(self.dev), 1 << self.n)
        p = Polynomial.new(self.s, limbs)
        self.keep.append(p)
        self.dev.append(LinearTerm.table(p, c))
        self.cref.append(("table", limbs, c))
        self.bytes += 32 << self.n
        self.mont += (64 / 136) * (1 << self.n)

    def compact(self, kind, device=True):
        c = self.coeff()
        m = 1 << self.n
        if kind in ("u128", "i128"):
            a = self.rng.integers(0, 1 << 64, size=(m, 2), dtype=np.uint64)
        else:
            dt = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i64": np.int64}[kind]
            info = np.iinfo(dt)
            a = self.rng.integers(info.min, info.max, m, dtype=dt, endpoint=True)
        if device:
            t = torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()
            self.keep.append(t)
            self.dev.append(LinearTerm.compact(t, c, kind=kind))
        else:   # host records in small_scalars' layout, passed as they are (no Python round trip for i128)
            self.dev.append(LinearTerm(jolt_b200._lib.JB_LC_COMPACT, m, c, ptr=a.ctypes.data, kind=SCALAR_KINDS[kind],
                                       T=m, keep=a))
        self.cref.append(("compact", a, SCALAR_KINDS[kind], m, c))
        self.bytes += BYTES[kind] * m
        self.mont += (8 * WORDS[kind] / 136) * m

    def one_hot(self, K):
        c = self.coeff()
        T = (1 << self.n) // K
        col = self.rng.integers(0, K, T).astype(np.uint8)
        col[self.rng.random(T) < 0.1] = 0xFF
        t = torch.from_numpy(col).cuda()
        self.keep.append(t)
        self.dev.append(LinearTerm.one_hot(t, K, c))
        self.cref.append(("one_hot", col, K, 0, c))
        self.bytes += T

    def call(self):
        return Polynomial.linear_combination(self.s, self.dev, 1 << self.n)


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
    threads = os.cpu_count()
    lines = []

    def run(label, w):
        P = w.call()
        ref = CR.linear_combination(w.cref, 1 << w.n)
        assert np.array_equal(P.evals(), ref), label
        P.free()
        ms = device_ms(lambda: w.call().free())

        def host_route():
            out = CR.linear_combination(w.cref, 1 << w.n)
            q = Polynomial.new(s, out)
            q.free()
        host_route()
        ht = []
        for _ in range(3):
            t0 = time.perf_counter()
            host_route()
            ht.append((time.perf_counter() - t0) * 1e3)
        host_ms = statistics.median(ht)
        hbm, alu = w.bytes / HBM_BYTES_PER_S, w.mont / mont_per_s
        bound = max(hbm, alu) * 1e3
        rec = dict(workload=label, log_n=w.n, terms=len(w.dev), card=name, power_limit=power, ms=round(ms, 4),
                   bytes=int(w.bytes), mont_products=int(w.mont), bound_ms=round(bound, 4),
                   bound_by="hbm" if hbm >= alu else "integer", fraction_of_bound=round(bound / ms, 3),
                   mont_products_per_s=round(mont_per_s / 1e9, 1), host_route_ms=round(host_ms, 2),
                   host_threads=threads, speedup_vs_host=round(host_ms / ms, 1))
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)

    for n in ([12, 14] if a.quick else [22, 24]):
        w = Workload(s, n, 1)
        for _ in range(8):
            w.table()
        run("8_field_tables", w)
        del w
        w = Workload(s, n, 2)
        for kind in ("u8", "u64", "i128"):
            w.compact(kind)
        for _ in range(5):
            w.table()
        run("8_mixed", w)
        del w
        w = Workload(s, n, 3)
        for _ in range(4):
            w.one_hot(16)
        for kind in ("u8", "u64", "i64", "i128"):
            w.compact(kind)
        for _ in range(2):
            w.table()
        run("jolt_shaped", w)
        del w
        for device in (True, False):
            w = Workload(s, n, 4)
            for kind in ("u8", "u64", "i64", "i128"):
                w.compact(kind, device)
            run("compact_device" if device else "compact_host", w)
            del w
        torch.cuda.empty_cache()
    if a.out:
        pathlib.Path(a.out).write_text("\n".join(lines) + "\n")
    s.close()


if __name__ == "__main__":
    main()
