"""Multilinear evaluation at a point on one GPU: jb_table_evaluate_batch, jb_small_evaluate_batch, jb_one_hot_evaluate
and jb_one_hot_pushforward against the route callers had before them - clone (or upload and promote) the table, then
bind it n times - after checking that both give the same value.

Workloads: field tables at 2^20, 2^22, 2^24 in batches of 1 and 8; u8, u64 and i128 columns of 2^24 entries from host
memory and from device memory; one-hot evaluation and pushforward at T = 2^24 with K = 16, 256 (u8) and 2^16 (u16).
Reports per workload the call's device time (CUDA events on the session's stream around the whole call: eq tables,
kernel, lanes; median of 10 after a warm-up), the clone + bind route's device time, and the call against its bound:
the larger of its table bytes over the data-sheet 3.35 TB/s HBM and its integer work over the Montgomery-product rate
measured in the same run (jb_diag_mul_throughput; an unreduced 256 x 256 product is counted as half a Montgomery
product, a 256 x 32w one as w/16). Reads the card's name and power limit in the same run.
Output: one JSON line per workload on stdout, and in FILE with --out.

usage: python tools/eval_bench.py [--out FILE] [--quick]"""
import argparse
import ctypes
import json
import pathlib
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import jolt_b200  # noqa: E402
from jolt_b200 import Polynomial, evaluate_small, one_hot_evaluate, one_hot_pushforward  # noqa: E402
from oracle import bn254 as O  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return f"unknown ({e})", "unknown"


def device_ms(fn, reps=10, warm=2):
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


def random_table(n, seed):
    """A device tensor of 2^n canonical Montgomery elements (top limb < 2^61) and its polynomial handle."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randint(-(1 << 63), (1 << 63) - 1, (1 << n, 4), dtype=torch.int64, device="cuda", generator=g)
    t[:, 3] &= (1 << 61) - 1
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small sizes only (a rehearsal of the script)")
    a = ap.parse_args()
    name, power = card()
    s = jolt_b200.Session(0, cuda_stream=torch.cuda.current_stream().cuda_stream)
    gops = ctypes.c_double()
    s.check(s.lib.jb_diag_mul_throughput(s.h, 0, 0, 4096, s_blocks(), ctypes.byref(gops)))
    mont_per_s = gops.value * 1e9
    lines = []

    def emit(rec, bytes_, mont_products, ms):
        bound = max(bytes_ / HBM_BYTES_PER_S, mont_products / mont_per_s) * 1e3
        rec.update(card=name, power_limit=power, ms=round(ms, 4), bound_ms=round(bound, 4),
                   bound_by="hbm" if bytes_ / HBM_BYTES_PER_S >= mont_products / mont_per_s else "integer",
                   fraction_of_bound=round(bound / ms, 3), mont_products_per_s=round(mont_per_s / 1e9, 1))
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)

    sizes = [12, 14] if a.quick else [20, 22, 24]
    big = sizes[-1]
    pt_all = O.random_fr(1, 48)
    # ---- field tables
    for n in sizes:
        for batch in (1, 8):
            keep = [random_table(n, 10 * n + b) for b in range(batch)]
            polys = [Polynomial.wrap_device(s, t.data_ptr(), 1 << n) for t in keep]
            pt = pt_all[:n]
            got = Polynomial.batch_evaluate(polys, pt)

            def clone_bind():
                out = []
                for p in polys:
                    q = p.clone()
                    for r in pt:
                        q.bind(r)
                    out.append(q.to_ints()[0])
                    q.free()
                return out
            assert clone_bind() == got
            ms = device_ms(lambda: Polynomial.batch_evaluate(polys, pt))
            ms_b = device_ms(clone_bind, reps=3, warm=1)
            N = batch << n
            emit(dict(workload="field", log_n=n, batch=batch, clone_bind_ms=round(ms_b, 4), speedup=round(ms_b / ms, 2)),
                 32 * N, N / 2, ms)
            for p in polys:
                p.free()
            del keep
            torch.cuda.empty_cache()
    # ---- compact columns
    rng = np.random.Generator(np.random.PCG64(5))
    pt = pt_all[:big]
    for kind, words in (("u8", 1), ("u64", 2), ("i128", 4)):
        if kind == "u8":
            col = rng.integers(0, 256, size=1 << big, dtype=np.uint8)
        elif kind == "u64":
            col = rng.integers(0, 1 << 64, size=1 << big, dtype=np.uint64)
        else:
            col = rng.integers(-(1 << 63), 1 << 63, size=(1 << big, 2), dtype=np.int64)
            col[:, 1] >>= 1                                                 # i128 values in (-2^126, 2^126)
        host_arr = np.ascontiguousarray(col)          # i128: (lo, hi) words, two's complement
        dev = torch.from_numpy(host_arr.view(np.uint8).reshape(-1)).cuda()
        got = evaluate_small(s, dev, pt, kinds=kind)

        def promote_bind():
            """The previous route: fused upload + promote + first bind (jb_table_bind_small), then n - 1 binds."""
            h = ctypes.c_uint64()
            s.check(s.lib.jb_table_bind_small(s.h, host_arr.ctypes.data_as(ctypes.c_void_p), 1 << big,
                                              jolt_b200.SCALAR_KINDS[kind],
                                              jolt_b200.api._p(jolt_b200.field.to_limbs(pt[0])), 0, ctypes.byref(h)))
            q = Polynomial(s, h.value)
            for r in pt[1:]:
                q.bind(r)
            v = q.to_ints()[0]
            q.free()
            return v
        assert [promote_bind()] == got
        host_ptr = (ctypes.c_void_p * 1)(host_arr.ctypes.data)
        kinds = (ctypes.c_int * 1)(jolt_b200.SCALAR_KINDS[kind])
        ptl = jolt_b200.point_limbs(pt)
        out = np.empty((1, 4), dtype=np.uint64)

        def host_call():
            s.check(s.lib.jb_small_evaluate_batch(s.h, host_ptr, 1, kinds, 1 << big, 0, jolt_b200.api._p(ptl), big,
                                                  jolt_b200.api._p(out)))
        host_call()
        assert jolt_b200.field.limbs_to_ints(out) == got
        ms_b = device_ms(promote_bind, reps=3, warm=1)
        nb = (1 << big) * jolt_b200.api._KIND_BYTES[kind]
        for where, fn in (("device", lambda: evaluate_small(s, dev, pt, kinds=kind)), ("host", host_call)):
            ms = device_ms(fn)
            emit(dict(workload="compact", kind=kind, columns=where, log_n=big, promote_bind_ms=round(ms_b, 4),
                      speedup=round(ms_b / ms, 2)), nb, (1 << big) * words / 16, ms)
    # ---- one-hot
    T = 1 << big
    for K, dt in ((16, np.uint8), (256, np.uint8), (1 << 16, np.uint16)):
        none = 0xFF if dt == np.uint8 else 0xFFFF
        col = rng.integers(0, min(K, none), size=T).astype(dt)
        dcol = torch.from_numpy(col.view(np.int16) if dt == np.uint16 else col).cuda()
        lk = K.bit_length() - 1
        ptk = pt_all[:big + lk]
        got = one_hot_evaluate(s, dcol, K, ptk)[0]
        G = one_hot_pushforward(s, dcol, K, ptk[:big])[0]
        eq_a = O.eq_evals(ptk[big:])
        assert got == sum(x * y for x, y in zip(eq_a, G.to_ints())) % O.R_MOD
        G.free()
        ms = device_ms(lambda: one_hot_evaluate(s, dcol, K, ptk))
        emit(dict(workload="one_hot_evaluate", K=K, log_t=big), T * col.itemsize, T / 2, ms)

        def pf():
            for g in one_hot_pushforward(s, dcol, K, ptk[:big]):
                g.free()
        ms = device_ms(pf)
        emit(dict(workload="one_hot_pushforward", K=K, log_t=big), T * col.itemsize, T, ms)
    if a.out:
        pathlib.Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(a.out).write_text("\n".join(lines) + "\n")
    s.close()


def s_blocks():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8


if __name__ == "__main__":
    main()
