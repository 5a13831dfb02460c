"""Per-kernel timings on one H100 (CUDA events on the launching stream, warm-up, L2-exceeding
inputs or explicit flush). Writes gpurun_out/microbench.jsonl. Not the driver's bench (bench.py)."""
import ctypes
import json
import os
import sys
import pathlib

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import jolt_b200
from jolt_b200 import HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, ProductMember, EqPolynomial
from jolt_b200.api import _p

OUT = ROOT / "gpurun_out"
OUT.mkdir(exist_ok=True)
quick = "--quick" in sys.argv
PEAK = 3350.0  # GB/s, H100 SXM data-sheet HBM3 bandwidth
try:
    PEAK = json.load(open(ROOT / "MEASURED_PEAKS.json"))["hbm_gbs"]
except Exception:
    pass

torch.cuda.set_device(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
sess = jolt_b200.Session(0, cuda_stream=stream.cuda_stream)
lib = sess.lib
results = []


def emit(**kw):
    results.append(kw)
    print(json.dumps(kw), flush=True)


def rand_table(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randint(0, 2**62, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    t[:, 3] &= (1 << 60) - 1
    return t


flush_buf = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")


def timed(fn, reps=10, warm=3, flush=True):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        if flush:
            flush_buf.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


# --- ALU ceilings -------------------------------------------------------------------------
for fld in (0, 1):
    for var, name in ((0, "mul_full"), (1, "mul_hi4"), (2, "addsub")):
        g = ctypes.c_double()
        sess.check(lib.jb_diag_mul_throughput(sess.h, fld, var, 2000, torch.cuda.get_device_properties(0).multi_processor_count * 8, ctypes.byref(g)))
        emit(kind="alu", field="Fr" if fld == 0 else "Fq", op=name, gops=round(g.value, 1))

ch125 = np.array([0, 0, 0x123456789ABCDEF1, 0x0FEDCBA987654321], dtype=np.uint64)
full = np.array([0x1111111111111111, 0x2222222222222222, 0x3333333333333333, 0x0444444444444444], dtype=np.uint64)

# --- bind ------------------------------------------------------------------------------------
sizes = [20, 22, 24] if quick else [16, 18, 20, 22, 24, 26]
for lg in sizes:
    n = 1 << lg
    buf = rand_table(n, lg)
    for order, oname in ((HIGH_TO_LOW, "h2l"), (LOW_TO_HIGH, "l2h")):
        for r, rname in ((ch125, "c125"), (full, "f254")):
            def one():
                p = Polynomial.wrap_device(sess, buf.data_ptr(), n)
                p.bind_with_order(r, order)
                p.free()
            med, best = timed(one)
            bytes_ = 48 * n
            emit(kind="bind", log_n=lg, order=oname, challenge=rname, ms=round(med, 4), ms_best=round(best, 4),
                 gbs=round(bytes_ / med / 1e6, 1), frac=round(bytes_ / med / 1e6 / PEAK, 3),
                 gfieldops=round(3 * (n / 2) / med / 1e6, 1))
    del buf

# --- fused rounds ------------------------------------------------------------------------------
eval_ms = {}
for lg in ([22, 24] if quick else [20, 22, 24, 26]):
    n = 1 << lg
    for m in (1, 2, 3):
        if lg == 26 and m == 3:
            continue
        bufs = [rand_table(n, 100 + j) for j in range(m)]
        for order, oname in ((HIGH_TO_LOW, "h2l"), (LOW_TO_HIGH, "l2h")):
            for mode in ("eval_only", "bind_eval_c125", "bind_eval_f254"):
                def one():
                    polys = [Polynomial.wrap_device(sess, b.data_ptr(), n) for b in bufs]
                    mem = ProductMember(sess, polys, order)
                    if mode == "eval_only":
                        mem.prove_round_evals(None, 0)
                    else:
                        out = np.empty((m + 1, 4), dtype=np.uint64)
                        r = ch125 if mode.endswith("c125") else full
                        sess.check(lib.jb_member_prove_round(mem.h, None, 0, None, _p(out)))
                        sess.check(lib.jb_member_prove_round(mem.h, _p(r), 1, None, _p(out)))
                    mem.close()
                med, best = timed(one)
                if mode != "eval_only":   # subtract the eval-only round 0 that had to precede the fused pass
                    med, best = med - eval_ms[(m, oname)], best - eval_ms[(m, oname)]
                else:
                    eval_ms[(m, oname)] = med
                bytes_ = m * (64 * (n // 2) if mode == "eval_only" else 48 * n)
                emit(kind="fused", log_n=lg, m=m, order=oname, mode=mode, ms=round(med, 4), ms_best=round(best, 4),
                     gbs=round(bytes_ / med / 1e6, 1), frac=round(bytes_ / med / 1e6 / PEAK, 3))
        del bufs

# --- eq ---------------------------------------------------------------------------------------
for lg, kind in [(l, k) for l in ([22] if quick else [20, 22, 24, 26]) for k in ("c125", "f254")]:
    r = np.ascontiguousarray(rand_table(lg, 7).cpu().numpy().view(np.uint64))
    if kind == "c125":
        r[:, 0] = 0
        r[:, 1] = 0
    def one():
        EqPolynomial.evals(sess, r).free()
    sess.timing_enable(True, 1 << 12)
    med, best = timed(one, flush=False)
    ks = [t["ms"] for t in sess.timing_collect() if t["kind"] == "eq"]
    sess.timing_enable(False)
    kms = sorted(ks)[len(ks) // 2] if ks else float("nan")
    bytes_ = 32 << lg
    emit(kind="eq", log_n=lg, point=kind, call_ms=round(med, 4), kernel_ms=round(kms, 4), gbs_call=round(bytes_ / med / 1e6, 1),
         gbs_kernel=round(bytes_ / kms / 1e6, 1), frac_kernel=round(bytes_ / kms / 1e6 / PEAK, 3))

with open(OUT / "microbench.jsonl", "w") as f:
    for r in results:
        f.write(json.dumps(r) + "\n")
