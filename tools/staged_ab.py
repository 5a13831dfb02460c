#!/usr/bin/env python
"""A/B of the resident kernel's staged large passes: in ONE process, Sessions created with JB_RES_STAGED=0 and =1
take turns on bench.py's workload (a degree-2 product sumcheck over 2 tables of 2^log_n Fr, a fresh copy of the
inputs per step). Reports ms/step (CUDA events) per alternation and its median / spread per variant, the device pass
time of rounds 0-3 from jb_ctx_run_log (%globaltimer stamps, as tools/round_probe.py reads them), checks that both
variants return identical proofs and final evaluations, and prints the GPU, its power limit and SM clock.
usage: python tools/staged_ab.py [--log-n 22] [--steps 20] [--alternations 3] [--orders l2h,h2l] [--json OUT]"""
import argparse
import ctypes
import json
import os
import pathlib
import statistics
import subprocess
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

ROUNDS = 4  # rounds 0..3: the passes over more than RES_THIN_PAIRS pairs at 2^22


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per variant per alternation")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--alternations", type=int, default=3)
    ap.add_argument("--orders", default="l2h,h2l")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    return ap.parse_args()


def gpu_info(torch):
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # report, the timings still stand with the name
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def main():
    args = parse()
    orders = [o for o in args.orders.split(",") if o]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("staged_ab.py: no CUDA device - the A/B is a measurement on the GPU")
    import jolt_b200
    from jolt_b200 import BatchMember, Polynomial, ProductMember
    from jolt_b200 import field as F
    from jolt_b200.api import _p

    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sessions = {}
    for v in (0, 1):
        os.environ["JB_RES_STAGED"] = str(v)
        sessions[v] = jolt_b200.Session(0, cuda_stream=stream.cuda_stream)
    del os.environ["JB_RES_STAGED"]
    n, m = 1 << args.log_n, 2

    def synth(seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        t = torch.randint(0, 2 ** 62, (n, 4), dtype=torch.int64, device="cuda", generator=g)
        t[:, 3] &= (1 << 60) - 1
        return t

    def run_log(sess):
        log = np.zeros((64, 8), dtype=np.uint64)
        cnt = ctypes.c_size_t()
        sess.check(sess.lib.jb_ctx_run_log(sess.h, _p(log), 64, ctypes.byref(cnt)))
        log = log[: cnt.value].astype(np.int64)
        return [(log[k, 1] - log[k, 0]) / 1e3 for k in range(min(ROUNDS, len(log)))]

    base = [synth(0xB200 + j) for j in range(m)]
    result = {"gpu": gpu_info(torch), "workload": f"degree-2 product sumcheck, 2 x 2^{args.log_n} Fr, 125-bit challenges",
              "steps_per_alternation": args.steps, "alternations": args.alternations, "orders": {}}
    for oname in orders:
        order = jolt_b200.LOW_TO_HIGH if oname == "l2h" else jolt_b200.HIGH_TO_LOW
        probe_bufs = [b.clone() for b in base]
        probe = ProductMember(sessions[0], [Polynomial.wrap_device(sessions[0], b.data_ptr(), n) for b in probe_bufs], order)
        ev = probe.prove_round_evals(None, 0)
        claim = (ev[0] + ev[1]) % F.R_MOD
        probe.close()
        del probe_bufs
        desc = [BatchMember(claim, 1, args.log_n, 0)]

        def step(sess, bufs):
            mem = ProductMember(sess, [Polynomial.wrap_device(sess, b.data_ptr(), n) for b in bufs], order)
            res = jolt_b200.prove_batch_native(desc, [mem], args.log_n, m, claim, seed=7, raw=True)
            fe = mem.final_evals(raw=True)
            mem.close()
            return res, fe

        ms = {0: [], 1: []}
        passes = {0: [], 1: []}
        outputs = {}
        for alt in range(args.alternations):
            for v in ((0, 1) if alt % 2 == 0 else (1, 0)):
                sess = sessions[v]
                for _ in range(args.warmup):
                    step(sess, [b.clone() for b in base])
                copies = [[b.clone() for b in base] for _ in range(args.steps)]
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for k in range(args.steps):
                    outputs[v] = step(sess, copies[k])
                    passes[v].append(run_log(sess))
                e1.record(stream)
                e1.synchronize()
                ms[v].append(e0.elapsed_time(e1) / args.steps)
                del copies
        (r0, f0), (r1, f1) = outputs[0], outputs[1]
        same = all((a == b).all() for a, b in zip(r0, r1)) and (f0 == f1).all()
        row = {"outputs_identical": bool(same)}
        for v, name in ((0, "unstaged"), (1, "staged")):
            med = statistics.median(ms[v])
            rounds = [statistics.median(p[k] for p in passes[v]) for k in range(ROUNDS)]
            row[name] = {"ms_per_step": ms[v], "median_ms": med, "spread_ms": max(ms[v]) - min(ms[v]), "round_pass_us_median": rounds}
        row["speedup"] = row["unstaged"]["median_ms"] / row["staged"]["median_ms"]
        result["orders"][oname] = row
        print(f"[{oname}] outputs identical: {same}")
        for name in ("unstaged", "staged"):
            r = row[name]
            print(f"  {name:9s} ms/step median {r['median_ms']:.4f} spread {r['spread_ms']:.4f}  ({', '.join(f'{x:.4f}' for x in r['ms_per_step'])})"
                  f"  rounds 0-3 pass us: {', '.join(f'{x:.1f}' for x in r['round_pass_us_median'])}")
        print(f"  speedup {row['speedup']:.3f}x")
        if not same:
            raise SystemExit(f"staged_ab.py: the staged and unstaged proofs differ ({oname})")
    print(f"GPU: {result['gpu']}")
    print(json.dumps(result))
    if args.json:
        pathlib.Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.json).write_text(json.dumps(result, indent=1))
    for s in sessions.values():
        s.close()


if __name__ == "__main__":
    main()
