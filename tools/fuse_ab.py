#!/usr/bin/env python
"""A/B of the folded large rounds of the resident kernel's staged runs: in ONE process, Sessions created with
JB_RES_FUSE=0 (one pass per round) and =1 (the round after a large pass is answered from its lookahead sums, the
next pass binds two variables) take turns on bench.py's workload (a degree-2 product sumcheck over 2 tables of
2^log_n Fr, a fresh copy of the inputs per step). Reports ms/step (CUDA events) per alternation with its median and
spread per variant, the device time of every command of a step (jb_ctx_run_log %globaltimer stamps) with the HBM
bytes its pass moves and the rate that gives, checks that both variants return identical proofs and final
evaluations, and prints the GPU, its power limit and SM clock.
usage: python tools/fuse_ab.py [--log-n 22] [--steps 20] [--alternations 3] [--orders l2h,h2l] [--json OUT]"""
import argparse
import ctypes
import json
import os
import pathlib
import statistics
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from staged_ab import gpu_info  # noqa: E402

RES_THIN_PAIRS = 1 << 17


def schedule(log_n: int, fuse: bool) -> list[tuple[str, int, int]]:
    """(pass, table entries it reads, HBM bytes for 2 tables) of every command before the thin rounds"""
    n = 1 << log_n
    fusable = lambda n: n // 4 > RES_THIN_PAIRS  # noqa: E731  (res_fusable, resident.cuh)
    out = [("eval+look" if fuse and fusable(n) else "eval", n, 2 * 32 * n)]
    while n // 4 > RES_THIN_PAIRS:  # bind passes that are not thin
        if fuse and fusable(n):  # this round is answered from lookahead; the next command binds twice
            out.append(("bind2+look", n, 2 * 32 * (n + n // 4)))
            n //= 4
        else:
            out.append(("bind+eval", n, 2 * 32 * (n + n // 2)))
            n //= 2
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per variant per alternation")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--alternations", type=int, default=3)
    ap.add_argument("--orders", default="l2h,h2l")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    orders = [o for o in args.orders.split(",") if o]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fuse_ab.py: no CUDA device - the A/B is a measurement on the GPU")
    import jolt_b200
    from jolt_b200 import BatchMember, Polynomial, ProductMember
    from jolt_b200 import field as F
    from jolt_b200.api import _p

    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sessions = {}
    for v in (0, 1):
        os.environ["JB_RES_FUSE"] = str(v)
        sessions[v] = jolt_b200.Session(0, cuda_stream=stream.cuda_stream)
    del os.environ["JB_RES_FUSE"]
    n, m = 1 << args.log_n, 2
    sched = {v: schedule(args.log_n, bool(v)) for v in (0, 1)}

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
        # per command: device pass (decode -> sums collected), then the idle gap until the next command's decode
        passes = [(log[k, 1] - log[k, 0]) / 1e3 for k in range(len(log))]
        idle = [(log[k + 1, 0] - log[k, 1]) / 1e3 for k in range(len(log) - 1)] + [0.0]
        return passes, idle

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
        logs = {0: [], 1: []}
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
                    logs[v].append(run_log(sess))
                e1.record(stream)
                e1.synchronize()
                ms[v].append(e0.elapsed_time(e1) / args.steps)
                del copies
        (r0, f0), (r1, f1) = outputs[0], outputs[1]
        same = all((a == b).all() for a, b in zip(r0, r1)) and (f0 == f1).all()
        row = {"outputs_identical": bool(same)}
        for v, name in ((0, "unfused"), (1, "fused")):
            ncmd = min(len(p) for p, _ in logs[v])
            pass_us = [statistics.median(p[k] for p, _ in logs[v]) for k in range(ncmd)]
            idle_us = [statistics.median(i[k] for _, i in logs[v]) for k in range(ncmd)]
            big = [{"pass": kind, "entries_read": ent, "hbm_bytes": by, "us": pass_us[k], "gb_per_s": by / (pass_us[k] * 1e-6) / 1e9}
                   for k, (kind, ent, by) in enumerate(sched[v]) if k < ncmd]
            row[name] = {"ms_per_step": ms[v], "median_ms": statistics.median(ms[v]), "spread_ms": max(ms[v]) - min(ms[v]),
                         "commands": ncmd, "command_pass_us_median": pass_us, "command_idle_us_median": idle_us,
                         "large_passes": big}
        row["speedup"] = row["unfused"]["median_ms"] / row["fused"]["median_ms"]
        result["orders"][oname] = row
        print(f"[{oname}] outputs identical: {same}")
        for name in ("unfused", "fused"):
            r = row[name]
            print(f"  {name:8s} ms/step median {r['median_ms']:.4f} spread {r['spread_ms']:.4f}  ({', '.join(f'{x:.4f}' for x in r['ms_per_step'])})"
                  f"  commands {r['commands']}")
            for b in r["large_passes"]:
                print(f"    {b['pass']:10s} reads 2 x {b['entries_read']:>8d}  {b['hbm_bytes'] / 1e6:7.1f} MB  {b['us']:7.1f} us  {b['gb_per_s']:7.1f} GB/s")
            print("    pass us: " + ", ".join(f"{x:.1f}" for x in r["command_pass_us_median"]))
            print("    idle us: " + ", ".join(f"{x:.1f}" for x in r["command_idle_us_median"]))
        print(f"  speedup {row['speedup']:.3f}x")
        if not same:
            raise SystemExit(f"fuse_ab.py: the fused and unfused proofs differ ({oname})")
    print(f"GPU: {result['gpu']}")
    print(json.dumps(result))
    if args.json:
        pathlib.Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.json).write_text(json.dumps(result, indent=1))
    for s in sessions.values():
        s.close()


if __name__ == "__main__":
    main()
