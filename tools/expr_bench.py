"""Complete sumchecks of expression members (jb_member_create_expr) at 2^N, both binding orders, beside the workaround
today's members need for the same relation: one member per monomial in one batch, every repeated table cloned, the
coefficient as the member's batch coefficient (the degree-6 product has no workaround: built products stop at 4).

Shapes: Booleanity eq * (f^2 - f); eq * (a b - c); read / write checking eq * (ra val + g wa val + g^2 wa inc) (tables
shared between terms); a degree-6 product f0 ... f5.

Per workload: the median wall time of the whole batched sumcheck (prove_batch_native: C++ engine, SplitMix stand-in
transcript with 125-bit challenges, ends in a device round trip), and the device-timed round-0 (eval-only) and round-1
(bind + eval) passes against their HBM bound (bytes over the H100 SXM data-sheet 3.35 TB/s) and integer-pipe bound
(Montgomery products over the rate jb_diag_mul_throughput measures on this card). Reads the card's name and power limit
in the same run. JSON lines on stdout (and to --out).

usage: python tools/expr_bench.py [--log-n 22] [--steps 3] [--orders l2h,h2l] [--shapes ...] [--out FILE]"""
import argparse
import ctypes
import json
import pathlib
import statistics
import subprocess
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

import jolt_b200  # noqa: E402
from jolt_b200 import (BatchMember, EqPolynomial, EqProductMember, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH,  # noqa: E402
                       Polynomial, ProductMember)
from jolt_b200 import field as F  # noqa: E402
from oracle.coracle import rand_challenge, rand_limbs  # noqa: E402

P = F.R_MOD
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s
SHAPES = {
    "booleanity": (1, [(1, [0, 0]), (-1, [0])], True),
    "ab_minus_c": (3, [(1, [0, 1]), (-1, [2])], True),
    "rw_checking": (4, [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA % P, [1, 3])], True),
    "degree6": (6, [(1, [0, 1, 2, 3, 4, 5])], False),
}


def card():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # the timings still stand with the card's name
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def mul_rate(sess):
    """sustained full Montgomery products per second on this card (jb_diag_mul_throughput, Fr)"""
    import torch
    g = ctypes.c_double()
    sess.check(sess.lib.jb_diag_mul_throughput(sess.h, 0, 0, 2000, torch.cuda.get_device_properties(0).multi_processor_count * 8,
                                               ctypes.byref(g)))
    return g.value * 1e9


def pass_work(T, mons, eq, bind):
    """(HBM bytes, full-product equivalents) per pair of one expression pass (s(1) from the claim)"""
    D = max(len(t) for _, t in mons)
    points = [0] + list(range(2, D)) + (["inf"] if D >= 2 else [])
    muls = 0.0
    for t in points:
        for c, tabs in mons:
            if t == "inf" and len(tabs) < D:
                continue
            muls += len(tabs) - 1 + (0 if c % P in (1, P - 1) else 1)
        muls += 1 if eq else 0
    muls += 1 if eq else 0            # the split-eq weight of the pair
    if bind:
        muls += 2 * T * 0.5           # two binds per table with a 125-bit challenge (~half a full product each)
    return (T * (4 * 32 + 2 * 32) if bind else T * 2 * 32), muls


def workaround_work(T, mons, eq, bind):
    b, m = 0, 0.0
    for c, tabs in mons:
        bb, mm = pass_work(len(tabs), [(1, list(range(len(tabs))))], eq, bind)
        b += bb
        m += mm
    return b, m


def claim_of(sess, tabs, tabs_idx, w, order):
    """s(0) + s(1) of prod_i f_{tabs_idx[i]} (times eq(w, x)) from the plain product member's first round"""
    polys = [tabs[i].clone() for i in tabs_idx]
    if w is not None:
        polys = [EqPolynomial.evals(sess, w)] + polys
    m = ProductMember(sess, polys, order)
    ev = m.prove_round_evals(None, 0, None)
    m.close()
    return (ev[0] + ev[1]) % P


def build(sess, kind, tabs, mons, w, order):
    """the members of one complete sumcheck, over fresh device clones of `tabs`"""
    if kind == "expr":
        mem = ExpressionMember(sess, [t.clone() for t in tabs], mons, w, order=order)
        return [mem]
    out = []
    for c, idx in mons:
        polys = [tabs[i].clone() for i in idx]
        out.append(EqProductMember(sess, polys, w, order=order) if w is not None else ProductMember(sess, polys, order))
    return out


def run(sess, tabs, shape, order, steps, rate, info, emit):
    T, mons, eq = SHAPES[shape]
    n = len(tabs[0]).bit_length() - 1
    w = np.stack([rand_challenge(0x5100 + i) for i in range(n)]) if eq else None
    mclaims = [claim_of(sess, tabs, idx, w, order) if len(idx) + (1 if eq else 0) <= 4 else None for _, idx in mons]
    if any(c is None for c in mclaims):   # (degree 6: the expression member's own first round without a claim)
        m = ExpressionMember(sess, [t.clone() for t in tabs], mons, w, order=order)
        ev = m.prove_round_evals(None, 0, None)
        m.close()
        total = (ev[0] + ev[1]) % P
    else:
        total = sum(c % P * k for (c, _), k in zip(mons, mclaims)) % P
    deg = max(len(t) for _, t in mons) + (1 if eq else 0)
    kinds = ["expr"] + (["workaround"] if all(len(t) <= (3 if eq else 4) for _, t in mons) else [])
    for kind in kinds:
        if kind == "expr":
            descs = [BatchMember(total, 1, n, 0)]
        else:
            descs = [BatchMember(k, c % P, n, 0) for (c, _), k in zip(mons, mclaims)]
        times = []
        proofs = []
        for rep in range(steps + 1):
            members = build(sess, kind, tabs, mons, w, order)
            sess.synchronize()
            timed = rep == steps   # the last run is device-timed per pass (kept out of the wall-time median)
            if timed:
                sess.timing_enable(True, 1 << (n - 3))
            t0 = time.perf_counter()
            res = jolt_b200.prove_batch_native(descs, members, n, deg, total, seed=7)
            sess.synchronize()
            dt = time.perf_counter() - t0
            if timed:
                passes = sess.timing_collect()
                sess.timing_enable(False)
            elif rep > 0:
                times.append(dt * 1e3)
            proofs.append((res.challenges, res.final_claim))
            for m in members:
                m.close()
        assert all(p == proofs[0] for p in proofs), "runs of one workload disagree"
        pairs0, pairs1 = 1 << (n - 1), 1 << (n - 2)
        r0 = sum(p["ms"] for p in passes if p["items"] == pairs0)
        r1 = sum(p["ms"] for p in passes if p["items"] == pairs1)
        wf = pass_work if kind == "expr" else workaround_work
        rec = dict(shape=shape, order="l2h" if order == LOW_TO_HIGH else "h2l", log_n=n, path=kind, degree=deg,
                   sumcheck_ms=round(statistics.median(times), 3), passes_round0=len([p for p in passes if p["items"] == pairs0]))
        for name, ms, bind, pairs in (("round0_eval", r0, False, pairs0), ("round1_bind", r1, True, pairs1)):
            b, m = wf(T, mons, eq, bind)
            t_hbm, t_int = b * pairs / HBM_PEAK * 1e3, m * pairs / rate * 1e3
            rec[name] = dict(ms=round(ms, 4), hbm_bound_ms=round(t_hbm, 4), int_bound_ms=round(t_int, 4),
                             bound="hbm" if t_hbm >= t_int else "int", share_of_bound=round(max(t_hbm, t_int) / ms, 3) if ms else None)
        rec.update(info)
        emit(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--orders", default="l2h,h2l")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    out = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()
    sess = jolt_b200.Session(0)
    rate = mul_rate(sess)
    emit(dict(kind="alu", full_products_per_s=rate, **info))
    n = a.log_n
    base = [Polynomial.new(sess, rand_limbs(0xB000 + j, 1 << n)) for j in range(6)]
    for o in a.orders.split(","):
        order = LOW_TO_HIGH if o == "l2h" else HIGH_TO_LOW
        for shape in a.shapes.split(","):
            run(sess, base[:SHAPES[shape][0]], shape, order, a.steps, rate, info, emit)
    sess.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
