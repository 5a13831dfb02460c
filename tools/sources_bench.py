"""Expression members over sources (jb_member_create_expr_sources) beside today's route to the same sumcheck: promote
the compact columns with jb_table_upload_small and gather the one-hot polynomials on the host, upload them, then
jb_member_create_expr. Both binding orders, at 2^N.

Workloads:
  read_checking   eq * (ra val + g wa val + g^2 wa inc): ra, wa one-hot (u8, K = 256), val a field table, inc i64
  ra_virt_K16     eq(r_cycle, j) * prod_{i<4} ra_i(r_addr_i, j): 4 one-hot chunks (u8, K = 16)
  ra_virt_K256    the same with K = 256
  booleanity      eq * (f^2 - f) over a u8 column of bits
  ab_minus_c      eq * (a b - c) over u64 columns

Per workload and route, the median wall time of the whole call - from the columns (host arrays, or device tensors for
the sources route) to the final claim: member creation, every round (fixed 125-bit challenges), the terminal bind and
the final evaluations. The routes alternate in one process, and their round polynomials and final evaluations are
checked equal before anything is timed. For the sources member, the device time of round 0 (eval-only) and round 1
(bind + eval) passes (jb_ctx_timing_*) against the larger of the HBM bound (bytes over the H100 SXM data-sheet
3.35 TB/s) and the integer bound (Montgomery products over the rate jb_diag_mul_throughput measures in the same run),
and the device bytes each member holds after creation (computed from the shapes). Reads the card's name and power
limit in the same run. JSON lines on stdout (and to --out).

usage: python tools/sources_bench.py [--log-n 22,24] [--steps 3] [--orders l2h,h2l] [--workloads ...] [--out FILE]"""
import argparse
import json
import pathlib
import statistics
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import numpy as np  # noqa: E402

import jolt_b200  # noqa: E402
from jolt_b200 import EqPolynomial, ExpressionMember, HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, Source  # noqa: E402
from jolt_b200 import field as F  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from oracle.coracle import rand_challenge, rand_limbs  # noqa: E402
from expr_bench import HBM_PEAK, card, mul_rate  # noqa: E402

P = F.R_MOD
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
WORKLOADS = ["read_checking", "ra_virt_K16", "ra_virt_K256", "booleanity", "ab_minus_c"]


def columns(name, n, seed=0xC0):
    """[(type, host array, K, r_addr)] and the monomials of a workload; type 'one_hot' | 'compact' | 'table'"""
    rng = np.random.default_rng(seed)
    T = 1 << n
    if name == "read_checking":
        ra, wa = (rng.integers(0, 255, T).astype(np.uint8) for _ in range(2))
        return ([("one_hot", ra, 256, O.random_fr(seed + 1, 8)), ("one_hot", wa, 256, O.random_fr(seed + 2, 8)),
                 ("table", rand_limbs(seed + 3, T), 0, None), ("compact", rng.integers(-(1 << 40), 1 << 40, T), 0, None)],
                [(1, [0, 2]), (GAMMA, [1, 2]), (GAMMA * GAMMA % P, [1, 3])])
    if name.startswith("ra_virt"):
        K = 16 if name.endswith("K16") else 256
        hi = K if K == 16 else 255
        return ([("one_hot", rng.integers(0, hi, T).astype(np.uint8), K, O.random_fr(seed + i, K.bit_length() - 1))
                 for i in range(4)], [(1, [0, 1, 2, 3])])
    if name == "booleanity":
        return [("compact", rng.integers(0, 2, T).astype(np.uint8), 0, None)], [(1, [0, 0]), (-1, [0])]
    return ([("compact", rng.integers(0, 1 << 63, T, dtype=np.uint64) * 2 + 1, 0, None) for _ in range(3)],
            [(1, [0, 1]), (-1, [2])])


def gathered(addr, K, r_addr):
    eq = np.concatenate([F.ints_to_limbs(O.eq_evals(list(r_addr))), np.zeros((1, 4), np.uint64)])
    idx = addr.astype(np.int64)
    idx[idx >= K] = K
    return np.ascontiguousarray(eq[idx])


def make_member(sess, route, cols, dev_cols, mons, w, order):
    if route == "today":
        polys = []
        for (kind, a, K, r) in cols:
            if kind == "one_hot":
                polys.append(Polynomial.new(sess, gathered(a, K, r)))
            elif kind == "compact":
                polys.append(Polynomial.from_small(sess, a))
            else:
                polys.append(Polynomial.new(sess, a))
        return ExpressionMember(sess, polys, mons, w, order=order)
    srcs = []
    for (kind, a, K, r), d in zip(cols, dev_cols):
        col = d if route == "sources_device" else a
        if kind == "one_hot":
            srcs.append(Source.one_hot(col, K, r))
        elif kind == "compact":
            srcs.append(Source.compact(col))
        else:
            srcs.append(Source.table(Polynomial.new(sess, a)))
    return ExpressionMember.from_sources(sess, srcs, mons, w, order=order)


def whole_call(sess, route, cols, dev_cols, mons, w, order, n, claim):
    """member creation, every round, the terminal bind and the final evaluations; returns (ms, round evals, finals)"""
    sess.synchronize()
    t0 = time.perf_counter()
    m = make_member(sess, route, cols, dev_cols, mons, w, order)
    polys, bind = [], None
    for rnd in range(n):
        ev = m.prove_round_evals(bind, rnd, claim)
        polys.append(ev)
        bind = rand_challenge(0xD000 + rnd)
        claim = jolt_b200.UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
    m.finish_rounds(bind)
    fin = m.final_evals()
    dt = (time.perf_counter() - t0) * 1e3
    m.close()
    return dt, polys, fin


def member_bytes(route, cols, n, order):
    T = 1 << n
    alt = order == LOW_TO_HIGH
    b = 0
    for kind, a, K, _ in cols:
        if route == "today" or kind == "table":
            b += T * 32 + (T // 2 * 32 if alt else 0)
        else:
            b += a.nbytes + T // 2 * 32 + (T // 4 * 32 if alt else 0) + (K * 32 if kind == "one_hot" else 0)
    return b


def pass_work(cols, mons, bind):
    """(HBM bytes, full-product equivalents) per pair of a source pass (eq weighted, s(1) from the claim)"""
    D = max(len(t) for _, t in mons)
    muls = 2.0   # the split-eq weight, and its product with the pair's sum
    for t in [0] + list(range(2, D)) + ["inf"]:
        for c, tabs in mons:
            if t == "inf" and len(tabs) < D:
                continue
            muls += len(tabs) - 1 + (0 if c % P in (1, P - 1) else 1)
        muls += 1
    reads = 4 if bind else 2
    by = 0
    for kind, a, K, _ in cols:
        w = a.itemsize if a.ndim == 1 else 32
        by += reads * (32 if kind == "table" else w) + (2 * 32 if bind else 0) + (2 * 32 if bind and kind == "table" else 0)
        if kind == "compact":
            muls += reads          # the promotions (one product each)
        if bind:
            muls += 2 * 0.5        # two binds with a 125-bit challenge (~half a product each)
    return by, muls


def run(sess, name, n, order, steps, rate, info, emit):
    import torch
    cols, mons = columns(name, n)
    dev_cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() if k != "table" else None for k, a, _, _ in cols]
    w = np.stack([rand_challenge(0x5100 + i) for i in range(n)])
    # the claim: s(0) + s(1) of the first round with eq(w, .) as a table (an eq member needs the claim to start)
    m = make_member(sess, "today", [("table", EqPolynomial.evals(sess, w).evals(), 0, None)] + cols, None,
                    [(c, [0] + [t + 1 for t in tabs]) for c, tabs in mons], None, order)
    ev = m.prove_round_evals(None, 0, None)
    claim = (ev[0] + ev[1]) % P
    m.close()
    routes = ["today", "sources_host", "sources_device"]
    ref = None
    for r in routes:   # the outputs must agree before anything is timed
        _, polys, fin = whole_call(sess, r, cols, dev_cols, mons, w, order, n, claim)
        ref = ref or (polys, fin)
        assert (polys, fin) == ref, f"{name}: route {r} disagrees with today's route"
    times = {r: [] for r in routes}
    for _ in range(steps):
        for r in routes:
            times[r].append(whole_call(sess, r, cols, dev_cols, mons, w, order, n, claim)[0])
    sess.timing_enable(True, 1 << (n - 3))
    whole_call(sess, "sources_device", cols, dev_cols, mons, w, order, n, claim)
    passes = sess.timing_collect()
    sess.timing_enable(False)
    pairs0, pairs1 = 1 << (n - 1), 1 << (n - 2)
    rec = dict(workload=name, order="l2h" if order == LOW_TO_HIGH else "h2l", log_n=n,
               whole_call_ms={r: round(statistics.median(t), 2) for r, t in times.items()},
               member_bytes={r: member_bytes(r, cols, n, order) for r in ("today", "sources_host")})
    for label, bind, pairs in (("round0_eval", False, pairs0), ("round1_bind", True, pairs1)):
        ms = sum(p["ms"] for p in passes if p["items"] == pairs and p["kind"] == ("fused_bind_eval" if bind else "eval_only"))
        b, mu = pass_work(cols, mons, bind)
        t_hbm, t_int = b * pairs / HBM_PEAK * 1e3, mu * pairs / rate * 1e3
        rec[label] = dict(ms=round(ms, 4), hbm_bound_ms=round(t_hbm, 4), int_bound_ms=round(t_int, 4),
                          bound="hbm" if t_hbm >= t_int else "int", share_of_bound=round(max(t_hbm, t_int) / ms, 3) if ms else None)
    rec.update(info)
    emit(rec)
    del dev_cols


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="22,24")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--orders", default="l2h,h2l")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
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
    for n in (int(x) for x in a.log_n.split(",")):
        for o in a.orders.split(","):
            for name in a.workloads.split(","):
                run(sess, name, n, LOW_TO_HIGH if o == "l2h" else HIGH_TO_LOW, a.steps, rate, info, emit)
    sess.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
