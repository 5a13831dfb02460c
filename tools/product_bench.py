"""Product members over sources (jb_member_create_product_sources) at 2^N.

Workloads (all factors one-hot address columns with 5 % none values; eq(w, .) kept split unless noted):
  d4_u8, d6_u8      4 / 6 one-hot u8 chunks (K = 256) with eq - shapes the expression member over sources
                    (jb_member_create_expr_sources, one monomial) also runs: both are timed, alternating
  d8_u8, d12_u8     8 / 12 one-hot u8 chunks (K = 256) with eq
  d8_u16, d12_u16   8 / 12 one-hot u16 chunks (K = 2^16) with eq
  d9_u16_val        8 one-hot u16 chunks (K = 2^16) and a value table, with eq
  d16_u8, d16_u16   16 one-hot chunks (K = 256 / 2^16), no eq (a 128-bit index in 16 chunks of 8 bits)

Per workload, the median wall time of the whole call from device columns (torch tensors) - member creation, every round
(fixed 125-bit challenges, s(1) from the claim), the terminal bind and the final evaluations; for d >= 8 also the
same call from host columns. Round polynomials and final evaluations of every route are checked equal before anything
is timed (and the final claim against the product of the final evaluations). Then the device time of the round-0
(eval-only), round-1 (source bind) and round-2 (field-table bind) passes (jb_ctx_timing_*), each against the larger
of its HBM bound (bytes over the H100 SXM data-sheet 3.35 TB/s) and its integer bound (full Montgomery products of
DESIGN section 4 over the rate jb_diag_mul_throughput measures in the same run; a 125-bit bind counts as half a
product). Reads the card's name and power limit in the same run. JSON lines on stdout (and to --out).

usage: python tools/product_bench.py [--log-n 22,24] [--steps 3] [--workloads ...] [--out FILE]"""
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
from jolt_b200 import EqPolynomial, ExpressionMember, LOW_TO_HIGH, Polynomial, ProductMember, Source  # noqa: E402
from jolt_b200 import field as F  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from oracle.coracle import rand_challenge, rand_limbs  # noqa: E402
from expr_bench import HBM_PEAK, card, mul_rate  # noqa: E402

P = F.R_MOD
# name -> (one-hot chunks, address dtype, K, value table, eq)
WORKLOADS = {
    "d4_u8": (4, np.uint8, 256, False, True), "d6_u8": (6, np.uint8, 256, False, True),
    "d8_u8": (8, np.uint8, 256, False, True), "d8_u16": (8, np.uint16, 1 << 16, False, True),
    "d9_u16_val": (8, np.uint16, 1 << 16, True, True),
    "d12_u8": (12, np.uint8, 256, False, True), "d12_u16": (12, np.uint16, 1 << 16, False, True),
    "d16_u8": (16, np.uint8, 256, False, False), "d16_u16": (16, np.uint16, 1 << 16, False, False),
}


def tree_products(d, eq):
    """full Montgomery products per pair of product_round_kernel with s(1) from the claim (binary-counter merges:
    a + b + 1 per merge, the root skips s(1); with eq the pair's weight and its product into the first leaf)"""
    stk, cost = [], 0
    for _ in range(d):
        stk.append((1, 1))
        while len(stk) >= 2 and stk[-1][1] == stk[-2][1]:
            (a, la), (b, lb) = stk.pop(-2), stk.pop()
            stk.append((a + b, la + lb))
            cost += a + b + 1
    while len(stk) >= 2:
        (a, la), (b, lb) = stk.pop(-2), stk.pop()
        stk.append((a + b, la + lb))
        cost += a + b + 1
    return cost - (1 if d >= 2 else 0) + (3 if eq else 0)


def expr_products(d, eq):
    """the same for the expression pass with one monomial: (d - 1) products per point, one weighting per point"""
    pts = d if d >= 2 else 1
    return pts * (d - 1) + (pts + 1 if eq else 0)


def pass_work(shape, rnd, products):
    """(HBM bytes, full-product equivalents) per pair of pass `rnd` (0: read the columns, 1: bind them, 2: tables)"""
    by = 0
    for itemsize in shape:
        if rnd == 0:
            by += 2 * itemsize
        elif rnd == 1:
            by += 4 * itemsize + 2 * 32
        else:
            by += 4 * 32 + 2 * 32
    return by, products + (len(shape) if rnd else 0)   # two 125-bit binds per factor ~ one product


class Workload:
    def __init__(self, sess, name, n):
        import torch
        d, dt, K, val, eq = WORKLOADS[name]
        rng = np.random.default_rng(0x7700 + n)
        self.cols = []
        for _ in range(d):
            a = rng.integers(0, K, 1 << n).astype(dt)
            a[rng.random(1 << n) < 0.05] = np.iinfo(dt).max
            self.cols.append(a)
        self.dev = [torch.from_numpy(a).cuda() for a in self.cols]
        self.K = K
        self.r = [O.random_fr(0x7800 + i, K.bit_length() - 1) for i in range(d)]
        self.val = rand_limbs(0x7900, 1 << n) if val else None
        self.w = np.stack([rand_challenge(0x7A00 + i) for i in range(n)]) if eq else None
        self.n, self.d = n, d + (1 if val else 0)
        self.shape = [a.itemsize for a in self.cols] + ([32] if val else [])
        # the claim: s(0) + s(1) of round 0 of the product without eq (eq(w, .) as one more table source, d <= 13)
        srcs = self.sources(sess, True) + ([Source.table(EqPolynomial.evals(sess, self.w))] if eq else [])
        m = ProductMember.from_sources(sess, srcs)
        ev = m.prove_round_evals(None, 0, None)
        m.close()
        self.claim = (ev[0] + ev[1]) % P

    def sources(self, sess, device):
        srcs = [Source.one_hot(dc if device else a, self.K, r) for a, dc, r in zip(self.cols, self.dev, self.r)]
        if self.val is not None:
            srcs.append(Source.table(Polynomial.new(sess, self.val)))
        return srcs

    def member(self, sess, route):
        srcs = self.sources(sess, route != "product_host")
        if route == "expr":
            return ExpressionMember.from_sources(sess, srcs, [(1, list(range(self.d)))], self.w, order=LOW_TO_HIGH)
        return ProductMember.from_sources(sess, srcs, self.w, order=LOW_TO_HIGH)


def whole_call(sess, wl, route):
    sess.synchronize()
    t0 = time.perf_counter()
    m = wl.member(sess, route)
    polys, bind, claim = [], None, wl.claim
    for rnd in range(wl.n):
        ev = m.prove_round_evals(bind, rnd, claim)
        polys.append(ev)
        bind = rand_challenge(0x7B00 + rnd)
        claim = jolt_b200.UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
    m.finish_rounds(bind)
    fin = m.final_evals()
    dt = (time.perf_counter() - t0) * 1e3
    prod = m.eq_scalar() if wl.w is not None else 1
    for v in fin:
        prod = prod * v % P
    assert prod == claim, f"{route}: final claim != eq scalar x prod of the final evaluations"
    m.close()
    return dt, polys, fin


def passes(sess, wl, route):
    sess.timing_enable(True, 1 << (wl.n - 3))
    whole_call(sess, wl, route)
    ps = sess.timing_collect()
    sess.timing_enable(False)
    out = {}
    for rnd, kind in ((0, "eval_only"), (1, "fused_bind_eval"), (2, "fused_bind_eval")):
        pairs = 1 << (wl.n - 1 - rnd)
        out[rnd] = sum(p["ms"] for p in ps if p["items"] == pairs and p["kind"] == kind)
    return out


def run(sess, name, n, steps, rate, info, emit):
    wl = Workload(sess, name, n)
    routes = ["product_device", "expr"] if wl.d <= 6 else ["product_device", "product_host"]
    ref = None
    for r in routes:   # the outputs must agree before anything is timed
        _, polys, fin = whole_call(sess, wl, r)
        ref = ref or (polys, fin)
        assert (polys, fin) == ref, f"{name}: route {r} disagrees"
    times = {r: [] for r in routes}
    for _ in range(steps):
        for r in routes:
            times[r].append(whole_call(sess, wl, r)[0])
    rec = dict(workload=name, log_n=n, d=wl.d, eq=wl.w is not None,
               whole_call_ms={r: round(statistics.median(t), 2) for r, t in times.items()})
    eq = wl.w is not None
    for r in (routes if wl.d <= 6 else routes[:1]):
        ms = passes(sess, wl, r)
        prods = tree_products(wl.d, eq) if r != "expr" else expr_products(wl.d, eq)
        per = {}
        for rnd, label in ((0, "round0_read"), (1, "round1_source_bind"), (2, "round2_table_bind")):
            pairs = 1 << (n - 1 - rnd)
            b, mu = pass_work(wl.shape, rnd, prods)
            t_hbm, t_int = b * pairs / HBM_PEAK * 1e3, mu * pairs / rate * 1e3
            per[label] = dict(ms=round(ms[rnd], 4), hbm_bound_ms=round(t_hbm, 4), int_bound_ms=round(t_int, 4),
                              bound="hbm" if t_hbm >= t_int else "int",
                              share_of_bound=round(max(t_hbm, t_int) / ms[rnd], 3) if ms[rnd] else None)
        rec[f"passes_{r}"] = dict(products_per_pair=prods, **per)
    rec.update(info)
    emit(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="22,24")
    ap.add_argument("--steps", type=int, default=3)
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
        for name in a.workloads.split(","):
            run(sess, name, n, a.steps, rate, info, emit)
    sess.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
