"""The booleanity member (jb_member_create_booleanity) on one GPU: the whole call from device columns.

Workloads (uniform random addresses, 10 % none cycles), each at T = 2^20, 2^22, 2^24:
  - d = 16, K = 256, u8 (instruction-RA-shaped chunks);
  - d = 32, K = 16, u8;
  - d = 8, K = 2^16, u16.
Reports per workload:
  - ms: host wall time of creation + every round + final evaluations (final_evals waits for the device); median of 3
    after 1 warm-up, 125-bit challenges;
  - addr_dev_ms / cycle_dev_ms: device time of the address-phase and cycle-phase round passes (CUDA events around each
    launch, one extra run with timing on);
  - cycle_bound_ms: the cycle rounds after the column rounds against the larger of their byte bound (d x 96 B per
    pair of the table they bind: two entries read, one written, over the data-sheet 3.35 TB/s) and their integer bound
    (per pair of the round they evaluate 6 d + 3 Montgomery products - two binds, lo^2, (hi - lo)^2 and two c_i
    products per table, the split-eq weight - over the jb_diag_mul_throughput rate measured in the same run);
  - today_ms / member_cycle_ms: today's route for the cycle phase - ceil(d / 8) expression members over one-hot sources
    (r_addr = the bound address point, eq point r_cycle, eq_scale = scale eq(r_addr, rho_addr)) proving the same rounds,
    driven round by round - against the member's own cycle rounds (host wall time of the rounds, the terminal bind and
    the final evaluations, both from the same state); the round polynomials are checked to agree (the members' sum).
Reads the card's name, power limit, maximum and current SM clock in the same run. One JSON line per workload on
stdout, and in FILE with --out.

usage: python tools/booleanity_bench.py [--out FILE] [--quick]"""
import argparse
import json
import pathlib
import statistics
import sys
import time

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import jolt_b200  # noqa: E402
from jolt_b200 import LOW_TO_HIGH, BooleanityMember, ExpressionMember, Source  # noqa: E402
from jolt_b200 import field as F  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from lincomb_bench import HBM_BYTES_PER_S, card  # noqa: E402
from expr_bench import mul_rate  # noqa: E402
from rw_bench import sm_clocks  # noqa: E402

P = O.R_MOD


def challenges(seed, n):
    rng = np.random.default_rng(seed)
    return [F.from_limbs(np.array([0, 0, int(rng.integers(0, 1 << 63)), int(rng.integers(0, 1 << 61))], dtype=np.uint64))
            for _ in range(n)]


def columns(seed, K, T, d):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    none = 0xFF if K <= 256 else 0xFFFF
    out = []
    for _ in range(d):
        a = torch.randint(0, min(K, none), (T,), generator=g, device="cuda", dtype=torch.int32)
        a[torch.rand(T, generator=g, device="cuda") < 0.1] = none
        out.append(a.to(torch.uint8) if K <= 256 else a.to(torch.int16))
    torch.cuda.synchronize()
    return out


def drive(m, ch, first, claim, stop=None):
    """Rounds first .. stop - 1 of m at ch (bind = ch[round - 1]); returns (polys, claim)."""
    polys = []
    stop = len(ch) if stop is None else stop
    for rnd in range(first, stop):
        s = m.prove_round_evals(ch[rnd - 1] if rnd else None, rnd, claim)
        polys.append(s)
        claim = O.uni_evaluate(O.uni_from_evals(s), ch[rnd])
    return polys, claim


def run(sess, K, T, d, mrate, reps, order=LOW_TO_HIGH):
    cols = columns(K + d, K, T, d)
    lk, lt = K.bit_length() - 1, T.bit_length() - 1
    n = lk + lt
    coeffs = O.random_fr(1, d)
    r_addr, r_cycle, scale = O.random_fr(2, lk), O.random_fr(3, lt), O.random_fr(4, 1)[0]
    ch = challenges(5, n)

    def whole():
        m = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, scale, order)
        drive(m, ch, 0, 0)
        m.finish_rounds(ch[-1])
        m.final_evals()
        m.close()

    whole()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        whole()
        ts.append((time.perf_counter() - t0) * 1e3)

    sess.timing_enable(True)
    whole()
    passes = [t for t in sess.timing_collect() if t["kind"] in ("fused_bind_eval", "eval_only") and t["m"] == 2]
    sess.timing_enable(False)
    addr = passes[:lk]
    cyc = passes[lk:]
    # cycle rounds 2 .. lt - 1 bind field tables: pairs of the round they evaluate = items
    bound_s = 0.0
    for t in cyc[2:]:
        pairs = t["items"]
        bytes_ = d * 96 * (2 * pairs)
        prods = (6 * d + 3) * pairs
        bound_s += max(bytes_ / HBM_BYTES_PER_S, prods / mrate)
    out = dict(d=d, K=K, T=T, ms=round(statistics.median(ts), 2), addr_dev_ms=round(sum(t["ms"] for t in addr), 3),
               cycle_dev_ms=round(sum(t["ms"] for t in cyc), 3),
               cycle_tables_dev_ms=round(sum(t["ms"] for t in cyc[2:]), 3), cycle_bound_ms=round(bound_s * 1e3, 3))

    # today's route against the member's cycle rounds, from the same state (the first run warms both up)
    compare(sess, cols, K, T, d, coeffs, r_addr, r_cycle, scale, ch, order)
    out.update(compare(sess, cols, K, T, d, coeffs, r_addr, r_cycle, scale, ch, order))
    return out


def compare(sess, cols, K, T, d, coeffs, r_addr, r_cycle, scale, ch, order):
    lk, lt = K.bit_length() - 1, T.bit_length() - 1
    # today's route for the cycle phase, from the same state: the address rounds of the member (and of one member per
    # group of 8 columns, whose running claims seed the expression members) at the same challenges
    groups = [list(range(g, min(d, g + 8))) for g in range(0, d, 8)]
    m = BooleanityMember(sess, cols, K, coeffs, r_addr, r_cycle, scale, order)
    _, claim = drive(m, ch, 0, 0, lk)
    ra_bound = ch[:lk][::-1] if order == LOW_TO_HIGH else ch[:lk]
    eq_scale = scale * O.evaluate(O.eq_evals(r_addr), ra_bound) % P
    seeds = []
    for grp in groups:
        sub = BooleanityMember(sess, [cols[i] for i in grp], K, [coeffs[i] for i in grp], r_addr, r_cycle, scale, order)
        seeds.append(drive(sub, ch, 0, 0, lk)[1])
        sub.close()
    exprs = []
    for grp in groups:
        srcs = [Source.one_hot(cols[i], K, ra_bound) for i in grp]
        mons = [mo for j, i in enumerate(grp) for mo in ((coeffs[i], [j, j]), ((P - coeffs[i]) % P, [j]))]
        exprs.append(ExpressionMember.from_sources(sess, srcs, mons, w_limbs=F.ints_to_limbs(r_cycle), scale=eq_scale,
                                                   order=order))
    # the member's cycle rounds, then the expression members' rounds at the same challenges
    ch_c = ch[lk:]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    polys = []
    c = claim
    for rnd in range(lt):
        s = m.prove_round_evals(ch[lk + rnd - 1] if lk + rnd else None, lk + rnd, c)
        polys.append(s)
        c = O.uni_evaluate(O.uni_from_evals(s), ch_c[rnd])
    m.finish_rounds(ch[-1])
    m.final_evals()
    member_ms = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    claims = list(seeds)
    sums = []
    for rnd in range(lt):
        ps = [e.prove_round_evals(ch_c[rnd - 1] if rnd else None, rnd, cl) for e, cl in zip(exprs, claims)]
        sums.append([sum(v) % P for v in zip(*ps)])
        claims = [O.uni_evaluate(O.uni_from_evals(p), ch_c[rnd]) for p in ps]
    for e in exprs:
        e.finish_rounds(ch[-1])
        e.final_evals()
    today_ms = (time.perf_counter() - t0) * 1e3
    m.close()
    for e in exprs:
        e.close()
    return dict(member_cycle_ms=round(member_ms, 2), today_ms=round(today_ms, 2), today_members=len(exprs),
                agree=sums == polys)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--quick", action="store_true", help="T = 2^20 only")
    args = ap.parse_args()
    name, power = card()
    smax, scur = sm_clocks()
    sess = jolt_b200.Session(0)
    mrate = mul_rate(sess)
    head = dict(card=name, power_limit=power, sm_clock_max=smax, sm_clock=scur, mul_rate_gops=round(mrate / 1e9, 1))
    print(json.dumps(head), flush=True)
    lines = [head]
    for d, K in ((16, 256), (32, 16), (8, 1 << 16)):
        for lt in ((20,) if args.quick else (20, 22, 24)):
            r = run(sess, K, 1 << lt, d, mrate, 3)
            print(json.dumps(r), flush=True)
            lines.append(r)
    sess.close()
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))
    return 0 if all(x.get("agree", True) for x in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
