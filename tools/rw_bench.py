"""The read-write checking member (jb_member_create_read_write) on one GPU: the whole call from device columns.

Workloads:
  - registers-shaped: K = 128, A = 3 (rs1, rs2 reads, rd write, each its own u8 column, 10 % none), T = 2^20, 2^22, 2^24;
  - RAM-shaped: K = 2^16, one u16 column read (c = 1, d = 0) and written (c = gamma, d = 1), 5 % none cycles, T = 2^22,
    with uniform addresses and with a local stream (a random walk of step -2..2);
  - RAM at a real address space: K = 2^22, one u32 column (none = 0xFFFFFFFF), otherwise as above, T = 2^22.
Values are u64 columns, inc an i64 column (0 where the write is none), init u64. The member does not check the value
precondition and the rounds' cost does not depend on it, so the values are random. Reports per workload:
  - ms: host wall time of creation + every round + final evaluations (final_evals waits for the device); median of 3
    after 1 warm-up; create_ms and round_ms (per round: its bind and evaluation passes and the read-back of its result,
    host wall time) of the last repetition;
  - live: the live entries after each cycle bind (computed on the host from the columns);
  - bound_ms: entry bytes over the data-sheet 3.35 TB/s: per cycle round the evaluation and the bind read the n live
    entries and the bind writes the n' bound ones, (2 n + n') x (8 + 32 (A + 3)) bytes.
Dense route (registers, T = 2^20): the expression member over the materialised tables (ra_a, Val, inc and a replicated
eq table, 6 x 2^27 entries) proving the same rounds, tables already on the device: dense_rounds_ms (every round + final
evaluations, median of 2 after 1 warm-up) next to the member's rw_ms on the same columns; both agree round by round.
With --cycle-rounds-first P,... every workload runs once per p (jb_member_create_read_write_phases; "t" and "t/2" stand
for log2 T and its half) instead of the dense route, and also reports phase_ms: the host wall time of the p cycle
rounds, of the log2 K address rounds and of the remaining cycle rounds (the first address round includes the re-sort by
key, the first remaining cycle round the dense tables).
Reads the card's name, power limit, maximum and current SM clock in the same run. One JSON line per workload on stdout, and in FILE with --out.

usage: python tools/rw_bench.py [--out FILE] [--quick] [--only PREFIX] [--cycle-rounds-first P,...]"""
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
sys.path.insert(0, str(ROOT / "tests"))
import jolt_b200  # noqa: E402
from jolt_b200 import ReadWriteCheckingMember, Source, evaluate_small  # noqa: E402
from oracle import bn254 as O  # noqa: E402
from lincomb_bench import HBM_BYTES_PER_S, card  # noqa: E402
import rw_ref as R  # noqa: E402


def sm_clocks():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return [f"unknown ({e})", "unknown"]


def none_of(K):
    return 0xFF if K <= 256 else 0xFFFF if K <= (1 << 16) else 0xFFFFFFFF


def columns(rng, K, T, n, none_frac, local):
    none = none_of(K)
    hi = min(K, none)
    out = []
    for _ in range(n):
        a = (np.cumsum(rng.integers(-2, 3, T)) % hi) if local else rng.integers(0, hi, T)
        a = a.astype(np.uint8 if K <= 256 else np.uint16 if K <= (1 << 16) else np.uint32)
        a[rng.random(T) < none_frac] = none
        out.append(a)
    return out


def live_entries(cols, K, T):
    """Distinct (row, address) pairs after each of the log2 T cycle binds, starting from the unbound matrix."""
    none = none_of(K)
    j = np.arange(T, dtype=np.int64)
    x = np.concatenate([j[c != none] * K + c[c != none].astype(np.int64) for c in cols])
    x = np.unique(x)
    out = [int(x.size)]
    while T > 1:
        x = np.unique((x // K >> 1) * K + x % K)
        T //= 2
        out.append(int(x.size))
    return out


def run(sess, wl, reps, p=None):
    K, T, cols, acc_spec, write = wl["K"], wl["T"], wl["cols"], wl["acc"], wl["write"]
    rng = np.random.default_rng(1)
    dev_cols = [torch.from_numpy(c.view({1: np.uint8, 2: np.int16, 4: np.int32}[c.itemsize])).cuda() for c in cols]
    vals = [torch.from_numpy(rng.integers(0, 1 << 62, T).astype(np.int64)).cuda() for _ in acc_spec]
    wcol = cols[acc_spec[write][0]]
    none = none_of(K)
    inc = rng.integers(-(1 << 40), 1 << 40, T).astype(np.int64)
    inc[wcol == none] = 0
    inc_t = torch.from_numpy(inc).cuda()
    init_t = torch.from_numpy(rng.integers(0, 1 << 62, K).astype(np.int64)).cuda()
    t, kappa = T.bit_length() - 1, K.bit_length() - 1
    w = O.random_fr(3, t)
    ch = O.random_fr(4, t + kappa)
    coeffs = O.random_fr(5, len(acc_spec))

    times = {}

    def once():
        t0 = time.perf_counter()
        acc = [(dev_cols[ci], Source.compact(vals[a], "u64"), coeffs[a], d) for a, (ci, d) in enumerate(acc_spec)]
        m = ReadWriteCheckingMember(sess, acc, write, Source.compact(inc_t, "i64"), Source.compact(init_t, "u64"), K, w,
                                    cycle_rounds_first=p)
        times["create_ms"] = (time.perf_counter() - t0) * 1e3
        claim, bind, rounds = 1, None, []
        for rnd in range(t + kappa):
            t1 = time.perf_counter()
            m.prove_round_evals(bind, rnd, claim)
            rounds.append(round((time.perf_counter() - t1) * 1e3, 3))
            bind = ch[rnd]
        times["round_ms"] = rounds
        m.finish_rounds(bind)
        m.final_evals()
        m.close()

    once()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        once()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), times


def dense_comparison(sess, reps):
    """The member and the dense expression route on the same registers-shaped columns at T = 2^20."""
    K, T = 128, 1 << 20
    wl = R.columns_workload(5, K, T, "registers")
    t, kappa = 20, 7
    w = O.random_fr(6, t)
    ch = O.random_fr(7, t + kappa)

    def rw_call():
        acc = [(a, Source.compact(v, "u64"), c, d) for a, v, c, d in zip(wl["addrs"], wl["values"], wl["coeffs"], wl["ds"])]
        m = ReadWriteCheckingMember(sess, acc, wl["write"], Source.compact(wl["inc"], "u64"),
                                    Source.compact(wl["init"], "u64"), K, w)
        return m

    ev = evaluate_small(sess, wl["values"] + [wl["inc"]], w, "u64")
    claim0 = sum(c * (v + d * ev[-1]) for c, v, d in zip(wl["coeffs"], ev, wl["ds"])) % O.R_MOD

    def prove(m, out):
        bind, claim = None, claim0
        for rnd in range(t + kappa):
            out.append(m.prove_round_evals(bind, rnd, claim))
            bind = ch[rnd]
            claim = O.uni_evaluate(O.uni_from_evals(out[-1]), bind)
        m.finish_rounds(bind)
        return m.final_evals()

    rw_ts, dense_ts = [], []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        m = rw_call()
        got = []
        fin = prove(m, got)
        rw_ts.append((time.perf_counter() - t0) * 1e3)
        m.close()
        d = R.dense_member(sess, wl, w)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        want = []
        dfin = prove(d, want)
        dense_ts.append((time.perf_counter() - t0) * 1e3)
        d.close()
        assert got == want and fin == dfin[:-1]
    return dict(workload="registers_T2^20_dense_route", K=K, T=T, rw_ms=round(statistics.median(rw_ts[1:]), 3),
                dense_rounds_ms=round(statistics.median(dense_ts[1:]), 3), rounds_agree=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--quick", action="store_true", help="T = 2^16 only (a rehearsal)")
    ap.add_argument("--only", default=None, help="only the workloads whose name starts with this (no dense route)")
    ap.add_argument("--cycle-rounds-first", default=None,
                    help="comma-separated p values (integers, t or t/2): each workload once per p (no dense route)")
    args = ap.parse_args()
    splits = args.cycle_rounds_first.split(",") if args.cycle_rounds_first else [None]

    def resolve(tok, t):
        return None if tok is None else t if tok == "t" else t // 2 if tok == "t/2" else int(tok)
    rng = np.random.default_rng(0)
    name, power = card()
    sess = jolt_b200.Session(0)
    wls = []
    for logt in ([16] if args.quick else [20, 22, 24]):
        T = 1 << logt
        wls.append(dict(name=f"registers_T2^{logt}", K=128, T=T, cols=columns(rng, 128, T, 3, 0.1, False),
                        acc=[(0, 0), (1, 0), (2, 1)], write=2))
    for local in (False, True):
        logt = 16 if args.quick else 22
        T = 1 << logt
        wls.append(dict(name=f"ram_{'local' if local else 'uniform'}_T2^{logt}", K=1 << 16, T=T,
                        cols=columns(rng, 1 << 16, T, 1, 0.05, local), acc=[(0, 0), (0, 1)], write=1))
    for local in (False, True):
        logt, logk = (16, 18) if args.quick else (22, 22)
        T = 1 << logt
        wls.append(dict(name=f"ram_u32_K2^{logk}_{'local' if local else 'uniform'}_T2^{logt}", K=1 << logk, T=T,
                        cols=columns(rng, 1 << logk, T, 1, 0.05, local), acc=[(0, 0), (0, 1)], write=1))
    if args.only:
        wls = [wl for wl in wls if wl["name"].startswith(args.only)]
    lines = []
    for wl in wls:
        A = len(wl["acc"])
        live = live_entries(wl["cols"], wl["K"], wl["T"])
        ebytes = 8 + 32 * (A + 3)
        bound_bytes = sum((2 * live[m] + live[m + 1]) * ebytes for m in range(len(live) - 1))
        t, kappa = wl["T"].bit_length() - 1, wl["K"].bit_length() - 1
        for tok in splits:
            p = resolve(tok, t)
            ms, times = run(sess, wl, 3, p)
            sm_max, sm_now = sm_clocks()
            rec = dict(workload=wl["name"], K=wl["K"], T=wl["T"], A=A, ms=round(ms, 3), live=live,
                       bound_ms=round(bound_bytes / HBM_BYTES_PER_S * 1e3, 3), entry_bytes=ebytes,
                       create_ms=round(times["create_ms"], 3), round_ms=times["round_ms"], card=name, power_limit=power,
                       sm_clock_max=sm_max, sm_clock_after=sm_now)
            if p is not None:
                r = times["round_ms"]
                rec.update(cycle_rounds_first=p, phase_ms=[round(sum(r[:p]), 3), round(sum(r[p:p + kappa]), 3),
                                                           round(sum(r[p + kappa:]), 3)])
            print(json.dumps(rec), flush=True)
            lines.append(json.dumps(rec))
    if not args.quick and not args.only and splits == [None]:
        rec = dense_comparison(sess, 2)
        rec.update(card=name, power_limit=power, sm_clock_max=sm_clocks()[0])
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
    if args.out:
        pathlib.Path(args.out).write_text("\n".join(lines) + "\n")
    sess.close()


if __name__ == "__main__":
    main()
