"""The LT and eq+1 tables on one GPU: jb_lt_evals / jb_eq_plus_one_evals against their bound and against the host route
a caller had before them (the threaded C build of tests/native/structured_ref.c, then jb_table_upload), after checking
that both give the same table.

Workloads: 2^20, 2^22, 2^24 and 2^26 outputs, with a 125-bit point ([0,0,lo,hi] Montgomery limbs, the sumcheck
challenges the relations are evaluated at) and a full 254-bit point, scaled. Reports per workload:
  - ms: the call's device time (CUDA events on the session's stream around the whole call, allocation and the small
    leading tables included; median of 7 after 2 warm-ups), and eq_ms, jb_eq_evals of the same point timed the same way;
  - bound_ms: the larger of 32 B written per output over the data-sheet 3.35 TB/s HBM and the integer work over the
    Montgomery-product rates measured in the same run (jb_diag_mul_throughput, full and [0,0,lo,hi] products). Both
    tables take one full product per 8 outputs and 7 products by a coordinate (the 4-row product for a 125-bit point);
  - host_ms: the host route's wall time (C build on every core, then the upload; median of 3).
Reads the card's name and power limit in the same run. Output: one JSON line per workload on stdout, and in FILE with
--out.

usage: python tools/structured_bench.py [--out FILE] [--quick]"""
import argparse
import ctypes
import json
import pathlib
import statistics
import sys
import time

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import jolt_b200  # noqa: E402
from jolt_b200 import EqPlusOnePolynomial, EqPolynomial, LtPolynomial, Polynomial  # noqa: E402
from oracle import coracle as C  # noqa: E402
import structured_ref as R  # noqa: E402
from lincomb_bench import HBM_BYTES_PER_S, card, device_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small sizes only (a rehearsal of the script)")
    a = ap.parse_args()
    name, power = card()
    s = jolt_b200.Session(0, cuda_stream=torch.cuda.current_stream().cuda_stream)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    rate = {}
    for variant in (0, 1):
        gops = ctypes.c_double()
        s.check(s.lib.jb_diag_mul_throughput(s.h, 0, variant, 4096, sm * 8, ctypes.byref(gops)))
        rate[variant] = gops.value * 1e9
    lines = []
    tables = {"lt": (LtPolynomial, R.lt_evals_c), "eq_plus_one": (EqPlusOnePolynomial, R.eq_plus_one_evals_c)}
    for n in ([12, 14] if a.quick else [20, 22, 24, 26]):
        for kind in ("short", "full"):
            if kind == "short":
                r = np.stack([C.rand_challenge(0x7000 + n * 64 + i) for i in range(n)])
            else:
                r = C.rand_limbs(0x7100 + n, n)
            sc = C.rand_limbs(0x7200 + n, 1)[0]
            for table, (cls, cref) in tables.items():
                got = cls.evals(s, r, sc)
                host = cref(r, sc)
                assert np.array_equal(got.evals(), host), (table, n, kind)
                got.free()
                ms = device_ms(lambda: cls.evals(s, r, sc).free())
                eq_ms = device_ms(lambda: EqPolynomial.evals(s, r, sc).free())

                def host_route():
                    t0 = time.perf_counter()
                    p = Polynomial.new(s, cref(r, sc))
                    dt = (time.perf_counter() - t0) * 1e3
                    p.free()
                    return dt
                host_ms = statistics.median(host_route() for _ in range(3))
                N = 1 << n
                hbm = 32 * N / HBM_BYTES_PER_S
                alu = N / 8 / rate[0] + 7 * N / 8 / rate[1 if kind == "short" else 0]
                bound = max(hbm, alu) * 1e3
                rec = dict(table=table, log_n=n, point=kind, card=name, power_limit=power, ms=round(ms, 4),
                           eq_ms=round(eq_ms, 4), bound_ms=round(bound, 4), bound_by="hbm" if hbm >= alu else "integer",
                           fraction_of_bound=round(bound / ms, 3), full_mont_per_s_g=round(rate[0] / 1e9, 1),
                           hi4_mont_per_s_g=round(rate[1] / 1e9, 1), host_ms=round(host_ms, 2),
                           speedup_vs_host=round(host_ms / ms, 1))
                line = json.dumps(rec)
                print(line, flush=True)
                lines.append(line)
    s.close()
    if a.out:
        pathlib.Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
