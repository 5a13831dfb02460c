"""A/B of the degree-2 eval-only sweep (round 0 of the 2^22 m = 2 sumcheck): two LDG.128 per element per thread + software pipelining
(fused_round_kernel) against TMA-staged evaluation blocks (eval2_tma_kernel, cp.async.bulk + mbarrier). Both through the
C ABI with one launch per round (JB_NO_TAIL) so the kernels can be timed with CUDA events and captured by ncu.
Usage: python tools/tma_ab.py [log_n]   (run under ncu with -k regex:'eval2_tma|fused_round' for the full captures)"""
import json, os, sys, pathlib
import numpy as np
import torch
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import jolt_b200
from jolt_b200 import HIGH_TO_LOW, LOW_TO_HIGH, Polynomial, ProductMember
from jolt_b200 import field as F

lg = int(sys.argv[1]) if len(sys.argv) > 1 else 22
n = 1 << lg
peak = 3350.0  # GB/s, H100 SXM data-sheet HBM3 bandwidth
try:
    peak = json.load(open(ROOT / "MEASURED_PEAKS.json"))["hbm_gbs"]
except Exception:
    pass
stream = torch.cuda.Stream()      # the session runs on torch's current stream: the L2 flush is ordered before each pass
torch.cuda.set_stream(stream)
g = torch.Generator(device="cuda").manual_seed(1)
tabs = []
for j in range(2):
    t = torch.randint(0, 2 ** 62, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    t[:, 3] &= (1 << 60) - 1
    tabs.append(t)
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
out = {}
os.environ["JB_NO_TAIL"] = "1"
for variant in ("ldg", "tma"):
    if variant == "tma":
        os.environ["JB_EVAL_TMA"] = "1"
    else:
        os.environ.pop("JB_EVAL_TMA", None)
    sess = jolt_b200.Session(0, cuda_stream=stream.cuda_stream)
    for order, oname in ((LOW_TO_HIGH, "l2h"), (HIGH_TO_LOW, "h2l")):
        probe = ProductMember(sess, [Polynomial.wrap_device(sess, t.data_ptr(), n) for t in tabs], order)
        ev = probe.prove_round_evals(None, 0)       # all points, no claim: the reference value
        claim = (ev[0] + ev[1]) % F.R_MOD
        sess.timing_enable(True, min_items=1)
        sess.timing_collect()
        res = None
        for rep in range(11):
            flush.zero_()
            mem = ProductMember(sess, [Polynomial.wrap_device(sess, t.data_ptr(), n) for t in tabs], order)
            res = mem.prove_round_evals(None, 0, claim)   # eval-only, s(1) from the claim
            mem.close()
        ms = [t["ms"] for t in sess.timing_collect() if t["kind"] == "eval_only"][1:]
        sess.timing_enable(False)
        assert res == ev, "variant disagrees with the all-points pass"
        best = min(ms)
        out[f"{variant}_{oname}"] = {"ms_best": best, "ms_median": sorted(ms)[len(ms) // 2],
                                     "gb_per_s": 2 * 64 * (n // 2) / (best * 1e-3) / 1e9,
                                     "frac_of_hbm_peak": 2 * 64 * (n // 2) / (best * 1e-3) / 1e9 / peak}
        probe.close()
    sess.close()
print(json.dumps({"log_n": lg, "m": 2, "algorithmic_bytes": 2 * 64 * (n // 2), "peak_gb_per_s": peak, "runs": out}, indent=1))
