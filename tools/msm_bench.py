"""G1 MSM throughput on one H100 (BASELINE config 3): terms/s at 2^16..2^24, synthetic bases
(i+1)*G generated on the device, uniform 253-bit scalars resident in HBM; the result is checked
against the closed form at every size. CPU = the C restatement's Pippenger on all host cores."""
import json, sys, time, pathlib
import numpy as np
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import jolt_b200
from jolt_b200 import G1Bases, Polynomial, g1_jacobian_to_affine
from oracle import bn254 as O
from oracle import coracle as C
from test_gpu_msm import _weighted_sum, G

sizes = [int(a) for a in sys.argv[1:] if a.isdigit()] or [16, 20, 22, 24]
cpu = "--cpu" in sys.argv
sess = jolt_b200.Session(0)
out = []
for lg in sizes:
    n = 1 << lg
    t0 = time.perf_counter()
    bases = G1Bases.generate_multiples(sess, G, n)
    gen_s = time.perf_counter() - t0
    pre_s = 0.0
    if "--pre" in sys.argv:
        t0 = time.perf_counter()
        cw = [int(a[4:]) for a in sys.argv if a.startswith("--c=")]
        bases.precompute(cw[0] if cw else 0)
        pre_s = time.perf_counter() - t0
    sc = C.rand_limbs(0x5CA1A2, n)
    tab = Polynomial.new(sess, sc)
    sess.synchronize()
    sess.timing_enable(True, 0)
    res = bases.msm(tab)            # warm-up + correctness
    ok = g1_jacobian_to_affine(res) == O.g1_scalar_mul(O.G1_GEN, _weighted_sum(sc))
    sess.timing_collect()
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        bases.msm(tab)
        ts.append(time.perf_counter() - t0)
    acc = [t["ms"] for t in sess.timing_collect() if t["kind"] == "msm_accumulate"]
    sess.timing_enable(False)
    t0 = time.perf_counter()
    bases.msm(sc)                   # host scalars: + H2D of 32 B/term
    e2e = time.perf_counter() - t0
    rec = dict(kind="msm", log_n=lg, ok=bool(ok), ms=round(min(ts) * 1e3, 3), mterms_per_s=round(n / min(ts) / 1e6, 1),
               accumulate_ms=round(sum(acc) / max(len(acc), 1), 3), e2e_ms=round(e2e * 1e3, 3), srs_generate_s=round(gen_s, 2), precompute_s=round(pre_s, 2))
    if cpu and lg <= 20:
        xy = bases.affine()
        t0 = time.perf_counter()
        C.g1_msm_pippenger(xy, sc, 0, C.max_threads())
        rec["cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        rec["cpu_cores"] = C.max_threads()
    if "--small" in sys.argv:
        # primitive-integer columns (legacy msm_u8 .. msm_i64): host scalars, so each time includes the H2D of
        # 1..8 B/term; checked against the same closed form over the integers
        rng = np.random.default_rng(lg)
        cols = {"u8": rng.integers(0, 256, size=n, dtype=np.uint8), "binary": rng.integers(0, 2, size=n).astype(np.uint8),
                "u16": rng.integers(0, 1 << 16, size=n, dtype=np.uint16), "u32": rng.integers(0, 1 << 32, size=n, dtype=np.uint32),
                "u64": rng.integers(0, 1 << 64, size=n, dtype=np.uint64), "i64": rng.integers(-(1 << 63), 1 << 63, size=n, dtype=np.int64)}
        small = {}
        for name, col in cols.items():
            r0 = bases.msm_small(col)
            wsum = int((col.astype(object) * np.arange(1, n + 1, dtype=object)).sum()) % O.R_MOD if n <= (1 << 20) else None
            good = wsum is None or g1_jacobian_to_affine(r0) == O.g1_scalar_mul(O.G1_GEN, wsum)
            tt = []
            for _ in range(3):
                t0 = time.perf_counter()
                bases.msm_small(col)
                tt.append(time.perf_counter() - t0)
            small[name] = dict(ms=round(min(tt) * 1e3, 3), ok=bool(good))
        rec["small"] = small
    print(json.dumps(rec), flush=True)
    out.append(rec)
    bases.free(); tab.free()
(ROOT / "gpurun_out").mkdir(exist_ok=True)
with open(ROOT / "gpurun_out" / "msm_bench.jsonl", "w") as f:
    for r in out:
        f.write(json.dumps(r) + "\n")
