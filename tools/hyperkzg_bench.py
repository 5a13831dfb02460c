"""HyperKZG commit + open timing on one H100 (device-resident SRS and polynomial)."""
import json, sys, time, pathlib
import numpy as np
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import jolt_b200
from jolt_b200 import G1Bases, HyperKZG, Polynomial
from oracle import bn254 as O
from oracle import coracle as C

G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
sess = jolt_b200.Session(0)
pre = "--pre" in sys.argv
for ell in [int(a) for a in sys.argv[1:] if a.isdigit()] or [14, 18, 20, 22]:
    n = 1 << ell
    bases = G1Bases.generate_multiples(sess, G, n)
    if pre:
        bases.precompute()
    poly = Polynomial.new(sess, C.rand_limbs(1, n))
    point = np.stack([C.rand_challenge(7 + i) for i in range(ell)])
    HyperKZG.commit(bases, poly)
    t0 = time.perf_counter(); HyperKZG.commit(bases, poly); tc = time.perf_counter() - t0
    HyperKZG.open(bases, poly, point, lambda c: 12345, lambda v: 6789)
    l0 = sess.launch_count
    t0 = time.perf_counter(); HyperKZG.open(bases, poly, point, lambda c: 12345, lambda v: 6789); to = time.perf_counter() - t0
    print(json.dumps(dict(kind="hyperkzg", ell=ell, precomputed_srs=pre, commit_ms=round(tc * 1e3, 3), open_ms=round(to * 1e3, 3),
                          open_launches=sess.launch_count - l0)), flush=True)
    bases.free(); poly.free()
