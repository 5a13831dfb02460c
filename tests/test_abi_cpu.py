"""CPU-side checks: the C-ABI library loads without a GPU, exports every symbol include/jolt_b200.h
declares, fails loudly (no fallback) when no device exists, and the host glue matches the oracle."""
import ctypes
import pathlib
import re

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import _lib, field as F
from jolt_b200.api import UnivariatePoly
from oracle import bn254 as O

ROOT = pathlib.Path(__file__).resolve().parents[1]


def _has_gpu():
    return _lib.load().jb_device_count() > 0


def test_header_symbols_exported():
    header = (ROOT / "include" / "jolt_b200.h").read_text()
    declared = set(re.findall(r"\b(jb_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 35
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/jolt_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)


def test_version_and_status_strings():
    lib = _lib.load()
    assert b"sm_90a" in lib.jb_version()
    assert b"no CPU fallback" in lib.jb_status_str(_lib.JB_ERR_NO_DEVICE)


def test_no_device_fails_loudly():
    if _has_gpu():
        pytest.skip("a CUDA device is present")
    with pytest.raises(jolt_b200.JoltB200Error) as e:
        jolt_b200.Session(0)
    assert e.value.status == _lib.JB_ERR_NO_DEVICE


def test_field_helpers_match_oracle():
    vals = O.random_fr(7, 20) + [0, 1, O.R_MOD - 1]
    limbs = F.ints_to_limbs(vals)
    assert [list(map(int, row)) for row in limbs] == [O.to_mont_limbs(v) for v in vals]
    assert F.limbs_to_ints(limbs) == vals
    assert list(F.challenge_from_bytes(bytes.fromhex("dae623d2aa29f41845b9a32a1d819bb6"))) == \
        O.challenge_to_mont_limbs(*O.challenge_limbs(bytes.fromhex("dae623d2aa29f41845b9a32a1d819bb6")))


@pytest.mark.parametrize("deg", [1, 2, 3, 4, 7])
def test_univariate_from_evals_matches_oracle(deg):
    coeffs = O.random_fr(100 + deg, deg + 1)
    ev = [O.uni_evaluate(coeffs, x) for x in range(deg + 1)]
    poly = UnivariatePoly.from_evals(ev)
    assert poly.coefficients == coeffs == O.uni_from_evals(ev)
    x = O.random_fr(5, 1)[0]
    assert poly.evaluate(x) == O.uni_evaluate(coeffs, x)
    assert poly.compress() == O.uni_compress(coeffs)
    hint = (ev[0] + ev[1]) % O.R_MOD
    assert UnivariatePoly.from_evals_and_hint(hint, [ev[0]] + ev[2:]).coefficients == coeffs


class _OracleMember:
    """host-only stand-in so the engine (host logic) can be tested without a GPU"""
    def __init__(self, tables):
        self.inner = O.ProductMember(tables)
    def num_rounds(self):
        return self.inner.num_rounds()
    def prove_round(self, b, rnd, claim):
        return UnivariatePoly(self.inner.prove_round(b, rnd, claim))
    def finish_rounds(self, b):
        self.inner.finish_rounds(b)


def test_engine_host_logic_matches_oracle_engine():
    # two members of different lengths (front-loaded padding, prover.rs:246-280)
    t_a = [O.random_fr(1, 16), O.random_fr(2, 16)]
    t_b = [O.dense_member_with_sum(2, 555, 41)]
    claim_a = sum(x * y for x, y in zip(*t_a)) % O.R_MOD
    desc = [dict(input_claim=claim_a, coefficient=3, rounds=4, offset=0),
            dict(input_claim=555, coefficient=5, rounds=2, offset=2)]
    total = (3 * claim_a + 5 * 555 * 4) % O.R_MOD
    pts = O.synthetic_point(4, 401)
    want = O.prove_batch(desc, [O.ProductMember(t_a), O.ProductMember(t_b)], 4, 2, total, lambda r, c: pts[r])
    got = jolt_b200.prove_batch([jolt_b200.BatchMember(**d) for d in desc], [_OracleMember(t_a), _OracleMember(t_b)],
                                4, 2, total, lambda r, poly: pts[r])
    assert got.challenges == want["challenges"] and got.final_claim == want["final_claim"]
    assert got.member_claims == want["member_claims"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    with pytest.raises(jolt_b200.SumcheckError):
        jolt_b200.prove_batch([jolt_b200.BatchMember(**desc[0])], [_OracleMember(t_a)], 4, 2, total + 1, lambda r, p: 1)


def test_small_scalar_encoding_host_side():
    """jb_scalar_kind byte layouts (include/jolt_b200.h): dtype -> kind, 128-bit values as 16 LE bytes."""
    import numpy as np
    from jolt_b200 import SCALAR_KINDS, small_scalars

    a, k, n = small_scalars(np.array([1, 0, 1], dtype=np.bool_))
    assert (k, n, a.dtype) == (SCALAR_KINDS["u8"], 3, np.uint8)
    a, k, n = small_scalars(np.array([-1, 2], dtype=np.int64))
    assert (k, n) == (SCALAR_KINDS["i64"], 2) and a.tobytes() == (-1).to_bytes(8, "little", signed=True) + (2).to_bytes(8, "little")
    a, k, n = small_scalars([-(1 << 127), -1, (1 << 127) - 1], "i128")
    assert k == SCALAR_KINDS["i128"]
    assert a.tobytes() == b"".join(v.to_bytes(16, "little", signed=True) for v in (-(1 << 127), -1, (1 << 127) - 1))
    a, k, n = small_scalars([(1 << 128) - 1, 5], "u128")
    assert a.tobytes() == ((1 << 128) - 1).to_bytes(16, "little") + (5).to_bytes(16, "little")
    with pytest.raises(ValueError):
        small_scalars([1 << 128], "u128")
    with pytest.raises(ValueError):
        small_scalars(np.zeros(2, dtype=np.float64))


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("skip1", [0, 1])
def test_round_evals_from_kernel_values(m, skip1):
    """The host half of jb_member_prove_round (no device): s(1) from the claim, s(m) from the leading coefficient
    s(inf) the kernels emit instead of s(m) - checked against direct evaluation of random degree-m polynomials."""
    import ctypes
    import numpy as np
    from jolt_b200 import field as F
    from jolt_b200._lib import JB_OK
    from jolt_b200.api import _p
    lib = jolt_b200.load()
    for seed in range(5):
        coeffs = O.random_fr(100 * m + 10 * skip1 + seed, m + 1)
        s = [O.uni_evaluate(coeffs, t) for t in range(m + 1)]
        claim = (s[0] + s[1]) % O.R_MOD
        vals = [s[0]] + ([] if skip1 else [s[1]])
        if m >= 2:
            vals += s[2:m] + [coeffs[m]]                    # s(2..m-1), then the leading coefficient
        vin = F.ints_to_limbs(vals)
        out = np.zeros((m + 1, 4), dtype=np.uint64)
        cl = F.ints_to_limbs([claim])
        assert lib.jb_round_evals_from_kernel_values(m, skip1, _p(vin), _p(cl), _p(out)) == JB_OK
        assert F.limbs_to_ints(out) == s
        if not skip1:   # verify mode: a wrong claim is a round-check failure; no claim, no check
            bad = F.ints_to_limbs([(claim + 1) % O.R_MOD])
            assert lib.jb_round_evals_from_kernel_values(m, 0, _p(vin), _p(bad), _p(out)) == jolt_b200._lib.JB_ERR_ROUND_CHECK
            assert lib.jb_round_evals_from_kernel_values(m, 0, _p(vin), None, _p(out)) == JB_OK
    assert lib.jb_round_evals_from_kernel_values(5, 0, _p(vin), None, _p(out)) == jolt_b200._lib.JB_ERR_INVALID


def test_wide_lanes_reduce_host_matches_big_int():
    """jb_wide_lanes_reduce_host (the host tail of a resident-kernel round): 17 u64 lanes of 32-bit limb column sums
    -> (sum) * R^-1 mod r, against Python integers; includes the all-ones extreme and real sums of products."""
    lib = _lib.load()
    rng = np.random.Generator(np.random.PCG64(11))
    rows = [rng.integers(0, 1 << 63, size=17, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=17, dtype=np.uint64)
            for _ in range(6)]
    rows.append(np.full(17, (1 << 64) - 1, dtype=np.uint64))
    rows.append(np.zeros(17, dtype=np.uint64))
    # genuine accumulators: sum of 1000 products of Montgomery-form operands, limb columns summed separately
    a = [O.mont_raw(O.to_mont_limbs(v)) for v in O.random_fr(1, 1000)]
    b = [O.mont_raw(O.to_mont_limbs(v)) for v in O.random_fr(2, 1000)]
    cols = [0] * 17
    for x, y in zip(a, b):
        pr = x * y
        for w in range(16):
            cols[w] += (pr >> (32 * w)) & 0xFFFFFFFF
    rows.append(np.array(cols, dtype=np.uint64))
    lanes = np.ascontiguousarray(np.stack(rows))
    out = np.zeros((len(rows), 4), dtype=np.uint64)
    assert lib.jb_wide_lanes_reduce_host(lanes.ctypes.data_as(_lib.c_u64p), len(rows), out.ctypes.data_as(_lib.c_u64p)) == 0
    rinv = pow(1 << 256, -1, O.R_MOD)
    for row, got in zip(rows, out):
        v = sum(int(x) << (32 * w) for w, x in enumerate(row))
        assert O.mont_raw([int(t) for t in got]) == v * rinv % O.R_MOD
    # the last row is sum a_i b_i in Montgomery form: (sum aR bR) R^-1 = (sum a b) R
    want = sum(x * y for x, y in zip(O.random_fr(1, 1000), O.random_fr(2, 1000))) % O.R_MOD
    assert O.from_mont_limbs([int(t) for t in out[-1]]) == want
