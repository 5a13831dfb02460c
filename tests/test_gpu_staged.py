"""The resident kernel's staged large passes (tables brought into shared memory by bulk copies) against the pass that
loads every element itself (JB_RES_STAGED=0) and against one launch per round: a batch of two degree-2 members large
enough for two staged rounds each, both binding orders, full 254-bit and 125-bit challenges, inputs over all of [0, p)."""
import os

import pytest

import jolt_b200
from jolt_b200 import HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, Polynomial, ProductMember
from jolt_b200 import field as F
from gpu_util import rand_challenge
from sumcheck_ref import rand_limbs_full

pytestmark = pytest.mark.gpu


def _session(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return jolt_b200.Session(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def sessions():
    ss = {"staged": _session(JB_RES_STAGED="1"), "unstaged": _session(JB_RES_STAGED="0"), "launch": _session(JB_NO_TAIL="1")}
    yield ss
    for s in ss.values():
        s.close()


def absorb(rnd, poly):
    # a deterministic stand-in transcript that alternates full scalars and 125-bit challenges
    return F.from_limbs(rand_challenge(700 + rnd)) if rnd % 2 else (0x5EED_0000 + rnd) * 0x9E3779B97F4A7C15F39CC0605CEDC835 % F.R_MOD


def batch(sess, tabs, order):
    n = len(tabs[0][0]).bit_length() - 1
    mems, desc, total = [], [], 0
    for k, pair in enumerate(tabs):
        probe = ProductMember(sess, [Polynomial.new(sess, t) for t in pair], order)
        ev = probe.prove_round_evals(None, 0)
        probe.close()
        claim = (ev[0] + ev[1]) % F.R_MOD
        mems.append(ProductMember(sess, [Polynomial.new(sess, t) for t in pair], order))
        desc.append(BatchMember(claim, 1 + k, n, 0))
        total = (total + (1 + k) * claim) % F.R_MOD
    res = jolt_b200.prove_batch_native(desc, mems, n, 2, total, absorb_round=absorb)
    fe = [m.final_evals() for m in mems]
    for m in mems:
        m.close()
    return res, fe


@pytest.mark.parametrize("order", [LOW_TO_HIGH, HIGH_TO_LOW], ids=["L2H", "H2L"])
def test_staged_passes_equal_unstaged_and_launch_per_round(sessions, order):
    n = 20  # rounds 0 (eval over 2^19 pairs) and 1 (bind + eval over 2^18 pairs) are staged
    tabs = [[rand_limbs_full(0x57A6 + 8 * k + j, 1 << n) for j in range(2)] for k in range(2)]
    out = {name: batch(s, tabs, order) for name, s in sessions.items()}
    ref_res, ref_fe = out["launch"]
    for name in ("staged", "unstaged"):
        res, fe = out[name]
        assert res.challenges == ref_res.challenges, name
        assert [p.coefficients for p in res.round_polynomials] == [p.coefficients for p in ref_res.round_polynomials], name
        assert res.final_claim == ref_res.final_claim and res.member_claims == ref_res.member_claims, name
        assert fe == ref_fe, name
