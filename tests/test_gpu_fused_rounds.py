"""Folded large rounds of the resident kernel's staged runs (degree-2 products): the first pass over large tables
returns lookahead sums, the round after it is answered from them without a device pass, and the next pass binds both
challenges in one read of the tables. Every round polynomial and the final evaluations must be the C oracle's and
those of the same session type with folding off (JB_RES_FUSE=0) and with one launch per round (JB_NO_TAIL=1), bit
for bit, including every way a run can end while a challenge is pending on the host."""
import os
import time

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, Polynomial, ProductMember, UnivariatePoly
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
from gpu_util import rand_challenge, rand_limbs
from sumcheck_ref import extreme_table, rand_limbs_full

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
    s = {"fused": _session(), "unfused": _session(JB_RES_FUSE="0"), "launch": _session(JB_NO_TAIL="1")}
    yield s
    for x in s.values():
        x.close()


def challenge(rnd, phase):
    """125-bit and full 254-bit challenges alternate; `phase` picks which comes first, so a double bind meets both
    (full, 125-bit) and (125-bit, full)"""
    return rand_challenge(5000 + rnd) if (rnd + phase) % 2 else rand_limbs_full(5000 + rnd, 1)[0]


def oracle_run(sess, tabs, order, phase):
    """every round against the C oracle, then the terminal bind and the final evaluations"""
    thr = C.max_threads()
    n = int(np.log2(tabs[0].shape[0]))
    gpu = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], order)
    cur, bind, got_all = tabs, None, []
    for rnd in range(n):
        if bind is not None:
            cur = [C.bind(t, bind, order, thr) for t in cur]
        want = C.mont_to_ints(C.product_round_evals(cur, 2, order, thr))
        got = gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % O.R_MOD)
        assert got == want, f"n={n} round {rnd}"
        got_all.append(got)
        bind = challenge(rnd, phase)
    cur = [C.bind(t, bind, order, thr) for t in cur]
    gpu.finish_rounds(bind)
    fe = gpu.final_evals()
    assert fe == [C.mont_to_ints(t)[0] for t in cur]
    gpu.close()
    return got_all, fe


@pytest.mark.parametrize("n", [2, 3, 9, 17, 18, 19, 20, 21, 22])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_fused_rounds_vs_c_oracle_every_round(sessions, n, order):
    tabs = [rand_limbs_full(0xF05E + 16 * n + j, 1 << n) for j in range(2)]
    a = oracle_run(sessions["fused"], tabs, order, n % 2)
    if n >= 19:
        assert a == oracle_run(sessions["unfused"], tabs, order, n % 2)


@pytest.mark.parametrize("phase", [0, 1])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_fused_rounds_limb_extremes(sessions, phase, order):
    """tables that hold every ordered pair of limb-extreme values, at 2^20 (two double binds) and 2^21 (one)"""
    for n in (20, 21):
        tabs = [extreme_table(0xE7 + j, n, order, rotate=j) for j in range(2)]
        oracle_run(sessions["fused"], tabs, order, phase)


def _batch(sess, tabs, order, rounds, offsets, seed):
    mems = [ProductMember(sess, [Polynomial.new(sess, t) for t in tb], order) for tb in tabs]
    max_vars = max(r + o for r, o in zip(rounds, offsets))
    claims = []
    for tb in tabs:
        probe = ProductMember(sess, [Polynomial.new(sess, t) for t in tb], order)
        ev = probe.prove_round_evals(None, 0)
        probe.close()
        claims.append((ev[0] + ev[1]) % F.R_MOD)
    desc = [BatchMember(c, 1, r, o) for c, r, o in zip(claims, rounds, offsets)]
    total = sum(c * pow(2, max_vars - r, F.R_MOD) for c, r in zip(claims, rounds)) % F.R_MOD
    res = jolt_b200.prove_batch_native(desc, mems, max_vars, 2, total, seed=seed)
    fe = [m.final_evals() for m in mems]
    for m in mems:
        m.close()
    return res.challenges, res.final_claim, [p.coefficients for p in res.round_polynomials], fe


@pytest.mark.parametrize("shape", [
    ([22], [0]),                         # bench.py's workload
    ([20] * 2, [0, 0]),                  # homogeneous batch of 2: one command per batch round
    ([19] * 8, [0] * 8),                 # homogeneous batch of 8
    ([21, 20, 20], [0, 1, 0]),           # ragged: members in different states share the run
])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_fused_batches_equal_unfused_and_launched(sessions, shape, order):
    rounds, offsets = shape
    tabs = [[rand_limbs(0xBA7C + 8 * i + j, 1 << r) for j in range(2)] for i, r in enumerate(rounds)]
    got = {k: _batch(s, tabs, order, rounds, offsets, 11) for k, s in sessions.items()}
    assert got["fused"] == got["unfused"] == got["launch"]


def _manual(sess, tabs, order, hook=None, finish_after=None):
    """rounds through jb_member_prove_round; hook(rnd) runs after round rnd; finish_after: stop proving after that
    round and bind every remaining variable with finish_rounds"""
    n = int(np.log2(tabs[0].shape[0]))
    gpu = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], order)
    probe = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], order)
    e = probe.prove_round_evals(None, 0)
    probe.close()
    claim, bind, out = (e[0] + e[1]) % F.R_MOD, None, []
    for rnd in range(n):
        ev = gpu.prove_round_evals(bind, rnd, claim)
        out.append(ev)
        if hook:
            hook(rnd)
        bind = challenge(rnd, 0)
        claim = UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
        if finish_after == rnd:
            for k in range(rnd, n):
                gpu.finish_rounds(challenge(k, 0))
            break
    else:
        gpu.finish_rounds(bind)
    fe = gpu.final_evals()
    gpu.close()
    return out, fe


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_run_stopped_right_after_a_skipped_round(sessions, order):
    """other context work that needs the device right after a round answered from lookahead (rounds 1 and 3 at
    2^21): the run ends, its pending challenge is bound by launches, the member continues and the proof is unchanged"""
    sess = sessions["fused"]
    tabs = [rand_limbs(0x5707 + j, 1 << 21) for j in range(2)]

    def interleave(rnd):
        if rnd in (1, 3):
            r = F.ints_to_limbs(O.random_fr(rnd, 12))
            assert jolt_b200.EqPolynomial.evals(sess, r).to_ints() == O.eq_evals(O.random_fr(rnd, 12))

    assert _manual(sess, tabs, order) == _manual(sess, tabs, order, interleave) == _manual(sessions["launch"], tabs, order)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_finish_rounds_right_after_a_skipped_round(sessions, order):
    """finish_rounds right after round 1 (answered from lookahead, its challenge pending) binds the pending challenge
    first: binding every remaining variable that way ends at the oracle's final evaluations"""
    n = 20
    tabs = [rand_limbs(0xF1 + j, 1 << n) for j in range(2)]
    got = _manual(sessions["fused"], tabs, order, finish_after=1)
    assert got == _manual(sessions["launch"], tabs, order, finish_after=1)
    cur = tabs
    for k in range(n):
        cur = [C.bind(t, challenge(k, 0), order, C.max_threads()) for t in cur]
    assert got[1] == [C.mont_to_ints(t)[0] for t in cur]


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_lost_kernel_with_a_pending_challenge_is_recovered(sessions, order):
    """a resident kernel that stops waiting for commands (3 ms patience, a host that sleeps) while a challenge is
    pending on the host - after a skipped round, before the double bind that carries it - or with a double bind in
    flight: the run's binds are replayed with launches and every round is still the oracle's"""
    s2 = _session(JB_RESIDENT_TIMEOUT_S="0.003")
    n = 21
    thr = C.max_threads()
    tabs = [rand_limbs(0x7E58 + j, 1 << n) for j in range(2)]
    gpu = ProductMember(s2, [Polynomial.new(s2, t) for t in tabs], order)
    cur, bind = tabs, None
    for rnd in range(n):
        if bind is not None:
            cur = [C.bind(t, bind, order, thr) for t in cur]
        want = C.mont_to_ints(C.product_round_evals(cur, 2, order, thr))
        if rnd in (1, 2, 5):
            time.sleep(0.05)
        got = gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % O.R_MOD)
        assert got == want, f"round {rnd}"
        bind = challenge(rnd, 1)
    cur = [C.bind(t, bind, order, thr) for t in cur]
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == [C.mont_to_ints(t)[0] for t in cur]
    gpu.close()
    s2.close()


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_fused_run_posts_fewer_commands_than_rounds(sessions, order):
    """at 2^22 rounds 1 and 3 carry no command: the run log of the last run shows 21 commands for 22 rounds plus
    the terminal bind (with folding off: 23)"""
    import ctypes
    from jolt_b200.api import _p
    tabs = [rand_limbs(0xC0DE + j, 1 << 22) for j in range(2)]
    counts = {}
    for k in ("fused", "unfused"):
        sess = sessions[k]
        _manual(sess, tabs, order)
        log = np.zeros((64, 8), dtype=np.uint64)
        cnt = ctypes.c_size_t()
        sess.check(sess.lib.jb_ctx_run_log(sess.h, _p(log), 64, ctypes.byref(cnt)))
        counts[k] = cnt.value
    assert counts == {"fused": 21, "unfused": 23}
