"""The resident kernel service (one launch per batch, rounds driven through a mailbox), the sum-of-products member
(IncClaimReduction's shape) and the device RoundScheduler against the oracle and against the one-launch-per-round
path. Mirrors crates/jolt-kernels/src/optimized/parity.rs:79-118 (run_lockstep) and
crates/jolt-kernels/src/optimized/inc_claim_reduction.rs:210-300 (inc_claim_reduction_matches_reference)."""
import os

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, Polynomial, ProductMember, RoundScheduler,
                       SumOfProductsMember, UnivariatePoly)
from jolt_b200 import field as F
from oracle import bn254 as O
from oracle import coracle as C
from gpu_util import rand_challenge, rand_full, rand_limbs
from sumcheck_ref import rand_limbs_full

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sess_launch():
    """a context with the resident service off: one kernel launch per round all the way down"""
    os.environ["JB_NO_TAIL"] = "1"
    try:
        s = jolt_b200.Session(0)
    finally:
        del os.environ["JB_NO_TAIL"]
    yield s
    s.close()


def full_sumcheck(sess, tabs_limbs, order, seed, member_cls=ProductMember, **kw):
    polys = [Polynomial.new(sess, t) for t in tabs_limbs]
    mem = member_cls(sess, polys, order=order, **kw) if kw else member_cls(sess, polys, order)
    n = mem.num_rounds()
    probe_polys = [Polynomial.new(sess, t) for t in tabs_limbs]
    probe = member_cls(sess, probe_polys, order=order, **kw) if kw else member_cls(sess, probe_polys, order)
    ev = probe.prove_round_evals(None, 0)
    probe.close()
    claim = (ev[0] + ev[1]) % F.R_MOD
    res = jolt_b200.prove_batch_native([BatchMember(claim, 1, n, 0)], [mem], n, mem.degree(), claim, seed=seed)
    fe = mem.final_evals()
    mem.close()
    return claim, res, fe


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_resident_equals_launch_per_round(sess, sess_launch, m, order):
    """2^18 entries: the resident kernel runs with hundreds of live blocks, shrinking to one; every round polynomial,
    challenge and final evaluation must equal the one-launch-per-round path bit for bit."""
    n = 18
    tabs = [rand_limbs(0xE500 + 16 * m + j, 1 << n) for j in range(m)]
    l0 = sess.launch_count
    a = full_sumcheck(sess, tabs, order, 5)
    resident_launches = sess.launch_count - l0
    l0 = sess_launch.launch_count
    b = full_sumcheck(sess_launch, tabs, order, 5)
    per_round_launches = sess_launch.launch_count - l0
    assert a[0] == b[0] and a[2] == b[2]
    assert a[1].challenges == b[1].challenges and a[1].final_claim == b[1].final_claim
    assert [p.coefficients for p in a[1].round_polynomials] == [p.coefficients for p in b[1].round_polynomials]
    assert np.prod(a[2], dtype=object) % O.R_MOD == a[1].final_claim
    # the probe's eval pass + ONE resident kernel, against one launch per round
    assert resident_launches <= 3 and per_round_launches >= n


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_resident_2pow16_vs_c_oracle_every_round(sess, order):
    """BASELINE config 1 through the resident kernel: every round polynomial vs the 1-thread C oracle, mixing
    125-bit and 254-bit challenges (both bind products are selected inside the kernel from the mailbox line)."""
    n, m = 16, 2
    tabs = [rand_limbs(0xB200 + j, 1 << n) for j in range(m)]
    gpu = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], order)
    cur = [t.copy() for t in tabs]
    bind = None
    l0 = sess.launch_count
    for rnd in range(n):
        if bind is not None:
            cur = [C.bind(t, bind, order) for t in cur]
        want = C.mont_to_ints(C.product_round_evals(cur, m, order))
        got = gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % O.R_MOD)
        assert got == want, f"round {rnd}"
        bind = rand_challenge(3000 + rnd) if rnd % 2 else rand_full(3000 + rnd)
    cur = [C.bind(t, bind, order) for t in cur]
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == [C.mont_to_ints(t)[0] for t in cur]
    assert sess.launch_count - l0 == 1      # the whole sumcheck was ONE kernel launch


@pytest.mark.parametrize("m", [1, 3, 4])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_resident_2pow18_vs_c_oracle_every_round(sess, m, order):
    """products of 1, 3 and 4 tables at 2^18 (multi-block passes shrinking to one block) through the resident
    kernel, every round and the final evaluations against the threaded C oracle, inputs over all of [0, p)."""
    n = 18
    thr = C.max_threads()
    tabs = [rand_limbs_full(0xB218 + 8 * m + j, 1 << n) for j in range(m)]
    gpu = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], order)
    cur = tabs
    bind = None
    l0 = sess.launch_count
    for rnd in range(n):
        if bind is not None:
            cur = [C.bind(t, bind, order, thr) for t in cur]
        want = C.mont_to_ints(C.product_round_evals(cur, m, order, thr))
        got = gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % O.R_MOD)
        assert got == want, f"round {rnd}"
        bind = rand_challenge(6000 + rnd) if rnd % 2 else rand_limbs_full(6000 + rnd, 1)[0]
    cur = [C.bind(t, bind, order, thr) for t in cur]
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == [C.mont_to_ints(t)[0] for t in cur]
    assert sess.launch_count - l0 == 1      # the whole sumcheck was ONE kernel launch


def test_resident_run_survives_interleaved_context_work(sess):
    """Any other entry point that needs the device while an exclusive run is alive stops the run at a round
    boundary; the member continues with launches and the proof is unchanged."""
    n = 17
    tabs = [rand_limbs(0xA100 + j, 1 << n) for j in range(2)]
    ch = [rand_challenge(70 + i) for i in range(n)]

    def prove(interleave):
        gpu = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], LOW_TO_HIGH)
        ev = None
        out, bind, claim = [], None, None
        for rnd in range(n):
            if claim is None:
                probe = ProductMember(sess, [Polynomial.new(sess, t) for t in tabs], LOW_TO_HIGH)
                e = probe.prove_round_evals(None, 0)
                probe.close()
                claim = (e[0] + e[1]) % F.R_MOD
            ev = gpu.prove_round_evals(bind, rnd, claim)
            out.append(ev)
            if interleave and rnd in (2, 9):
                # an eq table build launches kernels on the context's stream and waits for them
                r = F.ints_to_limbs(O.random_fr(rnd, 12))
                assert jolt_b200.EqPolynomial.evals(sess, r).to_ints() == O.eq_evals(O.random_fr(rnd, 12))
            bind = ch[rnd]
            claim = UnivariatePoly.from_evals(ev).evaluate(F.from_limbs(bind))
        gpu.finish_rounds(bind)
        return out, gpu.final_evals()

    assert prove(False) == prove(True)


def test_lost_resident_kernel_is_recovered_with_launches(sess):
    """ADVICE r01: a resident kernel that stops waiting for commands (the host was held up - here a 3 ms device
    timeout and a host that sleeps) must not fail the member: the unexecuted binds are replayed with launches, the
    round is recomputed, and the proof is the oracle's, both in thin (lookahead) and in generic rounds, and in a
    scheduler batch whose short members run on their own small kernels."""
    import time
    os.environ["JB_RESIDENT_TIMEOUT_S"] = "0.003"
    try:
        s2 = jolt_b200.Session(0)
    finally:
        del os.environ["JB_RESIDENT_TIMEOUT_S"]
    for n, order, naps in ((9, LOW_TO_HIGH, (2, 5)), (9, HIGH_TO_LOW, (1, 2, 7)), (18, LOW_TO_HIGH, (1, 9, 16))):
        tabs = [rand_limbs(0x7E57 + j, 1 << n) for j in range(2)]
        gpu = ProductMember(s2, [Polynomial.new(s2, t) for t in tabs], order)
        cur = [t.copy() for t in tabs]
        bind, thr = None, C.max_threads()
        for rnd in range(n):
            if bind is not None:
                cur = [C.bind(t, bind, order, thr) for t in cur]
            want = C.mont_to_ints(C.product_round_evals(cur, 2, order, thr))
            if rnd in naps:
                time.sleep(0.05)      # far beyond the kernel's patience: it exits, possibly with commands in flight
            got = gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % O.R_MOD)
            assert got == want, f"n={n} round {rnd}"
            bind = rand_challenge(4000 + rnd)
        cur = [C.bind(t, bind, order, thr) for t in cur]
        time.sleep(0.05)
        gpu.finish_rounds(bind)
        assert gpu.final_evals() == [C.mont_to_ints(t)[0] for t in cur]
        gpu.close()
    # a batch of two shapes (not one resident kernel): each member is on its own small run once it is short, and the
    # host sleeps between rounds
    shapes = [(3, 14, 0), (2, 9, 5)]
    tabs, desc, total, max_vars = batch_fixture(shapes, 4100)
    pts = O.synthetic_point(max_vars, 403)
    want = O.prove_batch(desc, [O.ProductMember(t, LOW_TO_HIGH) for t in tabs], max_vars, 3, total, lambda r, c: pts[r])
    mems = [ProductMember(s2, [Polynomial.from_ints(s2, t) for t in tb], LOW_TO_HIGH) for tb in tabs]

    def draw(r, poly):
        if r in (2, 6, 10, 13):
            time.sleep(0.05)
        return pts[r]

    got = jolt_b200.prove_batch_native([BatchMember(**d) for d in desc], mems, max_vars, 3, total, draw)
    assert got.challenges == want["challenges"] and got.final_claim == want["final_claim"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for mem, tb, d in zip(mems, tabs, desc):
        assert mem.final_evals() == [O.evaluate(t, list(reversed(pts[d["offset"]:d["offset"] + d["rounds"]]))) for t in tb]
        mem.close()
    s2.close()


# ---- sum of products: IncClaimReduction -------------------------------------------------------------------
def inc_fixture(n, seed):
    pts = [O.synthetic_point(n, s) for s in (3, 5, 7, 11)]          # inc_claim_reduction.rs:236-241
    gamma = 29                                                       # :243-245
    ram_inc = O.random_fr(seed, 1 << n)
    rd_inc = O.random_fr(seed + 1, 1 << n)
    return pts, gamma, ram_inc, rd_inc


@pytest.mark.parametrize("n", [1, 2, 5, 10])
def test_inc_claim_reduction_lockstep(sess, n):
    """run_lockstep (parity.rs:79-118) of the device sum-of-products member against the oracle restatement of the
    optimized IncClaimReduction kernel: byte-equal round polynomials, equal output claims."""
    pts, gamma, ram_inc, rd_inc = inc_fixture(n, 77)
    ref = O.IncClaimReductionKernel(pts, gamma, ram_inc, rd_inc)
    tabs = ref.tables()
    gpu = SumOfProductsMember(sess, [Polynomial.from_ints(sess, t) for t in tabs], 2, 2, LOW_TO_HIGH)
    assert gpu.num_rounds() == n and gpu.degree() == 2
    claim = sum(a * x + b * y for a, x, b, y in zip(*tabs)) % O.R_MOD
    assert claim != 0
    ch = O.synthetic_point(n, 401)
    bind = None
    for rnd in range(n):
        want = ref.prove_round(bind, rnd, claim)
        got = gpu.prove_round(bind, rnd, claim)
        assert got.coefficients == want, f"round {rnd}"
        bind = ch[rnd]
        claim = got.evaluate(bind)
    ref.finish_rounds(bind)
    gpu.finish_rounds(bind)
    fe = gpu.final_evals()
    assert fe == ref.final_evals()
    assert {"ram_inc": fe[1], "rd_inc": fe[3]} == ref.output_claims()
    assert (fe[0] * fe[1] + fe[2] * fe[3]) % O.R_MOD == claim


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_sum_of_products_all_modes_agree(sess, sess_launch, order):
    """resident (hint), launched with every point computed (verify), launched without a claim: identical evaluations."""
    n = 12
    tabs = [O.random_fr(300 + j, 1 << n) for j in range(4)]
    ch = O.random_fr(6, n)
    outs = []
    for s, mode in ((sess, "hint"), (sess, "verify"), (sess_launch, "hint"), (sess_launch, "noclaim")):
        s.set_verify_rounds(mode == "verify")
        gpu = SumOfProductsMember(s, [Polynomial.from_ints(s, t) for t in tabs], 2, 2, order)
        claim = sum(a * x + b * y for a, x, b, y in zip(*tabs)) % O.R_MOD
        bind, seq = None, []
        for rnd in range(n):
            ev = gpu.prove_round_evals(bind, rnd, None if mode == "noclaim" else claim)
            seq.append(ev)
            bind = ch[rnd]
            claim = UnivariatePoly.from_evals(ev).evaluate(bind)
        gpu.finish_rounds(bind)
        seq.append(gpu.final_evals())
        s.set_verify_rounds(False)
        outs.append(seq)
    assert outs[0] == outs[1] == outs[2] == outs[3]
    # t = 0..2 against the plain definition on the unbound tables
    half = 1 << (n - 1)
    pr = (lambda t, y: (t[y], t[y + half])) if order == HIGH_TO_LOW else (lambda t, y: (t[2 * y], t[2 * y + 1]))
    want = []
    for t in range(3):
        acc = 0
        for y in range(half):
            v = [lo + t * (hi - lo) for lo, hi in (pr(tb, y) for tb in tabs)]
            acc += v[0] * v[1] + v[2] * v[3]
        want.append(acc % O.R_MOD)
    assert outs[0][0] == want


# ---- device RoundScheduler ------------------------------------------------------------------------------
def batch_fixture(shapes, seed):
    """shapes: [(m, log_len, offset)] -> tables, descriptors, the honest combined claim"""
    tabs = [[O.random_fr(seed + 10 * i + j, 1 << ln) for j in range(m)] for i, (m, ln, off) in enumerate(shapes)]
    max_vars = max(ln + off for _, ln, off in shapes)
    desc, total = [], 0
    for i, (m, ln, off) in enumerate(shapes):
        claim = sum(int(np.prod([t[x] for t in tabs[i]], dtype=object)) for x in range(1 << ln)) % O.R_MOD
        coeff = O.random_fr(seed + 100 + i, 1)[0]
        desc.append(dict(input_claim=claim, coefficient=coeff, rounds=ln, offset=off))
        total = (total + coeff * claim * pow(2, max_vars - ln, O.R_MOD)) % O.R_MOD
    return tabs, desc, total, max_vars


@pytest.mark.parametrize("shapes", [
    [(2, 10, 0), (2, 10, 0), (2, 10, 0)],                    # homogeneous, aligned: one resident kernel
    [(2, 12, 0), (2, 7, 5), (2, 9, 3), (2, 3, 9)],           # homogeneous shape, different lengths / windows
    [(2, 10, 0), (3, 8, 2), (1, 10, 0)],                    # heterogeneous: overlapped launches + small runs
    [(3, 15, 0), (2, 15, 0)],                                # heterogeneous, big passes
])
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_scheduler_batches_match_oracle_engine(sess, shapes, order):
    tabs, desc, total, max_vars = batch_fixture(shapes, 4000)
    max_deg = max(m for m, _, _ in shapes)
    pts = O.synthetic_point(max_vars, 401)
    want = O.prove_batch(desc, [O.ProductMember(t, order) for t in tabs], max_vars, max_deg, total, lambda r, c: pts[r])
    mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], order) for tb in tabs]
    l0 = sess.launch_count
    got = jolt_b200.prove_batch_native([BatchMember(**d) for d in desc], mems, max_vars, max_deg, total,
                                       lambda r, poly: pts[r])
    launches = sess.launch_count - l0
    assert got.challenges == want["challenges"] and got.final_claim == want["final_claim"]
    assert got.member_claims == want["member_claims"]
    assert [p.coefficients for p in got.round_polynomials] == want["round_polys"]
    for mem, tb, d in zip(mems, tabs, desc):
        window = pts[d["offset"]:d["offset"] + d["rounds"]]
        point = window if order == HIGH_TO_LOW else list(reversed(window))
        assert mem.final_evals() == [O.evaluate(t, point) for t in tb]
    if len({m for m, _, _ in shapes}) == 1:
        assert launches == 1, launches     # the whole batch was ONE kernel launch


def test_scheduler_direct_api_and_sequential_agree(sess):
    """jb_scheduler_* driven directly (RoundScheduler::batch_prove_round) == jb_member_prove_round member by member."""
    n = 11
    tabs = [[O.random_fr(9000 + 10 * i + j, 1 << n) for j in range(2)] for i in range(4)]
    ch = O.synthetic_point(n, 17)

    def claims0():
        return [sum(a * b for a, b in zip(*tb)) % O.R_MOD for tb in tabs]

    # sequential
    mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], LOW_TO_HIGH) for tb in tabs]
    claims, seq = claims0(), []
    for rnd in range(n):
        polys = [m.prove_round(None if rnd == 0 else ch[rnd - 1], rnd, c) for m, c in zip(mems, claims)]
        seq.append([p.coefficients for p in polys])
        claims = [p.evaluate(ch[rnd]) for p in polys]
    for m in mems:
        m.finish_rounds(ch[-1])
    seq_final = [m.final_evals() for m in mems]
    # scheduler
    mems = [ProductMember(sess, [Polynomial.from_ints(sess, t) for t in tb], LOW_TO_HIGH) for tb in tabs]
    sched = RoundScheduler(sess, mems)
    claims, got = claims0(), []
    l0 = sess.launch_count
    for rnd in range(n):
        polys = sched.batch_prove_round([(i, rnd, None if rnd == 0 else ch[rnd - 1], claims[i]) for i in range(4)])
        got.append([p.coefficients for p in polys])
        claims = [p.evaluate(ch[rnd]) for p in polys]
    sched.batch_finish_rounds([(i, ch[-1]) for i in range(4)])
    assert sess.launch_count - l0 == 1
    assert got == seq and [m.final_evals() for m in mems] == seq_final
    sched.close()
