"""Stream ordering of the device memory the library reads in place and writes for the caller, and concurrent calls.

Every check runs under three session modes: "private" (Session(0): the library's own non-blocking stream), "legacy"
(the session on torch's current stream, the legacy default stream 0) and "side" (a torch.cuda.Stream made current and
the session created on it, as bench.py runs).

Inputs: each device input is produced on torch's current stream by a device kernel queued behind a delay kernel
(torch.cuda._sleep), over a buffer pre-filled with a sentinel that changes the answer if it is read instead of the
data (zeros for field tables, the none value for one-hot columns, another constant for compact columns). The producer
must still be running when the library is called (asserted with an event), so a result equal to the big-int or C
reference shows that the library's read was ordered after the producer. Outputs: the library's stream is held busy by
a delay kernel before it writes, and torch reads the result on its current stream with no session synchronisation.

The delay is DELAY_S of SM clock cycles at the clock rate the device reports: 79.2 M cycles at 1980 MHz on an H100
80GB HBM3 (700 W power limit), measured at 41.7, 42.6 and 51.9 ms with CUDA events in three runs
(test_delay_kernel_is_long_enough prints it). The whole file ran in 28 to 43 s there."""
import functools
import threading
import zlib

import numpy as np
import pytest
import torch

import jolt_b200
from jolt_b200 import (HIGH_TO_LOW, LOW_TO_HIGH, BatchMember, BooleanityMember, EqPlusOnePolynomial, EqPolynomial,
                       ExpressionMember, G1Bases, LinearTerm, LtPolynomial, Polynomial, ProductMember,
                       ReadWriteCheckingMember, Source, evaluate_small, g1_jacobian_to_affine, one_hot_evaluate,
                       one_hot_pushforward)
from jolt_b200 import field as F
from jolt_b200.api import small_scalars
from oracle import bn254 as O
from oracle import coracle as C
import booleanity_ref as B
import expr_ref as E
import lincomb_ref as LR
import mle_eval_ref as M
import rw_ref as RW
import source_ref as SR
import sumcheck_ref as S
import vmp_ref as V

pytestmark = pytest.mark.gpu
P = O.R_MOD
DELAY_S = 0.04
GAMMA = 0x1234567890ABCDEF1234567890ABCDEF
G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
MODES = ("private", "legacy", "side")
N = 14  # log2 of the table / column length: many blocks, quick references


# ---- sessions and streams -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sessions():
    side = torch.cuda.Stream()
    s = {"private": jolt_b200.Session(0),
         "legacy": jolt_b200.Session(0, cuda_stream=torch.cuda.current_stream().cuda_stream),
         "side": jolt_b200.Session(0, cuda_stream=side.cuda_stream)}
    assert s["legacy"].stream == 0 and s["side"].stream == side.cuda_stream and s["private"].stream not in (0, side.cuda_stream)
    yield s, side
    torch.cuda.synchronize()
    for x in s.values():
        x.close()


@pytest.fixture(params=MODES)
def sess(request, sessions):
    s, side = sessions
    if request.param == "side":
        with torch.cuda.stream(side):
            yield s["side"]
    else:
        yield s[request.param]
    torch.cuda.synchronize()


@functools.lru_cache(maxsize=None)
def _cycles() -> int:
    return int(torch.cuda.get_device_properties(0).clock_rate * 1e3 * DELAY_S)  # clock_rate is in kHz


def session_stream(sess):
    """The session's stream as a torch stream (independently of the library's own ordering helpers)."""
    return torch.cuda.default_stream(0) if sess.stream == 0 else torch.cuda.ExternalStream(sess.stream, device=0)


def late(arrays, sentinels):
    """CUDA tensors holding their sentinel until device copies of `arrays`, queued on torch's current stream behind one
    delay kernel, write the data; and an event recorded after the copies."""
    srcs = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    bufs = [torch.empty_like(s) for s in srcs]
    for b, v in zip(bufs, sentinels):
        b.fill_(v)
    torch.cuda.synchronize()
    torch.cuda._sleep(_cycles())
    for b, s in zip(bufs, srcs):
        b.copy_(s)
    done = torch.cuda.Event()
    done.record()
    return bufs, done


def pending(done):
    assert not done.query(), f"the producer finished before the library call: raise DELAY_S (now {DELAY_S} s)"


def race(arrays, sentinels, call):
    """call(tensors) first on the data already in place, then on tensors still being produced (late). The first run
    loads every kernel the call uses: a kernel's first launch in the process loads its module, which synchronises the
    device and would order the read after the producer by accident."""
    ready = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    call(ready)
    bufs, done = late(arrays, sentinels)
    pending(done)
    call(bufs)


def busy(sess):
    """Holds the session's stream with a delay kernel, so that what the library enqueues next is still to run."""
    with torch.cuda.stream(session_stream(sess)):
        torch.cuda._sleep(_cycles())


def session_event(sess):
    ev = torch.cuda.Event()
    ev.record(session_stream(sess))
    return ev


class _DeviceView:
    """A (n, 4) int64 view of n field entries of device memory, for torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 4), "typestr": "<i8", "data": (ptr, False), "version": 2}


def torch_reads(ptr, n) -> list[int]:
    """What torch's current stream reads at ptr: a device copy on that stream, then the host copy of it."""
    t = torch.as_tensor(_DeviceView(ptr, n), device="cuda").clone()
    return F.limbs_to_ints(t.cpu().numpy().view(np.uint64))


def limbs_tensor_input(limbs):
    return limbs.view(np.int64)


def ints(limbs):
    return F.limbs_to_ints(limbs)


# ---- data ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def table(seed, n=N):
    return C.rand_limbs(seed, 1 << n)


@functools.lru_cache(maxsize=None)
def point(seed, n=N):
    return tuple(O.random_fr(seed, n))


def challenges(seed, n):
    """full and 125-bit challenges, alternating"""
    return [F.from_limbs(C.rand_challenge(seed + i)) if i % 2 else O.random_fr(seed + i, 1)[0] for i in range(n)]


COMPACT_KINDS = ("u8", "u64", "i128", "s64")
COMPACT_SENTINEL = 7


@functools.lru_cache(maxsize=None)
def compact(kind, seed, n=N):
    """(the raw records as a numpy array for the device, the values as mle_eval_ref.promote takes them)"""
    rng = np.random.default_rng(seed)
    if kind == "u8":
        a = rng.integers(0, 256, 1 << n).astype(np.uint8)
        return a, [int(v) for v in a]
    if kind == "u64":
        a = rng.integers(0, 1 << 64, 1 << n, dtype=np.uint64)
        a[::97] = np.uint64((1 << 64) - 1)
        return a.view(np.int64), [int(v) for v in a]
    if kind == "i128":
        vals = [int(rng.integers(0, 1 << 62)) * int(rng.integers(1, 1 << 62)) * (-1 if i % 3 else 1) for i in range(1 << n)]
        vals[5], vals[6] = -(1 << 127), (1 << 127) - 1
    else:  # s64: (magnitude, is_positive), -0 included
        vals = [(int(rng.integers(0, 1 << 63)) * 2 + i % 2, bool(i % 3)) for i in range(1 << n)]
        vals[5], vals[6] = (0, False), ((1 << 64) - 1, False)
    rec, _k, _n = small_scalars(vals, kind)
    return rec.view(np.int64), vals


def one_hot_sentinel(dtype):
    return 0xFF if dtype == np.uint8 else -1  # the none value (u16 columns travel as int16 words)


@functools.lru_cache(maxsize=None)
def address_column(seed, T, K, dtype):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, K, T).astype(dtype)
    a[rng.random(T) < 0.2] = np.iinfo(dtype).max
    return a


def device_words(col):
    """What a column travels as: uint8 stays, uint16 as int16 words."""
    return col if col.dtype == np.uint8 else col.view(np.int16)


# ---- the delay itself ----------------------------------------------------------------------------------------------
def test_delay_kernel_is_long_enough():
    """The delay kernel behind every producer lasts at least a quarter of DELAY_S (it measured ~DELAY_S on an H100)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(_cycles())
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1)
    print(f"delay kernel: {_cycles()} cycles = {ms:.1f} ms")
    assert ms >= DELAY_S * 1e3 / 4


# ---- inputs: wrapped field tables -----------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_wrapped_table_bind(sess, order):
    t = table(1)
    r = challenges(11, 1)[0]
    want = ints(C.bind(t, F.to_limbs(r), order))

    def call(bufs):
        p = Polynomial.wrap_device(sess, bufs[0].data_ptr(), 1 << N)
        p.bind(r, order)
        assert p.to_ints() == want
        p.free()
    race([limbs_tensor_input(t)], [0], call)


@functools.lru_cache(maxsize=None)
def _evaluate_want():
    return [M.evaluate(ints(table(s)), list(point(21))) for s in (2, 3)]


def test_wrapped_table_evaluate(sess):
    want = _evaluate_want()

    def call(bufs):
        pa = Polynomial.wrap_device(sess, bufs[0].data_ptr(), 1 << N)
        pb = Polynomial.wrap_device(sess, bufs[1].data_ptr(), 1 << N)
        assert pa.evaluate(list(point(21))) == want[0]
        assert Polynomial.batch_evaluate([pa, pb], list(point(21))) == want
        pa.free()
        pb.free()
    race([limbs_tensor_input(table(2)), limbs_tensor_input(table(3))], [0, 0], call)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_wrapped_tables_product_member(sess, order):
    tabs = [table(4), table(5)]
    ch = challenges(31, N)
    want, cur, bind = [], tabs, None
    for rnd in range(N):
        if bind is not None:
            cur = [C.bind(t, F.to_limbs(bind), order) for t in cur]
        want.append(C.mont_to_ints(C.product_round_evals(cur, 2, order)))
        bind = ch[rnd]
    finals = [ints(C.bind(t, F.to_limbs(bind), order))[0] for t in cur]

    def call(bufs):
        gpu = ProductMember(sess, [Polynomial.wrap_device(sess, b.data_ptr(), 1 << N) for b in bufs], order)
        bind = None
        for rnd in range(N):
            assert gpu.prove_round_evals(bind, rnd, (want[rnd][0] + want[rnd][1]) % P) == want[rnd], f"round {rnd}"
            bind = ch[rnd]
        gpu.finish_rounds(bind)
        assert gpu.final_evals() == finals
        gpu.close()
    race([limbs_tensor_input(t) for t in tabs], [0, 0], call)


EXPR_MONOMIALS = [(1, [0, 1]), (GAMMA, [2, 2, 0]), (-1, [1])]


@functools.lru_cache(maxsize=None)
def _expression_want(order):
    ref = E.ExpressionMember([ints(table(s)) for s in (6, 7, 8)], EXPR_MONOMIALS, order)
    ch = challenges(41, N)
    claim, rounds, bind = ref.claim(), [], None
    for rnd in range(N):
        rounds.append(ref.round_evals(bind))
        bind = ch[rnd]
    ref.finish_rounds(bind)
    return claim, rounds, ref.final_evals()


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
def test_wrapped_tables_expression_member(sess, order):
    claim0, rounds, finals = _expression_want(order)
    ch = challenges(41, N)

    def call(bufs):
        gpu = ExpressionMember(sess, [Polynomial.wrap_device(sess, b.data_ptr(), 1 << N) for b in bufs], EXPR_MONOMIALS,
                               order=order)
        claim, bind = claim0, None
        for rnd in range(N):
            assert gpu.prove_round_evals(bind, rnd, claim) == rounds[rnd], f"round {rnd}"
            claim = O.uni_evaluate(O.uni_from_evals(rounds[rnd]), ch[rnd])
            bind = ch[rnd]
        gpu.finish_rounds(bind)
        assert gpu.final_evals() == finals
        gpu.close()
    race([limbs_tensor_input(table(s)) for s in (6, 7, 8)], [0, 0, 0], call)


def _weighted_sum(sc_limbs: np.ndarray) -> int:
    """sum_i s_i (i + 1) mod r from Montgomery limbs: the MSM over bases (i + 1) G is this multiple of G."""
    a = np.ascontiguousarray(sc_limbs, dtype=np.uint64).reshape(-1, 4)
    wts = np.arange(1, a.shape[0] + 1, dtype=object)
    total = 0
    for limb in range(4):
        for half in range(2):
            words = ((a[:, limb] >> np.uint64(32 * half)) & np.uint64(0xFFFFFFFF)).astype(object)
            total += int((words * wts).sum()) << (64 * limb + 32 * half)
    return total * pow(1 << 256, -1, P) % P


@functools.lru_cache(maxsize=None)
def _msm_want():
    return O.g1_scalar_mul(O.G1_GEN, _weighted_sum(table(9)))


def test_wrapped_table_msm(sess):
    bases = G1Bases.generate_multiples(sess, G, 1 << N)
    want = _msm_want()
    sess.synchronize()

    def call(bufs):
        p = Polynomial.wrap_device(sess, bufs[0].data_ptr(), 1 << N)
        assert g1_jacobian_to_affine(bases.msm(p)) == want
        p.free()
    race([limbs_tensor_input(table(9))], [0], call)
    bases.free()


# ---- inputs: device compact columns --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _compact_refs(kind):
    _a, vals = compact(kind, 51)
    prom = [M.promote(v) for v in vals]
    t = ints(table(52))
    terms = [("compact", vals, GAMMA), ("table", t, 3)]
    left = O.random_fr(53, 1 << (N - 7))
    return dict(eval=M.evaluate(prom, list(point(54))), lc=LR.linear_combination(terms, 1 << N),
                vmp=V.vector_matrix_product(terms, 1 << N, 1 << 7, left), left=left)


@pytest.mark.parametrize("kind", COMPACT_KINDS)
def test_compact_evaluate_small(sess, kind):
    want = _compact_refs(kind)["eval"]

    def call(bufs):
        assert evaluate_small(sess, bufs[0], list(point(54)), kind) == [want]
    race([compact(kind, 51)[0]], [COMPACT_SENTINEL], call)


@pytest.mark.parametrize("op", ["linear_combination", "vector_matrix_product"])
@pytest.mark.parametrize("kind", COMPACT_KINDS)
def test_compact_linear_term(sess, kind, op):
    ref = _compact_refs(kind)
    tp = Polynomial.new(sess, table(52))
    left = Polynomial.from_ints(sess, ref["left"])
    sess.synchronize()

    def call(bufs):
        terms = [LinearTerm.compact(bufs[0], GAMMA, kind), LinearTerm.table(tp, 3)]
        if op == "linear_combination":
            out = Polynomial.linear_combination(sess, terms)
            assert out.to_ints() == ref["lc"]
        else:
            out = Polynomial.vector_matrix_product(sess, terms, left, 1 << 7)
            assert out.to_ints() == ref["vmp"]
        out.free()
    race([compact(kind, 51)[0]], [COMPACT_SENTINEL], call)
    tp.free()
    left.free()


SOURCE_MONOMIALS = {"expression": [(1, [0, 1]), (GAMMA, [0, 0])], "product": [(1, [0, 1])]}


@functools.lru_cache(maxsize=None)
def _sources_want(sources_key, shape, order):
    if sources_key[0] == "compact":
        refsrc = [("compact", compact(sources_key[1], 61)[1]), ("table", ints(table(62)))]
    else:
        _tag, T, K, dtype = sources_key
        refsrc = [("one_hot", SR.addresses(address_column(63, T, K, dtype)), K, list(point(64, K.bit_length() - 1))),
                  ("table", ints(table(62)))]
    ref = SR.SourcesMember(refsrc, SOURCE_MONOMIALS[shape], order)
    ch = challenges(65, N)
    claim, rounds, bind = ref.claim(), [], None
    for rnd in range(N):
        rounds.append(ref.round_evals(bind))
        bind = ch[rnd]
    ref.finish_rounds(bind)
    return claim, rounds, ref.final_evals()


def _sources_member(sess, shape, source, order):
    src = [source, Source.table(Polynomial.new(sess, table(62)))]
    if shape == "expression":
        return ExpressionMember.from_sources(sess, src, SOURCE_MONOMIALS[shape], order=order)
    return ProductMember.from_sources(sess, src, order=order)


def _drive_sources(gpu, want):
    claim, rounds, finals = want
    ch = challenges(65, N)
    bind = None
    for rnd in range(N):
        assert gpu.prove_round_evals(bind, rnd, claim) == rounds[rnd], f"round {rnd}"
        claim = O.uni_evaluate(O.uni_from_evals(rounds[rnd]), ch[rnd])
        bind = ch[rnd]
    gpu.finish_rounds(bind)
    assert gpu.final_evals() == finals
    gpu.close()


@pytest.mark.parametrize("shape", ["expression", "product"])
@pytest.mark.parametrize("kind", COMPACT_KINDS)
def test_compact_source(sess, kind, shape):
    order = HIGH_TO_LOW if kind in ("u8", "i128") else LOW_TO_HIGH
    want = _sources_want(("compact", kind), shape, order)
    race([compact(kind, 61)[0]], [COMPACT_SENTINEL],
         lambda bufs: _drive_sources(_sources_member(sess, shape, Source.compact(bufs[0], kind), order), want))


# ---- inputs: device one-hot address columns --------------------------------------------------------------------------
ONE_HOT = [(np.uint8, 16), (np.uint16, 1024)]
ONE_HOT_IDS = ["u8", "u16"]


@pytest.mark.parametrize("dtype,K", ONE_HOT, ids=ONE_HOT_IDS)
def test_one_hot_evaluate(sess, dtype, K):
    T = 1 << N
    cols = [address_column(71, T, K, dtype), address_column(72, T, K, dtype)]
    pt = list(point(73, N + K.bit_length() - 1))
    want = [M.one_hot_evaluate_direct(SR.addresses(c), K, T, pt, "cycle_major") for c in cols]

    def call(bufs):
        assert one_hot_evaluate(sess, bufs, K, pt) == want
    race([device_words(c) for c in cols], [one_hot_sentinel(dtype)] * 2, call)


@pytest.mark.parametrize("dtype,K", ONE_HOT, ids=ONE_HOT_IDS)
def test_one_hot_pushforward(sess, dtype, K):
    T = 1 << N
    col = address_column(74, T, K, dtype)
    r = list(point(75))
    want = M.pushforward(SR.addresses(col), K, r)

    def call(bufs):
        (g,) = one_hot_pushforward(sess, bufs[0], K, r)
        assert g.to_ints() == want
        g.free()
    race([device_words(col)], [one_hot_sentinel(dtype)], call)


@functools.lru_cache(maxsize=None)
def _one_hot_lc_want(dtype, layout):
    T, K = 1 << 12, 16
    addr = SR.addresses(address_column(76, T, K, dtype))
    return LR.linear_combination([("one_hot", addr, K, layout, GAMMA), ("table", ints(table(77, 16)), 5)], K * T)


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16], ids=ONE_HOT_IDS)
def test_one_hot_linear_term(sess, dtype, layout):
    T, K = 1 << 12, 16
    want = _one_hot_lc_want(dtype, layout)
    tp = Polynomial.new(sess, table(77, 16))
    sess.synchronize()

    def call(bufs):
        out = Polynomial.linear_combination(sess, [LinearTerm.one_hot(bufs[0], K, GAMMA, layout), LinearTerm.table(tp, 5)])
        assert out.to_ints() == want
        out.free()
    race([device_words(address_column(76, T, K, dtype))], [one_hot_sentinel(dtype)], call)
    tp.free()


@pytest.mark.parametrize("shape", ["expression", "product"])
@pytest.mark.parametrize("dtype,K", ONE_HOT, ids=ONE_HOT_IDS)
def test_one_hot_source(sess, dtype, K, shape):
    T = 1 << N
    order = LOW_TO_HIGH if shape == "product" else HIGH_TO_LOW
    want = _sources_want(("one_hot", T, K, dtype), shape, order)
    r_addr = list(point(64, K.bit_length() - 1))
    race([device_words(address_column(63, T, K, dtype))], [one_hot_sentinel(dtype)],
         lambda bufs: _drive_sources(_sources_member(sess, shape, Source.one_hot(bufs[0], K, r_addr), order), want))


BOOL_K, BOOL_T, BOOL_D = 16, 1 << 12, 2


@functools.lru_cache(maxsize=None)
def _booleanity_inputs(dtype, order):
    addrs = B.random_columns(81, BOOL_K, BOOL_T, BOOL_D)
    lk, lt = BOOL_K.bit_length() - 1, BOOL_T.bit_length() - 1
    coeffs, r_addr, r_cycle = O.random_fr(82, BOOL_D), O.random_fr(83, lk), O.random_fr(84, lt)
    scale, ch = O.random_fr(85, 1)[0], challenges(86, lk + lt)
    want = B.sparse_prove(BOOL_K, BOOL_T, addrs, coeffs, r_addr, r_cycle, scale, ch, order)
    return addrs, coeffs, r_addr, r_cycle, scale, ch, want


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16], ids=ONE_HOT_IDS)
def test_one_hot_booleanity(sess, dtype, order):
    addrs, coeffs, r_addr, r_cycle, scale, ch, (want_rounds, want_final) = _booleanity_inputs(dtype, order)
    cols = B.column_arrays(addrs, BOOL_K, dtype)

    def call(bufs):
        m = BooleanityMember(sess, bufs, BOOL_K, coeffs, r_addr, r_cycle, scale, order)
        claim, bind = 0, None
        for rnd in range(len(ch)):
            got = m.prove_round_evals(bind, rnd, claim)
            assert got == want_rounds[rnd], f"round {rnd}"
            claim = O.uni_evaluate(O.uni_from_evals(got), ch[rnd])
            bind = ch[rnd]
        m.finish_rounds(bind)
        assert m.final_evals() == want_final
        m.close()
    race([device_words(c) for c in cols], [one_hot_sentinel(dtype)] * BOOL_D, call)


RW_K, RW_T = 16, 1 << 12


@functools.lru_cache(maxsize=None)
def _rw_inputs():
    wl = RW.workload(91, RW_K, RW_T, 3, "registers")
    t = RW_T.bit_length() - 1
    w, ch = O.random_fr(92, t), challenges(93, t + RW_K.bit_length() - 1)
    K, T, accesses, write, inc, init = wl
    return wl, w, ch, RW.sparse_prove(*wl, w, None, ch), RW.claimed_sum(T, accesses, inc, w)


def test_one_hot_read_write(sess):
    (K, T, accesses, write, inc, init), w, ch, (want_rounds, want_final), claim = _rw_inputs()
    addr = [np.array([0xFF if a is None else a for a in ad], dtype=np.uint8) for ad, _v, _c, _d in accesses]
    values = [F.ints_to_limbs(v) for _ad, v, _c, _d in accesses]
    inc_rec = np.array([x if x < (1 << 127) else x - P for x in inc], dtype=np.int64)
    init_rec = np.array(init, dtype=np.uint64).view(np.int64)
    arrays = addr + [limbs_tensor_input(v) for v in values] + [inc_rec, init_rec]

    def call(bufs):
        vals = [Source.table(Polynomial.wrap_device(sess, b.data_ptr(), T)) for b in bufs[3:6]]
        acc = [(bufs[i], vals[i], c, d) for i, (_ad, _v, c, d) in enumerate(accesses)]
        m = ReadWriteCheckingMember(sess, acc, write, Source.compact(bufs[6], "i64"), Source.compact(bufs[7], "u64"), K, w)
        cl, bind = claim, None
        for rnd in range(len(ch)):
            got = m.prove_round_evals(bind, rnd, cl)
            assert got == want_rounds[rnd], f"round {rnd}"
            cl = O.uni_evaluate(O.uni_from_evals(got), ch[rnd])
            bind = ch[rnd]
        m.finish_rounds(bind)
        assert m.final_evals() == want_final
        m.close()
        for v in vals:
            v.poly.free()
    race(arrays, [0xFF] * 3 + [0] * 3 + [COMPACT_SENTINEL] * 2, call)


# ---- outputs: the library writes, torch reads on its current stream ---------------------------------------------------
def test_bind_in_place_read_by_torch(sess):
    t = table(101)
    r = challenges(102, 1)[0]
    want = ints(C.bind(t, F.to_limbs(r), HIGH_TO_LOW))
    buf = torch.from_numpy(limbs_tensor_input(t)).cuda()
    warm = buf.clone()  # a first bind loads the kernel (see race)
    torch.cuda.synchronize()
    Polynomial.wrap_device(sess, warm.data_ptr(), 1 << N).bind(r, HIGH_TO_LOW)
    sess.synchronize()
    p = Polynomial.wrap_device(sess, buf.data_ptr(), 1 << N)
    busy(sess)
    p.bind(r, HIGH_TO_LOW)
    pending(session_event(sess))
    got = buf[: 1 << (N - 1)].clone()   # a copy on torch's current stream
    total = buf[: 1 << (N - 1)].sum(dim=0)  # and a reduction
    assert F.limbs_to_ints(got.cpu().numpy().view(np.uint64)) == want
    w = F.ints_to_limbs(want).view(np.int64).astype(object).sum(axis=0)
    assert [int(x) for x in total.cpu()] == [int((int(x) + (1 << 63)) % (1 << 64) - (1 << 63)) for x in w]
    p.free()


def test_export_table_read_by_torch(sess):
    t0, t1 = table(103), table(104)
    r = challenges(105, 1)[0]
    want = ints(C.bind(t0, F.to_limbs(r), LOW_TO_HIGH))
    m = ExpressionMember(sess, [Polynomial.new(sess, t0), Polynomial.new(sess, t1)], [(1, [0, 1]), (GAMMA, [1])],
                         order=LOW_TO_HIGH)
    m.prove_round_evals(None, 0)
    m.prove_round_evals(r, 1)
    dst = torch.zeros((1 << (N - 1), 4), dtype=torch.int64, device="cuda")
    m.export_table(1, dst)  # a first export loads what it uses (see race); then dst is zeroed again
    sess.synchronize()
    dst.zero_()
    torch.cuda.synchronize()
    busy(sess)
    assert m.export_table(0, dst) == 1 << (N - 1)
    pending(session_event(sess))
    got = dst.clone()
    assert F.limbs_to_ints(got.cpu().numpy().view(np.uint64)) == want
    m.close()


def _new_table_want(what, seed):
    e = O.eq_evals(list(point(seed)))
    if what == "eq":
        return e
    if what == "eq_plus_one":
        return [0] + e[:-1]
    lt, acc = [0] * len(e), 0  # LT[j] = sum_{t > j} eq(r, t)
    for j in range(len(e) - 1, -1, -1):
        lt[j] = acc
        acc = (acc + e[j]) % P
    return lt


# (linear_combination, vector_matrix_product and one_hot_pushforward synchronise before they return - they report bad
# addresses found on the device - so their tables are complete by then and there is no race to test here)
@pytest.mark.parametrize("what", ["eq", "lt", "eq_plus_one"])
def test_new_table_read_by_torch(request, sess, what):
    """The new table lands in a block of the stream-ordered pool, which keeps freed blocks: its old contents are what a
    read that is not ordered after the library's write sees. So the expected table is one no earlier call has built
    (a point of its own per test and mode), and the warm-up call builds another one at another point."""
    seed = 0x5EE0000 + zlib.crc32(request.node.name.encode())
    want = _new_table_want(what, seed)
    cls = {"eq": EqPolynomial, "lt": LtPolynomial, "eq_plus_one": EqPlusOnePolynomial}[what]
    cls.evals(sess, F.ints_to_limbs(list(point(seed + 1)))).free()  # a first call loads the kernels (see race)
    sess.synchronize()
    busy(sess)
    out = cls.evals(sess, F.ints_to_limbs(list(point(seed))))
    pending(session_event(sess))
    got = torch_reads(out.device_ptr(), len(want))
    assert got == want, f"{sum(a != b for a, b in zip(got, want))} of {len(want)} entries differ"
    out.free()


# ---- bench's configuration at test size ------------------------------------------------------------------------------
def _synth(seed, n, out=None):
    """bench.py's synthetic table: raw limbs < 2^252 < r, canonical Montgomery values, made by device kernels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randint(0, 2 ** 62, (1 << n, 4), dtype=torch.int64, device="cuda", generator=g, out=out)
    t[:, 3] &= (1 << 60) - 1
    return t


def _host_synth(seeds, n):
    """The values of bench's tables, on the host."""
    return [_synth(s, n).cpu().numpy().view(np.uint64).copy() for s in seeds]


def _late_synth(seeds, n):
    """bench's tables made again by the same generators behind a delay kernel on torch's current stream, over zeroed
    buffers; and an event recorded after them."""
    bufs = [torch.zeros((1 << n, 4), dtype=torch.int64, device="cuda") for _ in seeds]
    torch.cuda.synchronize()
    torch.cuda._sleep(_cycles())
    for s, b in zip(seeds, bufs):
        _synth(s, n, out=b)
    done = torch.cuda.Event()
    done.record()
    return bufs, done


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("log_n", [16, 18])
@pytest.mark.parametrize("m", [2, 3])
def test_bench_configuration_prove_batch(sessions, m, log_n, order):
    """A side-stream session proving bench's tables, wrapped while torch is still writing them, with no host
    synchronisation in between: every round polynomial and final evaluation equals the C oracle."""
    s, side = sessions
    sess = s["side"]
    thr = C.max_threads()
    seeds = [0xB200 + 16 * m + j for j in range(m)]
    with torch.cuda.stream(side):
        host = _host_synth(seeds, log_n)
        ev = C.mont_to_ints(C.product_round_evals(host, m, order, thr))
        claim = (ev[0] + ev[1]) % P
        bufs, done = _late_synth(seeds, log_n)
        pending(done)
        mem = ProductMember(sess, [Polynomial.wrap_device(sess, b.data_ptr(), 1 << log_n) for b in bufs], order)
        res = jolt_b200.prove_batch_native([BatchMember(claim, 1, log_n, 0)], [mem], log_n, m, claim, seed=7)
        fe = mem.final_evals()
        mem.close()
        torch.cuda.synchronize()
    cur = host
    for rnd in range(log_n):
        if rnd:
            cur = [C.bind(t, F.to_limbs(res.challenges[rnd - 1]), order, thr) for t in cur]
        want = S.trimmed_coeffs(C.mont_to_ints(C.product_round_evals(cur, m, order, thr)))
        assert res.round_polynomials[rnd].coefficients == want, f"round {rnd}"
    cur = [C.bind(t, F.to_limbs(res.challenges[-1]), order, thr) for t in cur]
    assert fe == [ints(t)[0] for t in cur]
    assert res.final_claim == int(np.prod(np.array(fe, dtype=object)) % P)


@pytest.mark.parametrize("order", [HIGH_TO_LOW, LOW_TO_HIGH])
@pytest.mark.parametrize("log_n", [16, 18])
@pytest.mark.parametrize("m", [2, 3])
def test_bench_configuration_interleaved_torch(sessions, m, log_n, order):
    """The same tables driven round by round, with torch kernels queued on the session's stream between the rounds
    and no host synchronisation: every round equals the C oracle, and torch's own results are intact."""
    s, side = sessions
    sess = s["side"]
    thr = C.max_threads()
    ch = challenges(0x5EED + m, log_n)
    seeds = [0xC300 + 16 * m + j for j in range(m)]
    with torch.cuda.stream(side):
        host = _host_synth(seeds, log_n)
        scratch = torch.arange(1 << 20, dtype=torch.int64, device="cuda")
        bufs, done = _late_synth(seeds, log_n)
        pending(done)
        gpu = ProductMember(sess, [Polynomial.wrap_device(sess, b.data_ptr(), 1 << log_n) for b in bufs], order)
        cur, bind = host, None
        for rnd in range(log_n):
            scratch.mul_(3).add_(1)  # torch work between the rounds, on the same stream
            if bind is not None:
                cur = [C.bind(t, F.to_limbs(bind), order, thr) for t in cur]
            want = C.mont_to_ints(C.product_round_evals(cur, m, order, thr))
            assert gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % P) == want, f"round {rnd}"
            bind = ch[rnd]
        gpu.finish_rounds(bind)
        assert gpu.final_evals() == [ints(C.bind(t, F.to_limbs(bind), order, thr))[0] for t in cur]
        gpu.close()
        x = np.arange(1 << 20, dtype=np.int64)
        for _ in range(log_n):
            x = x * 3 + 1
        assert np.array_equal(scratch.cpu().numpy(), x)


# ---- threads ------------------------------------------------------------------------------------------------------
def _run_threads(fns):
    """Runs every fn on its own thread, all released together; re-raises the first failure."""
    start = threading.Barrier(len(fns))
    errors = []

    def wrap(fn):
        try:
            start.wait()
            fn()
        except BaseException as e:  # noqa: BLE001 - reported on the main thread
            errors.append(e)

    ts = [threading.Thread(target=wrap, args=(f,)) for f in fns]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0]


TH_N = 12
REPEATS = 4


@functools.lru_cache(maxsize=None)
def _srs():
    beta = C.ints_to_mont([O.random_fr(0x7E4D, 1)[0]])[0]
    return C.g1_powers(1 << TH_N, G, beta)


def _pippenger(scalars_mont, n=None):
    bases = _srs()[: scalars_mont.shape[0] if n is None else n]
    xy, inf = C.g1_msm_pippenger(bases, scalars_mont, 0, C.max_threads())
    return None if inf else (O.from_mont_limbs(xy[:4], O.Q_MOD), O.from_mont_limbs(xy[4:], O.Q_MOD))


def _session_work(sess, bases, seed):
    """Six independent jobs on one session, each checked against its reference, each repeated."""
    n = 1 << TH_N
    sc = C.rand_limbs(seed, n)
    u8 = np.random.default_rng(seed).integers(0, 256, n).astype(np.uint8)
    u64 = np.random.default_rng(seed + 1).integers(0, 1 << 64, n // 2, dtype=np.uint64)
    want_msm, want_u8 = _pippenger(sc), _pippenger(C.ints_to_mont([int(v) for v in u8]))
    want_batch = [_pippenger(sc[: n // 4]), _pippenger(C.ints_to_mont([int(v) for v in u64]))]
    t1, t2 = C.rand_limbs(seed + 2, n), C.rand_limbs(seed + 3, n)
    pt = O.random_fr(seed + 4, TH_N)
    want_eval = M.evaluate(ints(t1), pt)
    want_lc = LR.linear_combination([("table", ints(t1), GAMMA), ("compact", [int(v) for v in u8], 5)], n)
    ch = challenges(seed + 5, TH_N)

    def msm():
        for _ in range(REPEATS):
            assert g1_jacobian_to_affine(bases.msm(sc)) == want_msm

    def msm_small():
        for _ in range(REPEATS):
            assert g1_jacobian_to_affine(bases.msm_small(u8)) == want_u8

    def batch_msm():
        for _ in range(REPEATS):
            got = bases.batch_msm([sc[: n // 4], u64])
            assert [g1_jacobian_to_affine(g) for g in got] == want_batch

    def evaluate():
        p = Polynomial.new(sess, t1)
        for _ in range(REPEATS):
            assert p.evaluate(pt) == want_eval
        p.free()

    def linear_combination():
        p = Polynomial.new(sess, t1)
        for _ in range(REPEATS):
            out = Polynomial.linear_combination(sess, [LinearTerm.table(p, GAMMA), LinearTerm.compact(u8, 5)])
            assert out.to_ints() == want_lc
            out.free()
        p.free()

    def member():
        for _ in range(REPEATS):
            gpu = ProductMember(sess, [Polynomial.new(sess, t1), Polynomial.new(sess, t2)], LOW_TO_HIGH)
            cur, bind = [t1, t2], None
            for rnd in range(TH_N):
                if bind is not None:
                    cur = [C.bind(t, F.to_limbs(bind), LOW_TO_HIGH) for t in cur]
                want = C.mont_to_ints(C.product_round_evals(cur, 2, LOW_TO_HIGH))
                assert gpu.prove_round_evals(bind, rnd, (want[0] + want[1]) % P) == want, f"round {rnd}"
                bind = ch[rnd]
            gpu.finish_rounds(bind)
            assert gpu.final_evals() == [ints(C.bind(t, F.to_limbs(bind), LOW_TO_HIGH))[0] for t in cur]
            gpu.close()

    return [msm, msm_small, batch_msm, evaluate, linear_combination, member]


def test_threads_share_one_session():
    """Six Python threads (ctypes drops the GIL during a call) call one session at once, each on its own data."""
    sess = jolt_b200.Session(0)
    try:
        bases = G1Bases.from_affine(sess, _srs())
        _run_threads(_session_work(sess, bases, 0x7A00))
        bases.free()
    finally:
        sess.close()


def test_two_sessions_two_threads():
    """Two sessions on one device, each driven by its own thread through all six jobs in turn."""
    sessions = [jolt_b200.Session(0), jolt_b200.Session(0)]
    try:
        bases = [G1Bases.from_affine(s, _srs()) for s in sessions]
        jobs = [_session_work(s, b, 0x7B00 + 64 * i) for i, (s, b) in enumerate(zip(sessions, bases))]
        _run_threads([lambda js=js: [j() for j in js] for js in jobs])
        for b in bases:
            b.free()
    finally:
        for s in sessions:
            s.close()
