// Sumcheck members on the device: ProveRounds (crates/jolt-sumcheck/src/prover.rs:52-72) for sum-of-products
// relations over dense tables, the split-eq (Gruen) member, the index-sharded member, and the device
// RoundScheduler (prover.rs:106-120). See include/jolt_b200.h for the per-function reference citations.
#include "../../include/jolt_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "columns.cuh"
#include "member.hpp"
#include "resident.cuh"
#include "sumcheck_host.hpp"

using namespace jb;
using namespace jbi;
using Guard = CtxGuard;


// result slots in host-mapped memory: slot s = h_result + s * JB_SLOT_U64: [0, 64) values, [64] sequence flag, [72, 76)
// a 17th value (the product pass of 16 factors in verify mode, slot_values)
constexpr int JB_SLOT_U64 = 128;

namespace {

// WEIGHTED: a split-eq member's pass (SKIP1: s(1) comes from the claim)
template <int M, int P, int ORDER, bool BIND, bool HI4, bool SKIP1, bool WEIGHTED>
int launch_fused(jb_ctx* c, const TablePtrs& tp, size_t pairs, const BindScalar& s, const RoundOut& out) {
    auto kernel = fused_round_kernel<M, P, ORDER, BIND, HI4, SKIP1, WEIGHTED>;
    constexpr size_t smem = FusedShape<M, SKIP1>::smem_bytes(FUSED_BLOCK);
    static int per_sm = [&] {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int nb = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, FUSED_BLOCK, smem) != cudaSuccess || nb < 1) nb = 1;
        return nb;
    }();
    return launch_round(c, kernel, FUSED_BLOCK, smem, per_sm, pairs, FusedShape<M, SKIP1>::K, BIND ? 0 : 2, M * P,
                        WEIGHTED ? "fused_round_kernel (weighted) launch" : "fused_round_kernel launch", out, tp, pairs, s);
}

template <int M, int P, int ORDER, bool SKIP1, bool WEIGHTED = false>
int dispatch_fused2(jb_ctx* c, const TablePtrs& tp, size_t pairs, bool bind, bool hi4, const BindScalar& s,
                    const RoundOut& out) {
    if (!bind) return launch_fused<M, P, ORDER, false, false, SKIP1, WEIGHTED>(c, tp, pairs, s, out);
    return hi4 ? launch_fused<M, P, ORDER, true, true, SKIP1, WEIGHTED>(c, tp, pairs, s, out)
               : launch_fused<M, P, ORDER, true, false, SKIP1, WEIGHTED>(c, tp, pairs, s, out);
}

int dispatch_weighted(jb_ctx* c, int m, int order, const TablePtrs& tp, size_t pairs, bool bind, bool hi4, const BindScalar& s,
                      const RoundOut& out) {
    const bool l2h = order == JB_LOW_TO_HIGH;
    switch (m) {
        case 1: return l2h ? dispatch_fused2<1, 1, ORDER_LOW_TO_HIGH, true, true>(c, tp, pairs, bind, hi4, s, out)
                           : dispatch_fused2<1, 1, ORDER_HIGH_TO_LOW, true, true>(c, tp, pairs, bind, hi4, s, out);
        case 2: return l2h ? dispatch_fused2<2, 1, ORDER_LOW_TO_HIGH, true, true>(c, tp, pairs, bind, hi4, s, out)
                           : dispatch_fused2<2, 1, ORDER_HIGH_TO_LOW, true, true>(c, tp, pairs, bind, hi4, s, out);
        case 3: return l2h ? dispatch_fused2<3, 1, ORDER_LOW_TO_HIGH, true, true>(c, tp, pairs, bind, hi4, s, out)
                           : dispatch_fused2<3, 1, ORDER_HIGH_TO_LOW, true, true>(c, tp, pairs, bind, hi4, s, out);
        default: return c->fail(JB_ERR_UNSUPPORTED, "eq member: m must be 1..3");
    }
}

template <int M, int P>
int dispatch_fused1(jb_ctx* c, int order, bool skip1, const TablePtrs& tp, size_t pairs, bool bind, bool hi4,
                    const BindScalar& s, const RoundOut& out) {
    if (order == JB_HIGH_TO_LOW)
        return skip1 ? dispatch_fused2<M, P, ORDER_HIGH_TO_LOW, true>(c, tp, pairs, bind, hi4, s, out)
                     : dispatch_fused2<M, P, ORDER_HIGH_TO_LOW, false>(c, tp, pairs, bind, hi4, s, out);
    return skip1 ? dispatch_fused2<M, P, ORDER_LOW_TO_HIGH, true>(c, tp, pairs, bind, hi4, s, out)
                 : dispatch_fused2<M, P, ORDER_LOW_TO_HIGH, false>(c, tp, pairs, bind, hi4, s, out);
}

// the instantiated shapes: products of 1..4 tables; the two-term degree-2 sum of products
bool shape_supported(int m, int terms) { return (terms == 1 && m >= 1 && m <= 4) || (terms == 2 && m == 2); }

int dispatch_fused(jb_ctx* c, int m, int terms, int order, bool skip1, const TablePtrs& tp, size_t pairs, bool bind,
                   bool hi4, const BindScalar& s, const RoundOut& out) {
    if (terms == 2 && m == 2) return dispatch_fused1<2, 2>(c, order, skip1, tp, pairs, bind, hi4, s, out);
    if (terms != 1) return c->fail(JB_ERR_UNSUPPORTED, "member: unsupported sum-of-products shape");
    switch (m) {
        case 1: return dispatch_fused1<1, 1>(c, order, skip1, tp, pairs, bind, hi4, s, out);
        case 2: return dispatch_fused1<2, 1>(c, order, skip1, tp, pairs, bind, hi4, s, out);
        case 3: return dispatch_fused1<3, 1>(c, order, skip1, tp, pairs, bind, hi4, s, out);
        case 4: return dispatch_fused1<4, 1>(c, order, skip1, tp, pairs, bind, hi4, s, out);
        default: return c->fail(JB_ERR_UNSUPPORTED, "member: m must be 1..4");
    }
}

// expression members (expr_pass.cuh): EXPR_BLOCK threads per block, shared memory by the member's table count
template <int ORDER, bool BIND, bool HI4, bool WEIGHTED>
int launch_expr(jb_ctx* c, const TablePtrs& tp, size_t pairs, const BindScalar& s, const ExprParams& ex, const RoundOut& out) {
    auto kernel = expr_round_kernel<ORDER, BIND, HI4, WEIGHTED>;
    static const bool attr = [&] {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)expr_smem_bytes(EXPR_MAX_TABLES));
        return true;
    }();
    (void)attr;
    static std::atomic<int> per_sm_by_tables[EXPR_MAX_TABLES + 1];  // occupancy depends on the shared memory size
    const size_t smem = expr_smem_bytes(ex.ntables);
    int per_sm = per_sm_by_tables[ex.ntables].load(std::memory_order_relaxed);
    if (per_sm == 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, EXPR_BLOCK, smem) != cudaSuccess || per_sm < 1)
            per_sm = 1;
        per_sm_by_tables[ex.ntables].store(per_sm, std::memory_order_relaxed);
    }
    return launch_round(c, kernel, EXPR_BLOCK, smem, per_sm, pairs, EXPR_MAX_POINTS, BIND ? 0 : 2, ex.D,
                        "expr_round_kernel launch", out, tp, pairs, s, ex);
}

template <int ORDER, bool WEIGHTED>
int dispatch_expr2(jb_ctx* c, const TablePtrs& tp, size_t pairs, bool bind, bool hi4, const BindScalar& s,
                   const ExprParams& ex, const RoundOut& out) {
    if (!bind) return launch_expr<ORDER, false, false, WEIGHTED>(c, tp, pairs, s, ex, out);
    return hi4 ? launch_expr<ORDER, true, true, WEIGHTED>(c, tp, pairs, s, ex, out)
               : launch_expr<ORDER, true, false, WEIGHTED>(c, tp, pairs, s, ex, out);
}

// The round's evaluation points in kernel-value order: 0, [1 unless skip1], 2, .., D-1, inf (D >= 2); 0, [1] (D == 1).
int dispatch_expr(jb_ctx* c, const jb_member* mem, bool weighted, bool skip1, const TablePtrs& tp, size_t pairs, bool bind,
                  bool hi4, const BindScalar& s, const RoundOut& out) {
    ExprParams ex = mem->ex;
    int n = 0;
    ex.point[n++] = 0;
    if (!skip1) ex.point[n++] = 1;
    for (int t = 2; t < ex.D; ++t) ex.point[n++] = (int8_t)t;
    if (ex.D >= 2) ex.point[n++] = EXPR_INF;
    ex.npoints = n;
    if (!mem->src.empty()) return sources_round(c, mem, weighted, tp, pairs, bind, s, ex, out);  // rounds 0 and 1
    if (mem->order == JB_LOW_TO_HIGH)
        return weighted ? dispatch_expr2<ORDER_LOW_TO_HIGH, true>(c, tp, pairs, bind, hi4, s, ex, out)
                        : dispatch_expr2<ORDER_LOW_TO_HIGH, false>(c, tp, pairs, bind, hi4, s, ex, out);
    return weighted ? dispatch_expr2<ORDER_HIGH_TO_LOW, true>(c, tp, pairs, bind, hi4, s, ex, out)
                    : dispatch_expr2<ORDER_HIGH_TO_LOW, false>(c, tp, pairs, bind, hi4, s, ex, out);
}

}  // namespace

jb_member* new_member(jb_ctx* c, MemberKind kind, int m, int terms, int order, size_t len) {
    jb_member* mem = new (std::nothrow) jb_member();
    if (!mem) return nullptr;
    mem->ctx = c;
    mem->kind = kind;
    mem->m = m;
    mem->terms = terms;
    mem->order = order;
    mem->len = len;
    mem->rounds = (size_t)log2_of(len);
    return mem;
}

extern "C" {

// ---- sumcheck member -------------------------------------------------------------------
// The T handles name distinct tables of the context with one power-of-two length (context lock held).
static int check_tables(jb_ctx* c, const jb_table* handles, size_t T, size_t* len_out) {
    size_t len = 0;
    for (size_t j = 0; j < T; ++j) {
        Table* t = c->find(handles[j]);
        if (!t) return c->fail(JB_ERR_INVALID, "member: unknown table handle");
        for (size_t k = 0; k < j; ++k)
            if (handles[k] == handles[j]) return c->fail(JB_ERR_INVALID, "member: duplicate table handle");
        if (j == 0) len = t->len;
        if (t->len != len) return c->fail(JB_ERR_INVALID, "member: tables differ in length");
    }
    if (len == 0 || (len & (len - 1))) return c->fail(JB_ERR_INVALID, "member: table length must be a power of two");
    *len_out = len;
    return JB_OK;
}

// A new member owning the T checked tables (context lock held).
static int adopt_tables(jb_ctx* c, MemberKind kind, const jb_table* handles, size_t T, size_t len, int m, int terms,
                        int order, jb_member** out) {
    jb_member* mem = new_member(c, kind, m, terms, order, len);
    if (!mem) return JB_ERR_OOM;
    for (size_t j = 0; j < T; ++j) {
        auto it = c->tables.find(handles[j]);
        mem->tables.push_back(it->second);
        c->tables.erase(it);  // ownership moves into the member
    }
    *out = mem;
    return JB_OK;
}

static int member_create_common(jb_ctx* c, const jb_table* handles, size_t m, size_t terms, int order, jb_member** out) {
    if (!c || !handles || !out) return JB_ERR_INVALID;
    Guard g(c);
    if (!shape_supported((int)m, (int)terms))
        return c->fail(JB_ERR_UNSUPPORTED, "member: supported shapes are products of 1..4 tables and 2 terms x 2 factors");
    if (order != JB_HIGH_TO_LOW && order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "member: unknown order");
    const size_t T = m * terms;
    size_t len = 0;
    int st = check_tables(c, handles, T, &len);
    if (st != JB_OK) return st;
    return adopt_tables(c, MemberKind::Dense, handles, T, len, (int)m, (int)terms, order, out);
}

int jb_member_create(jb_ctx* c, const jb_table* handles, size_t m, int order, jb_member** out) {
    return member_create_common(c, handles, m, 1, order, out);
}

int jb_member_create_sop(jb_ctx* c, const jb_table* handles, size_t factors, size_t terms, int order, jb_member** out) {
    return member_create_common(c, handles, factors, terms, order, out);
}

int jb_member_num_rounds(jb_member* mem, size_t* rounds) {
    if (!mem || !rounds) return JB_ERR_INVALID;
    *rounds = mem->rounds;
    return JB_OK;
}

// Whether the member's rounds take the split-eq host step (eq_prove_round): a member with split-eq weighting, and every
// read-write and booleanity member (a booleanity member with T = 1 has no eq tables, only its address rounds' factor).
static bool eq_rounds(const jb_member* mem) {
    return mem->eq || mem->kind == MemberKind::ReadWrite || mem->kind == MemberKind::Booleanity;
}

int jb_member_degree(jb_member* mem, size_t* degree) {
    if (!mem || !degree) return JB_ERR_INVALID;
    *degree = (size_t)mem->m + (eq_rounds(mem) ? 1 : 0);
    return JB_OK;
}

jb_ctx* jb_member_context(jb_member* mem) { return mem ? mem->ctx : nullptr; }

int jb_member_num_tables(jb_member* mem, size_t* tables) {
    if (!mem || !tables) return JB_ERR_INVALID;
    *tables = (size_t)mem->ntables();
    return JB_OK;
}

// Runs the fused pass; on return result slot `slot` will hold the K sums (canonical) or, if lanes_out,
// lanes_out holds them widened to one 32-bit limb per u64.
static void* const JB_LANES_EXCHANGE = (void*)(uintptr_t)1;  // sentinel: all-reduce in the kernel epilogue

using EqRound = EqWeights;

// Where a launched round pass reports: result slot `slot`, device lanes (lanes_out) or the peer exchange.
static RoundOut round_out(jb_ctx* c, void* lanes_out, int slot, uint64_t* seq_out) {
    RoundOut ro;
    ro.partial = nullptr;  // set by launch_round
    ro.counter = c->d_counter;
    ro.lanes = lanes_out ? 1 : 0;
    ro.world = 1;
    ro.rank = 0;
    ro.xseq = 0;
    ro.timeout_cycles = 0;
    for (int g2 = 0; g2 < 16; ++g2) ro.peer[g2] = nullptr;
    ro.seq = ++c->result_seq;
    if (seq_out) *seq_out = ro.seq;
    uint64_t* slot_dev = c->d_result_alias + (size_t)slot * JB_SLOT_U64;
    if (lanes_out == JB_LANES_EXCHANGE) {  // fused all-reduce over peer memory, totals (lanes) to the host
        ro.lanes = 2;
        ro.result = slot_dev;
        ro.flag = slot_dev + 64;
        for (int g2 = 0; g2 < 16; ++g2) ro.peer[g2] = c->xch_peer[g2];
        ro.world = c->world;
        ro.rank = c->rank;
        ro.xseq = ++c->xch_seq;
        ro.timeout_cycles = 20000000000LL;
    } else if (lanes_out) {
        ro.result = (uint64_t*)lanes_out;
        ro.flag = nullptr;
    } else {
        ro.result = slot_dev;
        ro.flag = slot_dev + 64;
    }
    return ro;
}

static int member_round(jb_member* mem, const uint64_t* bind, bool skip1, void* lanes_out, const EqRound* eqr = nullptr,
                        int slot = 0, uint64_t* seq_out = nullptr) {
    jb_ctx* c = mem->ctx;
    bool do_bind = bind != nullptr;
    bool hi4 = false;
    BindScalar s;
    std::memset(&s, 0, sizeof s);
    size_t len = mem->len;
    if (do_bind) {
        if (!canonical_fr(bind)) return c->fail(JB_ERR_INVALID, "prove_round: challenge limbs not canonical");
        if (len < 4) return c->fail(JB_ERR_INVALID, "prove_round: no round left after this bind (use finish_rounds)");
        s = make_scalar(bind, &hi4);
        len /= 2;
    } else if (len < 2) {
        return c->fail(JB_ERR_INVALID, "prove_round: member is fully bound");
    }
    size_t pairs = len / 2;
    TablePtrs tp;
    std::memset(&tp, 0, sizeof tp);
    const int T = mem->ntables();
    const bool from_src = !mem->src.empty();
    auto is_src = [&](int j) { return from_src && mem->src[j].type != JB_SOURCE_TABLE; };
    const uint64_t* ins[JB_PRODUCT_MAX_FACTORS];  // (a product member has up to 16 tables, TablePtrs holds 8)
    uint64_t* outs[JB_PRODUCT_MAX_FACTORS];
    for (int j = 0; j < T; ++j) {
        Table& t = mem->tables[j];
        ins[j] = t.buf;
        outs[j] = t.buf;
        if (is_src(j)) {  // read from its column; the bind writes the len/2 buffer allocated at creation
            ins[j] = nullptr;
            continue;
        }
        if (do_bind && mem->order == JB_LOW_TO_HIGH) {
            int st = c->ensure_alt(t, len);
            if (st != JB_OK) return st;
            outs[j] = t.alt;
        }
    }
    if (mem->kind != MemberKind::Product)
        for (int j = 0; j < T; ++j) {
            tp.in[j] = ins[j];
            tp.out[j] = outs[j];
        }
    if (eqr) {
        tp.e_out = eqr->e_out;
        tp.e_in = eqr->e_in;
        tp.in_bits = eqr->in_bits;
    }
    const RoundOut ro = round_out(c, lanes_out, slot, seq_out);
    int st;
    if (mem->kind == MemberKind::Product)
        st = product_round(c, mem, ins, outs, eqr, eqr ? true : skip1, pairs, do_bind, hi4, s, ro);
    else if (mem->kind == MemberKind::Dense)
        st = eqr ? dispatch_weighted(c, mem->m, mem->order, tp, pairs, do_bind, hi4, s, ro)
                 : dispatch_fused(c, mem->m, mem->terms, mem->order, skip1, tp, pairs, do_bind, hi4, s, ro);
    else  // Expr, and a ReadWrite member's address rounds (a Booleanity member has passes of its own)
        st = dispatch_expr(c, mem, eqr != nullptr, eqr ? true : skip1, tp, pairs, do_bind, hi4, s, ro);
    if (st != JB_OK) return st;
    if (do_bind) {
        for (int j = 0; j < T; ++j) {
            if (mem->order == JB_LOW_TO_HIGH && !is_src(j)) mem->tables[j].swap_buffers();
            mem->tables[j].len = len;
        }
        mem->len = len;
        if (from_src) sources_release(mem);  // (stream-ordered: the columns are freed after the pass has read them)
    }
    return JB_OK;
}

// Spin until the last block of the launch that took sequence number `want` has published into `slot`.
static int wait_round_result(jb_ctx* c, int slot, uint64_t want) {
    WaitAcc acc_(c);
    volatile uint64_t* flag = c->h_result + (size_t)slot * JB_SLOT_U64 + 64;
    uint64_t spins = 0;
    while (*flag != want) {
        if ((++spins & 0xfffff) == 0) {  // every ~1M spins make sure the stream has not died
            cudaError_t e = cudaStreamQuery(c->stream);
            if (e != cudaSuccess && e != cudaErrorNotReady) return c->check(e, "round kernel failed");
            if (e == cudaSuccess && *flag != want) return c->fail(JB_ERR_CUDA, "round kernel finished without publishing its result");
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    __atomic_thread_fence(__ATOMIC_ACQUIRE);
    return JB_OK;
}
static int wait_round_result0(jb_ctx* c) { return wait_round_result(c, 0, c->result_seq); }

static int sharded_prove_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim,
                               uint64_t* out_evals);
static int resident_values(int D, const uint64_t* lanes, uint64_t* vals);

static int eq_prove_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals);

struct RoundConsts {
    HostFr w[JB_PRODUCT_MAX_FACTORS], ipow[JB_PRODUCT_MAX_FACTORS], mpow;
    HostFr next[JB_PRODUCT_MAX_FACTORS + 1];  // q(M+1) = sum_{i<=M} next_i q(i) for deg q <= M: (-1)^(M-i) C(M+1, i)
};
// M in 1..16: products of up to 16 tables, expression members up to degree 6 (jb_round_evals_from_kernel_values stays
// at 4). The binomials come from Pascal's triangle (C(17, 8) = 24310 at most).
static const RoundConsts& round_consts(int M) {
    static RoundConsts table[JB_PRODUCT_MAX_FACTORS + 1];
    static const bool init = [] {
        constexpr int N = JB_PRODUCT_MAX_FACTORS + 2;
        uint64_t binom[N][N] = {{0}};
        for (int n = 0; n < N; ++n) {
            binom[n][0] = 1;
            for (int i = 1; i <= n; ++i) binom[n][i] = binom[n - 1][i - 1] + (i < n ? binom[n - 1][i] : 0);
        }
        for (int m = 1; m <= JB_PRODUCT_MAX_FACTORS; ++m) {
            for (int i = 0; i <= m; ++i) {
                const HostFr b = HostFr::from_u64(binom[m + 1][i]);
                table[m].next[i] = ((m - i) & 1) ? HostFr::zero() - b : b;
            }
            for (int i = 0; i < m; ++i) {
                HostFr ti = HostFr::one();  // i^m
                for (int e = 0; e < m; ++e) ti = ti * HostFr::from_u64((uint64_t)i);
                table[m].ipow[i] = ti;
                const HostFr b = HostFr::from_u64(binom[m][i]);
                table[m].w[i] = ((m - 1 - i) & 1) ? HostFr::zero() - b : b;
            }
            HostFr tm = HostFr::one();  // m^m
            for (int e = 0; e < m; ++e) tm = tm * HostFr::from_u64((uint64_t)m);
            table[m].mpow = tm;
        }
        return true;
    }();
    (void)init;
    return table[M];
}

// Assembles s(0..M) from the K published values. Kernel order: s(0), [s(1)], s(2..M-1), s(inf) for
// M >= 2 (s(0), [s(1)] for M == 1); with skip1, s(1) = claim - s(0). s(M) is rebuilt from the leading
// coefficient: q(t) = s(t) - s(inf) t^M has degree < M, so q(M) = sum_{i<M} (-1)^(M-1-i) C(M,i) q(i).
// In verify mode the claim is checked (naive.rs:301-308).
static int assemble_evals(jb_ctx* c, int M, bool skip1, const uint64_t* vals, const uint64_t* claim, size_t round,
                          uint64_t* out_evals) {
    HostFr ev[JB_PRODUCT_MAX_FACTORS + 1];
    int k = 0;
    ev[0] = HostFr::from_limbs(vals + 4 * k++);
    if (skip1) ev[1] = HostFr::from_limbs(claim) - ev[0];
    else ev[1] = HostFr::from_limbs(vals + 4 * k++);
    if (M >= 2) {
        for (int t = 2; t < M; ++t) ev[t] = HostFr::from_limbs(vals + 4 * k++);
        const HostFr lead = HostFr::from_limbs(vals + 4 * k++);
        // s(M) = sum_{i<M} w_i (s(i) - lead i^M) + lead M^M with w_i = (-1)^(M-1-i) C(M,i); the constants are built
        // once (this runs on the Fiat-Shamir round trip of every round)
        const RoundConsts& rc = round_consts(M);
        HostFr qM = HostFr::zero();
        for (int i = 0; i < M; ++i) qM = qM + rc.w[i] * (ev[i] - lead * rc.ipow[i]);
        ev[M] = qM + lead * rc.mpow;
    }
    for (int t = 0; t <= M; ++t) ev[t].store(out_evals + 4 * t);
    if (claim && !skip1 && (ev[0] + ev[1]) != HostFr::from_limbs(claim)) {
        char buf[96];
        std::snprintf(buf, sizeof buf, "RoundCheckFailed { round: %zu }", round);
        return c ? c->fail(JB_ERR_ROUND_CHECK, buf) : (int)JB_ERR_ROUND_CHECK;
    }
    return JB_OK;
}

// The kernel values of a degree-M round in a result slot: the first 16 lie below the slot's sequence flag (word 64),
// any further ones from word 72 (publish_round's SPLIT); they are copied together into buf when there are more.
static const uint64_t* slot_values(const uint64_t* slot, int M, bool skip1, uint64_t* buf) {
    const int k = M == 1 ? (skip1 ? 1 : 2) : (skip1 ? M : M + 1);
    if (k <= 16) return slot;
    std::memcpy(buf, slot, 64 * 8);
    std::memcpy(buf + 64, slot + 72, (size_t)(k - 16) * 32);
    return buf;
}

// One round through a launched pass: binds `bind` (if given), sweeps into result slot 0, waits for it and assembles
// s(0..m). The caller counts the round.
static int launched_round(jb_member* mem, const uint64_t* bind, bool skip1, const uint64_t* claim, size_t round,
                          uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    int st = member_round(mem, bind, skip1, nullptr);
    if (st == JB_OK) st = wait_round_result0(c);
    if (st != JB_OK) return st;
    uint64_t vals[JB_MAX_ROUND_EVALS * 4];
    return assemble_evals(c, mem->m, skip1, slot_values(c->h_result, mem->m, skip1, vals), claim, round, out_evals);
}

int jb_round_evals_from_kernel_values(int m, int skip_t1, const uint64_t* kernel_values, const uint64_t* claim_or_null,
                                      uint64_t* out_evals) {
    if (!kernel_values || !out_evals || m < 1 || m > 4) return JB_ERR_INVALID;
    if (skip_t1 && !claim_or_null) return JB_ERR_INVALID;
    const int k = m == 1 ? (skip_t1 ? 1 : 2) : (skip_t1 ? m : m + 1);
    for (int t = 0; t < k; ++t)
        if (!canonical_fr(kernel_values + 4 * t)) return JB_ERR_INVALID;
    if (claim_or_null && !canonical_fr(claim_or_null)) return JB_ERR_INVALID;
    return assemble_evals(nullptr, m, skip_t1 != 0, kernel_values, claim_or_null, 0, out_evals);
}

// ---- rounds served by a resident kernel -----------------------------------------------------------------
// K canonical kernel values (s(0), [s(2..D-1)], s(inf)) of one member from an answer's lanes.
static void answer_values(const jb_member* mem, const ResConsumed& info, const uint64_t* lanes, uint64_t* vals) {
    if (info.thin) {  // s(0) = S0 + S6, s(inf) = S2 + S7: add the integer lanes, reduce once each
        uint64_t sum[2 * 17];
        for (int w = 0; w < 17; ++w) {
            sum[w] = lanes[0 * 17 + w] + lanes[6 * 17 + w];
            sum[17 + w] = lanes[2 * 17 + w] + lanes[7 * 17 + w];
        }
        jb_wide_lanes_reduce_host(sum, 2, vals);
    } else {
        resident_values(mem->m, lanes, vals);
    }
}

// A thin answer also determines the NEXT round's polynomial as a function of the challenge that round binds.
static void harvest_lookahead(jb_member* mem, const ResConsumed& info, const uint64_t* lanes) {
    if ((info.act == RES_ACT_EVAL || info.act == RES_ACT_BIND_EVAL || info.act == RES_ACT_BIND2_EVAL) && info.thin &&
        info.nprime >= 4 && mem->ctx->lookahead) {
        jb_wide_lanes_reduce_host(lanes, 6, mem->look);
        mem->look_ok = true;
        mem->look_round = info.round + 1;
    } else if (info.act != RES_ACT_NONE) {
        mem->look_ok = false;
    }
}

// s(0)(r) = S0 + r (S1 - S0 - S2) + r^2 S2 and s(inf)(r) = S3 + r (S4 - S3 - S5) + r^2 S5 at the drawn challenge
static void lookahead_values(const jb_member* mem, const uint64_t* r_limbs, uint64_t* vals) {
    const HostFr r = HostFr::from_limbs(r_limbs);
    for (int h = 0; h < 2; ++h) {
        const HostFr a0 = HostFr::from_limbs(mem->look + (3 * h) * 4), a1 = HostFr::from_limbs(mem->look + (3 * h + 1) * 4),
                     lead = HostFr::from_limbs(mem->look + (3 * h + 2) * 4);
        ((lead * r + (a1 - a0 - lead)) * r + a0).store(vals + 4 * h);
    }
}

struct RunItem {
    jb_member* mem;
    const uint64_t* bind;   // null on the member's first round
    const uint64_t* claim;  // the running claim (s(1) = claim - s(0))
    size_t round;
    uint64_t* out_evals;
};

// One round of `n` members of one run: ONE mailbox command. Members whose previous answer carried lookahead sums
// are answered at once from those (their command stays in flight: the device's bind + next sums overlap the
// caller's Fiat-Shamir step); the others wait for this command's own answer.
//
// Large rounds of staged runs are folded (res_fusable): a first round over such tables returns lookahead sums
// (RES_FLAG_LOOK); the round after it is answered from them with NO command, its challenge left pending on the
// members; the next command binds the pending challenge and its own in one pass (RES_ACT_BIND2_EVAL) and again
// returns lookahead sums, so a round after it that is still large is skipped the same way. A round is skipped only
// when every member of the run takes part, in the same state: then every pending challenge of a run is the same one.
static int run_round(jb_ctx* c, ResidentRun* run, RunItem* items, int n, const uint64_t* shared_bind, bool exchange,
                     bool gather = false) {
    jb_member* mems[RES_MAX_MEMBERS];
    const int rn = run->n;
    for (int i = 0; i < rn; ++i) mems[i] = run->mem[i];
    const bool fuse = run->fuse && !exchange && !gather;
    bool skip = fuse && n == rn && resident_inflight(run) == 0, look = fuse;
    for (int i = 0; i < n; ++i) {
        const jb_member* m = items[i].mem;
        if (!items[i].bind) {
            skip = false;
            look = look && res_fusable(m->len);
        } else {
            skip = skip && !m->pend && m->look_ok && m->look_round == items[i].round && res_fusable(m->len) &&
                   m->len == items[0].mem->len;
        }
    }
    if (skip) {
        for (int i = 0; i < n; ++i) {
            jb_member* m = items[i].mem;
            uint64_t vals[JB_MAX_EVALS * 4];
            lookahead_values(m, items[i].bind, vals);
            m->look_ok = false;
            m->pend = true;
            std::memcpy(m->pend_r, items[i].bind, 32);
            int st = assemble_evals(c, m->m, true, vals, items[i].claim, items[i].round, items[i].out_evals);
            if (st != JB_OK) return st;
            m->rounds_done++;
        }
        return JB_OK;
    }
    unsigned actions[RES_MAX_MEMBERS] = {0};
    const uint64_t* pending = nullptr;
    for (int i = 0; i < n; ++i) {
        jb_member* m = items[i].mem;
        if (m->pend) pending = m->pend_r;
        actions[m->run_idx] = !items[i].bind ? RES_ACT_EVAL : m->pend ? RES_ACT_BIND2_EVAL : RES_ACT_BIND_EVAL;
    }
    int st = resident_post(run, actions, shared_bind, exchange, gather, pending, look);
    if (st != JB_OK) return st;
    uint64_t out[RES_MAX_MEMBERS * RES_SLOT_U64];
    ResConsumed info[RES_MAX_MEMBERS];
    bool lost = false;
    while (!lost && resident_inflight(run) > 1) {  // the previous command's answer: it carries this round's lookahead
        st = resident_consume(run, out, info);
        if (st == JB_RES_LOST) lost = true;
        else if (st != JB_OK) return st;
        else for (int i = 0; i < rn; ++i) harvest_lookahead(mems[i], info[i], out + (size_t)i * RES_SLOT_U64);
    }
    uint64_t vals[RES_MAX_MEMBERS][JB_MAX_EVALS * 4];
    bool hit[RES_MAX_MEMBERS], need_now = false;
    for (int i = 0; i < n && !lost; ++i) {
        jb_member* m = items[i].mem;
        hit[i] = c->lookahead && items[i].bind && m->look_ok && m->look_round == items[i].round && m->m == 2;
        if (hit[i]) lookahead_values(m, items[i].bind, vals[i]);
        else need_now = true;
    }
    if (need_now && !lost) {
        st = resident_consume(run, out, info);  // (cannot release the run: the members of this round are not fully bound)
        if (st == JB_RES_LOST) lost = true;
        else if (st != JB_OK) return st;
    }
    if (lost) {
        // the kernel gave up waiting (the host was held up): replay the unexecuted binds with launches and compute
        // this round's sums with one eval-only launch per member - the proof is unchanged, only slower
        st = resident_recover(run);
        if (st != JB_OK) return st;
        for (int i = 0; i < n; ++i) {
            st = launched_round(items[i].mem, nullptr, true, items[i].claim, items[i].round, items[i].out_evals);
            if (st != JB_OK) return st;
            items[i].mem->rounds_done++;
        }
        return JB_OK;
    }
    if (need_now) {
        for (int i = 0; i < n; ++i)
            if (!hit[i]) {
                const int idx = items[i].mem->run_idx;
                answer_values(items[i].mem, info[idx], out + (size_t)idx * RES_SLOT_U64, vals[i]);
            }
        for (int i = 0; i < rn; ++i) harvest_lookahead(mems[i], info[i], out + (size_t)i * RES_SLOT_U64);
    }
    for (int i = 0; i < n; ++i) {
        jb_member* m = items[i].mem;
        st = assemble_evals(c, m->m, true, vals[i], items[i].claim, items[i].round, items[i].out_evals);
        if (st != JB_OK) return st;
        m->rounds_done++;
    }
    return JB_OK;
}

// This round of one member through its resident kernel (starting one if the member is eligible). Returns
// JB_ERR_UNSUPPORTED if the member is not served by a run: the caller launches instead.
static int resident_member_prove(jb_member* mem, const uint64_t* bind, const uint64_t* claim, size_t round, bool exchange,
                                 uint64_t* out_evals, bool gather = false) {
    jb_ctx* c = mem->ctx;
    if (!mem->run) {
        if (!resident_eligible(mem)) return JB_ERR_UNSUPPORTED;
        jb_member* one[1] = {mem};
        int st = resident_begin(c, one, 1);
        if (st != JB_OK) return st;
    }
    RunItem it{mem, bind, claim, round, out_evals};
    int st = run_round(c, mem->run, &it, 1, bind, exchange, gather);
    if (st != JB_OK && mem->run) resident_end(mem->run, true);
    return st;
}

// The terminal bind of one member through its run (the run is released when every member is fully bound).
static int resident_member_final(jb_member* mem, const uint64_t* bind) {
    unsigned actions[RES_MAX_MEMBERS] = {0};
    actions[mem->run_idx] = RES_ACT_FINAL;
    int st = resident_round(mem->run, actions, bind, false, nullptr);
    if (st == JB_RES_LOST) return resident_recover(mem->run);  // (replays the terminal bind with a launch)
    if (st != JB_OK && mem->run) resident_end(mem->run, true);
    return st;
}

// Stops whatever resident kernel would be in the way of a launch for this member.
static void before_launch(jb_member* mem) {
    if (mem->run) resident_end(mem->run, true);
    mem->ctx->quiesce_resident(false);
}

// The checks of a round's arguments that every entry point makes first, in this order (context lock held).
static int check_round_args(jb_member* mem, const uint64_t* bind, size_t round) {
    jb_ctx* c = mem->ctx;
    if (round != mem->rounds_done) return c->fail(JB_ERR_INVALID, "prove_round: round index out of sequence");
    if ((mem->rounds_done == 0) != (bind == nullptr))
        return c->fail(JB_ERR_INVALID, "prove_round: bind must be absent exactly on the first round");
    if (bind && !canonical_fr(bind)) return c->fail(JB_ERR_INVALID, "prove_round: challenge limbs not canonical");
    return JB_OK;
}

int jb_member_prove_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim,
                          uint64_t* out_evals) {
    if (!mem || !out_evals) return JB_ERR_INVALID;
    jb_ctx* c = mem->ctx;
    if (mem->sharded) {
        int st = sharded_prove_round(mem, bind, round, claim, out_evals);
        if (st == JB_OK) mem->rounds_done++;
        return st;
    }
    Guard g(c, true);
    int st = check_round_args(mem, bind, round);
    if (st != JB_OK) return st;
    if (mem->len < (bind ? 4u : 2u))
        return c->fail(JB_ERR_INVALID, bind ? "prove_round: no round left after this bind (use finish_rounds)"
                                            : "prove_round: member is fully bound");
    if (eq_rounds(mem)) {
        before_launch(mem);
        st = eq_prove_round(mem, bind, round, claim, out_evals);
        if (st == JB_OK) mem->rounds_done++;
        return st;
    }
    // With a claim and round verification off (the default, = the reference's optimized tier) the
    // kernel skips t = 1 and s(1) = claim - s(0); with verification on (or no claim) it computes
    // every point and the claim, if given, is checked (the reference tier, naive.rs:301-308).
    const bool skip1 = claim != nullptr && !c->verify_rounds;
    if (skip1) {
        // the resident kernel serves this and every later round of the member: no launch per round
        st = resident_member_prove(mem, bind, claim, round, false, out_evals);  // (counts the round itself)
        if (st != JB_ERR_UNSUPPORTED) return st;
    }
    before_launch(mem);
    st = launched_round(mem, bind, skip1, claim, round, out_evals);
    if (st == JB_OK) mem->rounds_done++;
    return st;
}

// ---- split-eq member: one round ------------------------------------------------------------------------
// scalar <- scalar * eq(w_v, r) for the variable v just bound (GruenSplitEqPolynomial::bind, split_eq.rs:347-352)
static void eq_absorb_coord(jb_member* mem, const uint64_t* w, const uint64_t* r) {
    HostFr wv = HostFr::from_limbs(w), rr = HostFr::from_limbs(r);
    HostFr prod = wv * rr;
    HostFr f = HostFr::one() - wv - rr + prod + prod;
    (HostFr::from_limbs(mem->eq_scalar) * f).store(mem->eq_scalar);
}
static void eq_absorb_bind(jb_member* mem, size_t var, const uint64_t* r) { eq_absorb_coord(mem, mem->eq_w.data() + 4 * var, r); }

static int rw_address_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals);
static int rw_key_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals);
static int rw_end_keys(jb_member* mem, const uint64_t r[4]);
static int bool_address_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals);
static int eq_round_tail(jb_member* mem, const HostFr& l0, const HostFr& l1, const uint64_t* claim, size_t round,
                         uint64_t* out_evals);

// The split-eq weights of LowToHigh cycle round `round` (its variable w[n - 1 - round] is the pair index's lowest).
static EqRound eq_weights_l2h(const jb_member* mem, size_t round) {
    EqRound er;
    const size_t cur = mem->eq_n - round;  // unbound variables including the current one (index cur - 1)
    const size_t head = cur - 1;
    const size_t out_bits = head < mem->eq_split ? head : mem->eq_split;
    const size_t in_bits = head - out_bits;
    er.e_out = mem->eq_tabs + 4 * (((size_t)1 << out_bits) - 1);
    er.e_in = mem->eq_tabs + 4 * (mem->eq_in_base + ((size_t)1 << in_bits) - 1);
    er.in_bits = (int)in_bits;
    return er;
}

static int eq_prove_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    if (!claim) return c->fail(JB_ERR_INVALID, "eq member: the running claim is required (Gruen hint s(0)+s(1))");
    const size_t n = mem->eq_n;
    if (mem->kind == MemberKind::ReadWrite) {
        const RwState& rw = *mem->rw;
        if (rw.p == n && round >= n) return rw_address_round(mem, bind, round, claim, out_evals);
        if (rw.p < n && round >= rw.p) {  // mixed order: the address rounds, then cycle round p onwards
            if (round < rw.p + rw.kappa) return rw_key_round(mem, bind, round, claim, out_evals);
            if (round == rw.p + rw.kappa && bind) {  // the last address variable: the dense tables take over
                const int st = rw_end_keys(mem, bind);
                if (st != JB_OK) return st;
                bind = nullptr;
            }
            round -= rw.kappa;
        }
    }
    if (mem->kind == MemberKind::Booleanity) {  // the address rounds come first; the cycle rounds are its eq rounds
        const size_t ka = mem->bl->log_k;
        if (round < ka) return bool_address_round(mem, bind, round, claim, out_evals);
        if (round == ka && bind) {  // the last address variable
            eq_absorb_coord(mem, bool_addr_coord(*mem->bl, ka - 1), bind);
            const int st = bool_begin_cycles(mem, bind);
            if (st != JB_OK) return st;
            bind = nullptr;
        }
        round -= ka;
    }
    if (round >= n) return c->fail(JB_ERR_INVALID, "prove_round: member is fully bound");
    const bool l2h = mem->order == JB_LOW_TO_HIGH;
    if (bind) {
        if (!canonical_fr(bind)) return c->fail(JB_ERR_INVALID, "prove_round: challenge limbs not canonical");
        eq_absorb_bind(mem, l2h ? n - round : round - 1, bind);  // the previous round's variable
    }
    EqRound er;
    size_t cur_var;
    if (l2h) {
        er = eq_weights_l2h(mem, round);
        cur_var = n - round - 1;
    } else {
        // HighToLow (split_eq.rs:233-257): the current variable is w[round]; the remaining ones w[round + 1 .. n)
        // are the pair index MSB-first: the unbound suffix of in_point = w[1 .. 1 + s) on top of out_point =
        // w[1 + s .. n) (evals_cached_rev: suffix tables), then suffixes of out_point alone
        const size_t sp = mem->eq_split;  // s = |in_point|
        const size_t nlo = n - 1 - sp;    // |out_point|
        const size_t hi_k = round < sp ? round : sp;          // hi table: eq(w[1 + hi_k .. 1 + s))
        const size_t lo_k = round < sp ? 0 : round - sp;      // lo table: eq(w[1 + s + lo_k .. n))
        er.e_out = mem->eq_tabs + 4 * mem->eq_hi_off[hi_k];
        er.e_in = mem->eq_tabs + 4 * mem->eq_lo_off[lo_k];
        er.in_bits = (int)(nlo - lo_k);
        cur_var = round;
    }
    // the current variable's linear factor l(t) = l0 + t (l1 - l0) is known before the pass runs
    const HostFr scalar = HostFr::from_limbs(mem->eq_scalar);
    const HostFr wc = HostFr::from_limbs(mem->eq_w.data() + 4 * cur_var);
    const HostFr l1 = scalar * wc, l0 = scalar - l1;
    if (l1.is_zero()) return c->fail(JB_ERR_INVALID, "eq member: current eq evaluation at one must be invertible");
    int st = mem->kind == MemberKind::ReadWrite && mem->rw->cycles
                 ? rw_cycle_round(mem, bind, er, round_out(c, nullptr, 0, nullptr))
             : mem->kind == MemberKind::Booleanity ? bool_cycle_pass(mem, bind, er, round_out(c, nullptr, 0, nullptr))
                                                   : member_round(mem, bind, true, nullptr, &er);
    if (st != JB_OK) return st;
    return eq_round_tail(mem, l0, l1, claim, round, out_evals);
}

// The host half of a split-eq round whose pass is in flight: waits for q(0), q(2) .. q(M-1), q(inf) in result slot 0,
// takes q(1) from the claim, s(t) = l(t) q(t) for t = 0 .. M + 1 with l(t) = l0 + t (l1 - l0) (l1 invertible).
static int eq_round_tail(jb_member* mem, const HostFr& l0, const HostFr& l1, const uint64_t* claim, size_t round,
                         uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    const size_t M = (size_t)mem->m;
    // a field inversion is ~400 host multiplications (~13 us): do it while the device runs the pass (the
    // extrapolation constants below are built once)
    const HostFr l1_inv = l1.inverse();
    const RoundConsts& rc = round_consts((int)M);
    int st = wait_round_result0(c);
    if (st != JB_OK) return st;
    // kernel order: q(0), q(2), .., q(M-1), q(inf)   (M <= 16 values; q(0) only for M == 1)
    const HostFr q0 = HostFr::from_limbs(c->h_result);
    const HostFr q1 = (HostFr::from_limbs(claim) - l0 * q0) * l1_inv;
    uint64_t vals[JB_MAX_ROUND_EVALS * 4], qe[JB_MAX_ROUND_EVALS * 4];
    q0.store(vals);
    q1.store(vals + 4);
    if (M > 1) std::memcpy(vals + 8, c->h_result + 4, (M - 1) * 32);
    st = assemble_evals(c, (int)M, false, vals, nullptr, round, qe);  // q(0..M)
    if (st != JB_OK) return st;
    // q(M+1) by extrapolation (degree M: the (M+1)-th difference vanishes), then s(t) = l(t) q(t), t = 0..M+1
    HostFr qv[JB_PRODUCT_MAX_FACTORS + 2];
    qv[M + 1] = HostFr::zero();
    for (size_t t = 0; t <= M; ++t) {
        qv[t] = HostFr::from_limbs(qe + 4 * t);
        qv[M + 1] = qv[M + 1] + rc.next[t] * qv[t];
    }
    const HostFr dl = l1 - l0;
    HostFr lt = l0;
    for (size_t t = 0; t <= M + 1; ++t) {
        (lt * qv[t]).store(out_evals + 4 * t);
        lt = lt + dl;
    }
    return JB_OK;
}

// Makes a new member split-eq weighted by eq(w, x) * scale: the host state and the prefix / suffix eq tables of its
// order. w, nvars (== the member's rounds) and the scale have been checked. On failure the member is destroyed.
static int eq_setup(jb_member* mem, const uint64_t* w, size_t nvars, const uint64_t* scale_or_null, jb_member** out) {
    jb_ctx* c = mem->ctx;
    const int order = mem->order;
    int st = JB_OK;
    {
    Guard g(c);
    mem->eq = true;
    mem->eq_n = nvars;
    mem->eq_split = nvars / 2;
    mem->eq_w.assign(w, w + 4 * nvars);
    HostFr sc = scale_or_null ? HostFr::from_limbs(scale_or_null) : HostFr::one();
    sc.store(mem->eq_scalar);
    if (order == JB_LOW_TO_HIGH) {
        // prefix tables (EqPolynomial::evals_cached, eq.rs:322-340): Eo[k] over w[0..k), Ei[k] over w[split..split+k)
        const size_t split = mem->eq_split, nin = nvars - 1 - (split < nvars - 1 ? split : nvars - 1);
        const size_t out_max = split < nvars - 1 ? split : nvars - 1;
        mem->eq_in_base = ((size_t)2 << out_max) - 1;
        const size_t total = mem->eq_in_base + ((size_t)2 << nin) - 1;
        st = c->dev_alloc((void**)&mem->eq_tabs, total * 32);
        for (size_t k = 0; k <= out_max && st == JB_OK; ++k)
            st = eq_build(c, w, k, nullptr, mem->eq_tabs + 4 * (((size_t)1 << k) - 1));
        for (size_t k = 0; k <= nin && st == JB_OK; ++k)
            st = eq_build(c, w + 4 * split, k, nullptr, mem->eq_tabs + 4 * (mem->eq_in_base + ((size_t)1 << k) - 1));
    } else {
        // HighToLow (split_eq.rs:233-257): tail = w[1..], in_point = tail[..s], out_point = tail[s..] with
        // s = min(n / 2, n - 1); suffix tables (evals_cached_rev): hi[k] = eq(w[1 + k .. 1 + s)), lo[j] = eq(w[1 + s + j .. n))
        const size_t sp = mem->eq_split < nvars - 1 ? mem->eq_split : nvars - 1;
        mem->eq_split = sp;
        const size_t nlo = nvars - 1 - sp;
        size_t total = 0;
        for (size_t k = 0; k <= sp; ++k) {
            mem->eq_hi_off.push_back(total);
            total += (size_t)1 << (sp - k);
        }
        for (size_t j = 0; j <= nlo; ++j) {
            mem->eq_lo_off.push_back(total);
            total += (size_t)1 << (nlo - j);
        }
        st = c->dev_alloc((void**)&mem->eq_tabs, total * 32);
        for (size_t k = 0; k <= sp && st == JB_OK; ++k)
            st = eq_build(c, w + 4 * (1 + k), sp - k, nullptr, mem->eq_tabs + 4 * mem->eq_hi_off[k]);
        for (size_t j = 0; j <= nlo && st == JB_OK; ++j)
            st = eq_build(c, w + 4 * (1 + sp + j), nlo - j, nullptr, mem->eq_tabs + 4 * mem->eq_lo_off[j]);
    }
    }  // the context lock is released before the member is torn down (jb_member_destroy takes it)
    if (st != JB_OK) {
        jb_member_destroy(mem);
        *out = nullptr;
    }
    return st;
}

int jb_eq_member_create(jb_ctx* c, const jb_table* handles, size_t m, const uint64_t* w, size_t nvars,
                        const uint64_t* scale_or_null, int order, jb_member** out) {
    if (!c || !handles || !w || !out) return JB_ERR_INVALID;
    if (order != JB_LOW_TO_HIGH && order != JB_HIGH_TO_LOW) return c->fail(JB_ERR_INVALID, "eq member: unknown binding order");
    if (m < 1 || m > 3) return c->fail(JB_ERR_UNSUPPORTED, "eq member: m must be 1..3");
    for (size_t i = 0; i < nvars; ++i)
        if (!canonical_fr(w + 4 * i)) return c->fail(JB_ERR_INVALID, "eq member: point limbs not canonical");
    if (scale_or_null && !canonical_fr(scale_or_null)) return c->fail(JB_ERR_INVALID, "eq member: scale not canonical");
    int st = jb_member_create(c, handles, m, order, out);
    if (st != JB_OK) return st;
    jb_member* mem = *out;
    if (mem->rounds != nvars || nvars == 0) {
        jb_member_destroy(mem);
        *out = nullptr;
        return c->fail(JB_ERR_INVALID, "eq member: point length must equal log2(table length) >= 1");
    }
    return eq_setup(mem, w, nvars, scale_or_null, out);
}

// ---- expression member ---------------------------------------------------------------------------------
// The checks on the expression shared by both constructors (context lock held): D = the largest monomial degree;
// blocks = unit coefficients, every monomial of one degree, tables in consecutive blocks.
static int check_expr(jb_ctx* c, size_t ntables, const jb_monomial* monomials, size_t nmonomials,
                      const uint64_t* eq_w_or_null, size_t nvars, const uint64_t* eq_scale_or_null, int order, int* D_out,
                      bool* blocks_out) {
    int D = 0;
    bool blocks = true;
    if (ntables > JB_EXPR_MAX_TABLES || nmonomials > JB_EXPR_MAX_MONOMIALS)
        return c->fail(JB_ERR_UNSUPPORTED, "expr member: at most JB_EXPR_MAX_TABLES tables and JB_EXPR_MAX_MONOMIALS monomials");
    if (ntables == 0 || nmonomials == 0) return c->fail(JB_ERR_INVALID, "expr member: no tables or no monomials");
    if (order != JB_HIGH_TO_LOW && order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "expr member: unknown order");
    const HostFr one = HostFr::one();
    bool used[JB_EXPR_MAX_TABLES] = {false};
    for (size_t k = 0; k < nmonomials; ++k) {
        const jb_monomial& mo = monomials[k];
        if (mo.degree == 0) return c->fail(JB_ERR_INVALID, "expr member: a monomial of degree 0 (constant summands are not supported)");
        if (mo.degree > JB_EXPR_MAX_DEGREE) return c->fail(JB_ERR_UNSUPPORTED, "expr member: monomial degree above JB_EXPR_MAX_DEGREE");
        if (!canonical_fr(mo.coeff)) return c->fail(JB_ERR_INVALID, "expr member: coefficient limbs not canonical");
        for (uint32_t i = 0; i < mo.degree; ++i) {
            if (mo.table[i] >= ntables) return c->fail(JB_ERR_INVALID, "expr member: table index out of range");
            if (mo.table[i] != k * monomials[0].degree + i) blocks = false;
            used[mo.table[i]] = true;
        }
        if (mo.degree != monomials[0].degree || HostFr::from_limbs(mo.coeff) != one) blocks = false;
        D = std::max(D, (int)mo.degree);
    }
    for (size_t j = 0; j < ntables; ++j)
        if (!used[j]) return c->fail(JB_ERR_INVALID, "expr member: a table no monomial uses");
    if (ntables != nmonomials * monomials[0].degree) blocks = false;
    if (eq_scale_or_null && !eq_w_or_null) return c->fail(JB_ERR_INVALID, "expr member: a scale without an eq point");
    if (eq_w_or_null) {
        for (size_t i = 0; i < nvars; ++i)
            if (!canonical_fr(eq_w_or_null + 4 * i)) return c->fail(JB_ERR_INVALID, "expr member: point limbs not canonical");
        if (eq_scale_or_null && !canonical_fr(eq_scale_or_null))
            return c->fail(JB_ERR_INVALID, "expr member: scale not canonical");
    }
    *D_out = D;
    *blocks_out = blocks;
    return JB_OK;
}

// The kernel parameter form of the checked monomials into mem->ex.
static void make_expr(jb_member* mem, const jb_monomial* monomials, size_t nmonomials, size_t ntables, int D) {
    ExprParams& ex = mem->ex;
    std::memset(&ex, 0, sizeof ex);
    const HostFr one = HostFr::one(), minus_one = HostFr::zero() - one;
    for (size_t k = 0; k < nmonomials; ++k) {
        const jb_monomial& mo = monomials[k];
        const HostFr cf = HostFr::from_limbs(mo.coeff);
        for (int w = 0; w < 4; ++w) {
            ex.coeff[k][2 * w] = (uint32_t)mo.coeff[w];
            ex.coeff[k][2 * w + 1] = (uint32_t)(mo.coeff[w] >> 32);
        }
        for (uint32_t i = 0; i < mo.degree; ++i) ex.table[k][i] = (uint8_t)mo.table[i];
        ex.degree[k] = (uint8_t)mo.degree;
        ex.kind[k] = cf == one ? EXPR_COEFF_ONE : cf == minus_one ? EXPR_COEFF_MINUS_ONE : EXPR_COEFF_GENERAL;
    }
    ex.nmono = (int)nmonomials;
    ex.ntables = (int)ntables;
    ex.D = D;
}

// Everything is checked before anything is allocated. An expression that is exactly a built shape - unit
// coefficients, every table used once, monomials the consecutive blocks [kD, (k+1)D) of a product / sum of products
// (no eq) or a single product of 1..3 tables (eq) - gets that member, so it keeps the resident kernel and the
// specialised passes; anything else gets the expression pass.
int jb_member_create_expr(jb_ctx* c, const jb_table* handles, size_t ntables, const jb_monomial* monomials,
                          size_t nmonomials, const uint64_t* eq_w_or_null, size_t nvars, const uint64_t* eq_scale_or_null,
                          int order, jb_member** out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!handles || !monomials || !out) return JB_ERR_INVALID;
    size_t len = 0;
    int D = 0;
    bool blocks = true;  // unit coefficients, every monomial of one degree, tables in consecutive blocks
    bool own_pass = true;  // the expression pass serves it (else an existing member does)
    {
        Guard g(c);
        int st = check_expr(c, ntables, monomials, nmonomials, eq_w_or_null, nvars, eq_scale_or_null, order, &D, &blocks);
        if (st != JB_OK) return st;
        st = check_tables(c, handles, ntables, &len);
        if (st != JB_OK) return st;
        if (eq_w_or_null && (nvars == 0 || nvars >= 64 || ((size_t)1 << nvars) != len))
            return c->fail(JB_ERR_INVALID, "expr member: point length must equal log2(table length) >= 1");
        own_pass = !blocks || (eq_w_or_null ? !(nmonomials == 1 && D <= 3) : !shape_supported(D, (int)nmonomials));
        if (own_pass) {
            st = adopt_tables(c, MemberKind::Expr, handles, ntables, len, D, 1, order, out);
            if (st != JB_OK) return st;
            make_expr(*out, monomials, nmonomials, ntables, D);
        }
    }
    if (own_pass) return eq_w_or_null ? eq_setup(*out, eq_w_or_null, nvars, eq_scale_or_null, out) : JB_OK;
    if (eq_w_or_null) return jb_eq_member_create(c, handles, (size_t)D, eq_w_or_null, nvars, eq_scale_or_null, order, out);
    return member_create_common(c, handles, (size_t)D, nmonomials, order, out);
}

// ---- expression member over sources ---------------------------------------------------------------------
// The checks on one source (context lock held). log_k: log2 K of a one-hot source. Product members take u32 address
// columns (K <= 2^24), expression members u8 / u16 (K <= 2^16): widest is the widest address kind of the member.
static int check_source(jb_ctx* c, const jb_source& sr, size_t len, int widest, size_t* log_k) {
    if (sr.type == JB_SOURCE_TABLE) {
        const Table* t = c->find(sr.table);
        if (!t) return c->fail(JB_ERR_INVALID, "expr sources: unknown table handle");
        if (t->len != len) return c->fail(JB_ERR_INVALID, "expr sources: a table source of another length");
        return JB_OK;
    }
    if (sr.type != JB_SOURCE_COMPACT && sr.type != JB_SOURCE_ONE_HOT)
        return c->fail(JB_ERR_INVALID, "expr sources: unknown source type");
    if (sr.type == JB_SOURCE_COMPACT) return check_compact_column(c, "expr sources", sr.kind, sr.values, sr.on_device);
    // (here a K above the kind's limit is invalid, not unsupported)
    if (one_hot_kind(sr.kind, widest) && sr.K > one_hot_max_k(sr.kind))
        return c->fail(JB_ERR_INVALID, sr.kind == SK_U32 ? "product sources: K must be a power of two in [1, 2^24]"
                                                         : "expr sources: K must be a power of two in [1, 2^16]");
    const int st = check_one_hot_columns(c, "expr sources", sr.kind, len, sr.K, sr.on_device, &sr.values, 1, widest);
    if (st != JB_OK) return st;
    *log_k = (size_t)log2_of(sr.K);
    if (*log_k && !sr.r_addr) return c->fail(JB_ERR_INVALID, "expr sources: null r_addr");
    for (size_t i = 0; i < *log_k; ++i)
        if (!canonical_fr(sr.r_addr + 4 * i)) return c->fail(JB_ERR_INVALID, "expr sources: r_addr limbs not canonical");
    return JB_OK;
}

// Frees what a failed creation had allocated (context lock held; the table sources were not adopted yet).
static void discard_sources(jb_member* mem) {
    sources_release(mem);
    for (auto& t : mem->tables) mem->ctx->release(t);
    delete mem;
}

// The creation of a member over sources (expression or product): under the context lock, `check` (the relation's own
// checks, which return its status first), then the sources, then everything the rounds need is allocated; check sets
// the member's degree without eq.
}  // extern "C"
template <class Check>
static int create_over_sources(jb_ctx* c, MemberKind kind, const jb_source* sources, size_t nsources, size_t len,
                               const uint64_t* eq_w_or_null, size_t nvars, const uint64_t* eq_scale_or_null, int order,
                               Check check, jb_member** out) {
    jb_member* mem = nullptr;
    int st = JB_OK;
    {
        Guard g(c);
        int D = 0;
        st = check(&D);
        if (st != JB_OK) return st;
        if (len < 2 || (len & (len - 1))) return c->fail(JB_ERR_INVALID, "expr sources: len must be a power of two >= 2");
        if (eq_w_or_null && (nvars >= 64 || ((size_t)1 << nvars) != len))
            return c->fail(JB_ERR_INVALID, "expr member: point length must equal log2(table length) >= 1");
        size_t log_k[JB_PRODUCT_MAX_FACTORS] = {0};
        for (size_t i = 0; i < nsources; ++i) {
            if ((st = check_source(c, sources[i], len, kind == MemberKind::Product ? SK_U32 : SK_U16, &log_k[i])) != JB_OK)
                return st;
            for (size_t k = 0; k < i; ++k)
                if (sources[i].type == JB_SOURCE_TABLE && sources[k].type == JB_SOURCE_TABLE && sources[k].table == sources[i].table)
                    return c->fail(JB_ERR_INVALID, "member: duplicate table handle");
        }
        // everything is allocated here: the columns, the eq tables, the len/2 outputs, the LowToHigh ping-pong buffers
        mem = new_member(c, kind, D, 1, order, len);
        if (!mem) return JB_ERR_OOM;
        mem->tables.resize(nsources);
        mem->src.resize(nsources);
        Scratch scratch(c);
        unsigned int* d_flag = nullptr;
        st = scratch.alloc(sizeof(unsigned int), &d_flag);
        if (st == JB_OK) st = c->check(cudaMemsetAsync(d_flag, 0, sizeof(unsigned int), c->stream), "expr sources: flag memset");
        for (size_t i = 0; i < nsources && st == JB_OK; ++i) {
            const jb_source& sr = sources[i];
            SourceCol& sc = mem->src[i];
            sc.type = sr.type;
            if (sr.type == JB_SOURCE_TABLE) continue;
            sc.kind = sr.kind;
            sc.K = (uint32_t)sr.K;
            Table& t = mem->tables[i];
            st = c->dev_alloc((void**)&t.buf, len / 2 * 32);
            if (st != JB_OK) break;
            t.cap = len / 2;
            t.len = len;
            if (order == JB_LOW_TO_HIGH && (st = c->ensure_alt(t, std::max<size_t>(len / 4, 1))) != JB_OK) break;
            st = copy_column(c, sr.values, len * (size_t)small_kind_bytes(sr.kind), sr.on_device, &sc.values);
            if (st == JB_OK && sr.type == JB_SOURCE_ONE_HOT) st = sources_one_hot_eq(c, sc, len, sr.r_addr, log_k[i], d_flag);
        }
        unsigned int flag = 0;
        if (st == JB_OK) st = c->check(cudaMemcpyAsync(&flag, d_flag, sizeof flag, cudaMemcpyDeviceToHost, c->stream),
                                       "expr sources: flag D2H");
        // (the caller's columns are borrowed for the call only)
        if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "expr sources: creation sync");
        if (st == JB_OK && flag) st = fail_bad_address(c);
        if (st != JB_OK) {
            discard_sources(mem);
            return st;
        }
        for (size_t i = 0; i < nsources; ++i) {  // ownership of the table sources moves into the member
            if (sources[i].type != JB_SOURCE_TABLE) continue;
            auto it = c->tables.find(sources[i].table);
            mem->tables[i] = it->second;
            c->tables.erase(it);
            if (order == JB_LOW_TO_HIGH && st == JB_OK) st = c->ensure_alt(mem->tables[i], len / 2);
        }
    }
    if (st != JB_OK) {
        jb_member_destroy(mem);
        *out = nullptr;
        return st;
    }
    *out = mem;
    return eq_w_or_null ? eq_setup(mem, eq_w_or_null, nvars, eq_scale_or_null, out) : JB_OK;
}
extern "C" {

int jb_member_create_expr_sources(jb_ctx* c, const jb_source* sources, size_t nsources, size_t len,
                                  const jb_monomial* monomials, size_t nmonomials, const uint64_t* eq_w_or_null,
                                  size_t nvars, const uint64_t* eq_scale_or_null, int order, jb_member** out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!sources || !monomials || !out) return c->fail(JB_ERR_INVALID, "expr sources: null pointer");
    int D = 0;
    auto check = [&](int* D_out) {
        bool blocks = false;
        const int st = check_expr(c, nsources, monomials, nmonomials, eq_w_or_null, nvars, eq_scale_or_null, order, &D, &blocks);
        *D_out = D;
        return st;
    };
    const int st = create_over_sources(c, MemberKind::Expr, sources, nsources, len, eq_w_or_null, nvars,
                                       eq_scale_or_null, order, check, out);
    if (st == JB_OK) make_expr(*out, monomials, nmonomials, nsources, D);
    return st;
}

// ---- product member over sources ------------------------------------------------------------------------
int jb_member_create_product_sources(jb_ctx* c, const jb_source* sources, size_t nsources, size_t len,
                                     const uint64_t* eq_w_or_null, size_t nvars, const uint64_t* eq_scale_or_null,
                                     int order, jb_member** out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!sources || !out) return c->fail(JB_ERR_INVALID, "product sources: null pointer");
    // the checks of check_expr that apply to a product, in its order
    auto check = [&](int* D_out) {
        if (nsources > JB_PRODUCT_MAX_FACTORS)
            return c->fail(JB_ERR_UNSUPPORTED, "product sources: at most JB_PRODUCT_MAX_FACTORS sources");
        if (nsources == 0) return c->fail(JB_ERR_INVALID, "product sources: no sources");
        if (order != JB_HIGH_TO_LOW && order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "product sources: unknown order");
        if (eq_scale_or_null && !eq_w_or_null) return c->fail(JB_ERR_INVALID, "product sources: a scale without an eq point");
        if (eq_w_or_null) {
            for (size_t i = 0; i < nvars; ++i)
                if (!canonical_fr(eq_w_or_null + 4 * i)) return c->fail(JB_ERR_INVALID, "product sources: point limbs not canonical");
            if (eq_scale_or_null && !canonical_fr(eq_scale_or_null))
                return c->fail(JB_ERR_INVALID, "product sources: scale not canonical");
        }
        *D_out = (int)nsources;
        return (int)JB_OK;
    };
    return create_over_sources(c, MemberKind::Product, sources, nsources, len, eq_w_or_null, nvars, eq_scale_or_null,
                               order, check, out);
}

// ---- read-write checking member -------------------------------------------------------------------------
// The expression pass that finishes a read-write member, over its tables ra_0 .. ra_{A-1}, Val, inc: the monomials
// c_a e ra_a Val and c_a e ra_a inc (d_a = 1).
static void rw_make_expr(jb_member* mem, const HostFr& e) {
    RwState& rw = *mem->rw;
    const int A = rw.A;
    jb_monomial mo[2 * RW_MAX_ACCESSES];
    size_t nm = 0;
    for (int a = 0; a < A; ++a)
        for (int k = 0; k < 1 + rw.d[a]; ++k) {
            std::memset(&mo[nm], 0, sizeof mo[nm]);
            (HostFr::from_limbs(rw.coeff[a]) * e).store(mo[nm].coeff);
            mo[nm].degree = 2;
            mo[nm].table[0] = (uint32_t)a;
            mo[nm].table[1] = (uint32_t)(A + k);
            ++nm;
        }
    make_expr(mem, mo, nm, (size_t)A + 2, 2);
    rw.cycles = false;
}

// Binds a cycle variable of a read-write member (its eq factor has absorbed r); after the last one the member's address
// rounds are the expression pass over its K-entry tables ra_0 .. ra_{A-1}, Val, inc: sum_k e sum_a c_a ra_a(k) (Val(k) +
// d_a inc) with e = scale * eq(w_cycle, r_cycle).
static int rw_bind_cycle(jb_member* mem, const uint64_t r[4]) {
    int st = rw_cycle_bind(mem, r);
    if (st != JB_OK || mem->rw->rows > 1) return st;
    rw_make_expr(mem, HostFr::from_limbs(mem->eq_scalar));
    return JB_OK;
}

// An address round has degree 2; s(3) is extrapolated so the member keeps reporting degree 3.
static void rw_extrapolate_s3(uint64_t* out_evals) {
    const RoundConsts& rc = round_consts(2);
    HostFr s3 = HostFr::zero();
    for (int t = 0; t <= 2; ++t) s3 = s3 + rc.next[t] * HostFr::from_limbs(out_evals + 4 * t);
    s3.store(out_evals + 12);
}

// An address round: the first one binds the last cycle variable and hands the member over to its expression pass.
static int rw_address_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    if (round == mem->eq_n) {
        eq_absorb_bind(mem, 0, bind);
        const int st = rw_bind_cycle(mem, bind);
        if (st != JB_OK) return st;
        bind = nullptr;
    }
    const int st = launched_round(mem, bind, !c->verify_rounds, claim, round, out_evals);  // s(0..2)
    if (st != JB_OK) return st;
    rw_extrapolate_s3(out_evals);
    return JB_OK;
}

// An address round of a mixed order (p < t cycle rounds first). The first one binds the p-th cycle variable (p > 0) and
// re-sorts the entries by key; the others bind the previous address variable. The pass weights each row by
// eq(w[0 .. t - p), row), the host multiplies the eq scalar in; s(1) comes from the claim unless rounds are verified.
static int rw_key_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    const RwState& rw = *mem->rw;
    const size_t n = mem->eq_n;
    int st = JB_OK;
    if (round == rw.p && bind) {
        eq_absorb_bind(mem, n - round, bind);
        st = rw_cycle_bind(mem, bind);
    }
    if (st == JB_OK) st = round == rw.p ? rw_begin_keys(mem) : rw_key_bind(mem, bind);
    if (st == JB_OK)
        st = rw_key_pass(mem, eq_weights_l2h(mem, rw.p), mem->eq_w.data() + 4 * (n - rw.p - 1), round_out(c, nullptr, 0, nullptr));
    if (st == JB_OK) st = wait_round_result0(c);
    if (st != JB_OK) return st;
    const bool skip1 = !c->verify_rounds;
    const HostFr e = HostFr::from_limbs(mem->eq_scalar);
    uint64_t vals[3 * 4];  // q(0), [q(1)], q(inf), scaled
    int k = 0;
    for (int i = 0; i < 3; ++i)
        if (i != 1 || !skip1) (e * HostFr::from_limbs(c->h_result + 4 * i)).store(vals + 4 * k++);
    if ((st = assemble_evals(c, 2, skip1, vals, claim, round, out_evals)) != JB_OK) return st;
    rw_extrapolate_s3(out_evals);
    return JB_OK;
}

// The last address bind of a mixed order: the remaining cycle rounds are the expression pass over the dense tables,
// split-eq weighted over w[0 .. t - p) with the member's eq scalar.
static int rw_end_keys(jb_member* mem, const uint64_t r[4]) {
    const int st = rw_key_bind(mem, r);
    if (st == JB_OK) rw_make_expr(mem, HostFr::one());
    return st;
}

int jb_member_create_read_write_phases(jb_ctx* c, const jb_rw_access* accesses, size_t naccesses, size_t write_access,
                                       int addr_kind, int addr_on_device, size_t T, size_t K, const jb_source* inc,
                                       const jb_source* init, const uint64_t* w_cycle, size_t nvars,
                                       const uint64_t* scale_or_null, size_t cycle_rounds_first, int order,
                                       jb_member** out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    jb_member* mem = nullptr;
    {
        Guard g(c);
        const int st = rw_create(c, accesses, naccesses, write_access, addr_kind, addr_on_device, T, K, inc, init, w_cycle,
                                 nvars, scale_or_null, cycle_rounds_first, order, &mem);
        if (st != JB_OK) return st;
    }
    *out = mem;
    return eq_setup(mem, w_cycle, nvars, scale_or_null, out);
}

int jb_member_create_read_write(jb_ctx* c, const jb_rw_access* accesses, size_t naccesses, size_t write_access,
                                int addr_kind, int addr_on_device, size_t T, size_t K, const jb_source* inc,
                                const jb_source* init, const uint64_t* w_cycle, size_t nvars, const uint64_t* scale_or_null,
                                int order, jb_member** out) {
    // every cycle round first (p = log2 T; T itself is checked by rw_create)
    const size_t t = T >= 1 && (T & (T - 1)) == 0 ? (size_t)log2_of(T) : 0;
    return jb_member_create_read_write_phases(c, accesses, naccesses, write_access, addr_kind, addr_on_device, T, K, inc,
                                              init, w_cycle, nvars, scale_or_null, t, order, out);
}

// ---- booleanity member ----------------------------------------------------------------------------------
// An address round: the address coordinate of the previous round is absorbed into the eq scalar, the current one's
// factor l(t) is the host's, and the pass over the K-entry tables (which binds the previous variable) gives q.
static int bool_address_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim, uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    const BoolState& bl = *mem->bl;
    if (bind) eq_absorb_coord(mem, bool_addr_coord(bl, round - 1), bind);
    const HostFr scalar = HostFr::from_limbs(mem->eq_scalar);
    const HostFr l1 = scalar * HostFr::from_limbs(bool_addr_coord(bl, round)), l0 = scalar - l1;
    if (l1.is_zero()) return c->fail(JB_ERR_INVALID, "eq member: current eq evaluation at one must be invertible");
    const int st = bool_address_pass(mem, bind, round, round_out(c, nullptr, 0, nullptr));
    if (st != JB_OK) return st;
    return eq_round_tail(mem, l0, l1, claim, round, out_evals);
}

int jb_member_create_booleanity(jb_ctx* c, const void* const* columns, size_t count, int kind, int on_device, size_t T,
                                size_t K, const uint64_t* coeffs, const uint64_t* r_addr, const uint64_t* r_cycle,
                                const uint64_t* scale_or_null, int order, jb_member** out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    jb_member* mem = nullptr;
    {
        Guard g(c);
        const int st = bool_create(c, columns, count, kind, on_device, T, K, coeffs, r_addr, r_cycle, scale_or_null,
                                   order, &mem);
        if (st != JB_OK) return st;
    }
    *out = mem;
    if (T >= 2) return eq_setup(mem, r_cycle, mem->bl->log_t, scale_or_null, out);
    // T = 1: address rounds only, no cycle eq tables
    (scale_or_null ? HostFr::from_limbs(scale_or_null) : HostFr::one()).store(mem->eq_scalar);
    return JB_OK;
}

// eq(w, r) * scale after all rounds (the member's eq factor of the final claim)
int jb_eq_member_scalar(jb_member* mem, uint64_t out[4]) {
    if (!mem || !out || !eq_rounds(mem)) return JB_ERR_INVALID;
    std::memcpy(out, mem->eq_scalar, 32);
    return JB_OK;
}
// ---- index-sharded member ----------------------------------------------------------------------
// HighToLow shards are strided (rank g owns global[j * G + g]): gathered[g][j] -> global[j * G + g]
static __global__ void __launch_bounds__(256) interleave_shards_kernel(const uint64_t* gathered, uint64_t* global, size_t len,
                                                                       size_t G) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= len * G) return;
    const size_t g = idx / len, j = idx % len;
    st_elem(global, j * G + g, ld_elem<Fr>(gathered, idx));
}

static int gather_into_tail(jb_member* mem) {  // called with the context lock held
    jb_ctx* c = mem->ctx;
    const size_t len = mem->len, G = (size_t)c->world;
    jb_member* tail = new_member(c, MemberKind::Dense, mem->m, mem->terms, mem->order, len * G);
    if (!tail) return JB_ERR_OOM;
    int st = JB_OK;
    for (int j = 0; j < mem->ntables() && st == JB_OK; ++j) {
        Table t;
        st = c->dev_alloc((void**)&t.buf, tail->len * 32);
        if (st != JB_OK) break;
        t.cap = t.len = tail->len;
        tail->tables.push_back(t);  // owned by the tail from here on (released below on failure)
        if (mem->order == JB_LOW_TO_HIGH) {
            // rank order == global order for contiguous blocks under LowToHigh binding
            st = c->comm_allgather(mem->tables[j].buf, t.buf, len * 4);
        } else {
            Scratch scratch(c);
            uint64_t* tmp = nullptr;
            st = scratch.alloc(tail->len * 32, &tmp);
            if (st == JB_OK) st = c->comm_allgather(mem->tables[j].buf, tmp, len * 4);
            if (st == JB_OK) {
                interleave_shards_kernel<<<(unsigned)((tail->len + 255) / 256), 256, 0, c->stream>>>(tmp, t.buf, len, G);
                c->launches++;
                st = c->check(cudaGetLastError(), "interleave_shards launch");
            }
        }
    }
    if (st != JB_OK) {
        for (auto& t : tail->tables) c->release(t);
        delete tail;
        return st;
    }
    mem->tail = tail;
    return JB_OK;
}

static int sharded_prove_round(jb_member* mem, const uint64_t* bind, size_t round, const uint64_t* claim,
                               uint64_t* out_evals) {
    jb_ctx* c = mem->ctx;
    {
        Guard g(c, true);
        if (round != mem->rounds_done) return c->fail(JB_ERR_INVALID, "prove_round: round index out of sequence");
        if (bind && !canonical_fr(bind)) return c->fail(JB_ERR_INVALID, "prove_round: challenge limbs not canonical");
        if (mem->gathered) {
            // gathered inside the resident kernel: an ordinary member from here on
            if (bind && mem->len < 4) return c->fail(JB_ERR_INVALID, "prove_round: no round left after this bind (use finish_rounds)");
            const bool skip1 = claim != nullptr && !c->verify_rounds;
            int st = JB_ERR_UNSUPPORTED;
            if (skip1) {
                st = resident_member_prove(mem, bind, claim, round, false, out_evals);
                if (st == JB_OK) mem->rounds_done--;
                if (st != JB_ERR_UNSUPPORTED) return st;
            }
            before_launch(mem);
            return launched_round(mem, bind, skip1, claim, round, out_evals);
        }
        if (!mem->tail) {
            const size_t len_after = bind ? mem->len / 2 : mem->len;
            if (len_after > mem->gather_len) {
                // a sharded round: local fused pass -> lanes -> ONE all-reduce -> host fold
                const bool skip1 = claim != nullptr && !c->verify_rounds;
                const int K = skip1 ? mem->m : mem->m + 1;
                int st = JB_ERR_UNSUPPORTED;
                if (skip1 && c->xch_ready) {
                    // resident kernel: the all-reduce over NVLink peer memory rides in the round's own epilogue,
                    // no launch and no NCCL call per round
                    st = resident_member_prove(mem, bind, claim, round, true, out_evals);
                    if (st == JB_OK) mem->rounds_done--;  // (the caller counts sharded rounds)
                    if (st != JB_ERR_UNSUPPORTED) return st;
                }
                if (st == JB_ERR_UNSUPPORTED) {
                    before_launch(mem);
                    if (c->xch_ready) {
                        st = member_round(mem, bind, skip1, JB_LANES_EXCHANGE);
                    } else {
                        st = member_round(mem, bind, skip1, c->d_lanes);
                        if (st == JB_OK) st = c->comm_allreduce_lanes(c->d_lanes, (size_t)K * 8);
                        if (st == JB_OK) st = c->publish_lanes(c->d_lanes, K * 8);
                    }
                    if (st == JB_OK) st = wait_round_result0(c);
                    if (st != JB_OK) return st;
                    if (c->h_result[0] == ~0ull && c->h_result[1] == ~0ull)
                        return c->fail(JB_ERR_CUDA, "peer exchange timed out (a rank did not arrive)");
                }
                uint64_t vals[JB_MAX_EVALS * 4];
                st = jb_lanes_reduce_host(c->h_result, (size_t)K, vals);
                if (st != JB_OK) return st;
                return assemble_evals(c, mem->m, skip1, vals, claim, round, out_evals);
            }
            // the shard is small. If its resident kernel is alive and the arena holds the gathered tables, the
            // kernel itself gathers: it binds, writes the bound shard into every rank's arena over NVLink, waits for
            // the peers' shards and sweeps the gathered tables - no kernel exit, no NCCL call; from here on this
            // member proves its remaining rounds un-sharded (identically on every rank)
            const bool skip1g = claim != nullptr && !c->verify_rounds;
            if (bind && skip1g && mem->run && len_after == mem->gather_len && resident_gather_fits(c, mem, len_after)) {
                int st = resident_member_prove(mem, bind, claim, round, false, out_evals, true);
                if (st == JB_OK) {
                    mem->rounds_done--;  // (the caller counts sharded rounds)
                    mem->gathered = true;
                }
                return st;
            }
            // otherwise: stop the resident kernel (its tables are consistent at a round boundary),
            // apply the pending bind, gather with NCCL, continue on the tail
            if (mem->run) resident_end(mem->run, false);
            c->quiesce_resident(false);
            if (bind) {
                for (int j = 0; j < mem->ntables(); ++j) {
                    int st = bind_table(c, mem->tables[j], bind, mem->order);
                    if (st != JB_OK) return st;
                }
                mem->len /= 2;
                bind = nullptr;
            }
            int st = gather_into_tail(mem);
            if (st != JB_OK) return st;
        }
    }
    return jb_member_prove_round(mem->tail, bind, mem->tail->rounds_done, claim, out_evals);
}

int jb_sharded_member_create(jb_ctx* c, const jb_table* handles, size_t m, int order, size_t gather_log, jb_member** out) {
    if (!c || !out) return JB_ERR_INVALID;
    if (!c->nccl_comm) return c->fail(JB_ERR_INVALID, "sharded member: no communicator (jb_comm_init)");
    if (order != JB_LOW_TO_HIGH && order != JB_HIGH_TO_LOW) return c->fail(JB_ERR_INVALID, "sharded member: unknown binding order");
    int st = jb_member_create(c, handles, m, order, out);
    if (st != JB_OK) return st;
    jb_member* mem = *out;
    size_t log_g = 0;
    while ((1 << log_g) < c->world) ++log_g;
    mem->sharded = true;
    mem->gather_len = (size_t)1 << gather_log;
    if (mem->gather_len > mem->len) mem->gather_len = mem->len;
    mem->rounds += log_g;
    return JB_OK;
}

int jb_member_prove_round_partials(jb_member* mem, const uint64_t* bind, size_t round, int skip_t1, void* lanes_out) {
    (void)round;
    if (!mem || !lanes_out) return JB_ERR_INVALID;
    Guard g(mem->ctx, true);
    static const char* const names[] = {"dense", "expression", "product", "read-write", "booleanity"};  // by MemberKind
    if (mem->kind != MemberKind::Dense)
        return mem->ctx->fail(JB_ERR_UNSUPPORTED, (std::string("prove_round_partials: ") + names[(int)mem->kind] +
                                                   " members are not sharded").c_str());
    before_launch(mem);
    return member_round(mem, bind, skip_t1 != 0, lanes_out);
}

int jb_ctx_set_verify_rounds(jb_ctx* c, int on) {
    if (!c) return JB_ERR_INVALID;
    Guard g(c);
    c->verify_rounds = on != 0;
    return JB_OK;
}

// carry-propagate 8 x (sums of 32-bit limbs) and fold mod r: O(count) host work, no device needed.
int jb_lanes_reduce_host(const uint64_t* lanes, size_t count, uint64_t* out) {
    if (!lanes || !out) return JB_ERR_INVALID;
    for (size_t k = 0; k < count; ++k) {
        const uint64_t* lane = lanes + 8 * k;
        uint32_t w[10];
        unsigned __int128 carry = 0;
        for (int i = 0; i < 8; ++i) {
            carry += lane[i];
            w[i] = (uint32_t)carry;
            carry >>= 32;
        }
        w[8] = (uint32_t)carry;
        w[9] = (uint32_t)(carry >> 32);
        // value < 2^32 * r < 2^286; fold by subtracting (r << sh) from the top down
        uint64_t v[5] = {(uint64_t)w[0] | ((uint64_t)w[1] << 32), (uint64_t)w[2] | ((uint64_t)w[3] << 32),
                         (uint64_t)w[4] | ((uint64_t)w[5] << 32), (uint64_t)w[6] | ((uint64_t)w[7] << 32),
                         (uint64_t)w[8] | ((uint64_t)w[9] << 32)};
        for (int sh = 33; sh >= 0; --sh) {
            uint64_t ps[5] = {0, 0, 0, 0, 0};  // r << sh
            for (int i = 0; i < 4; ++i) {
                ps[i] |= sh ? (HostFr::P[i] << sh) : HostFr::P[i];
                if (sh) ps[i + 1] |= HostFr::P[i] >> (64 - sh);
            }
            bool ge = true;
            for (int i = 4; i >= 0; --i)
                if (v[i] != ps[i]) { ge = v[i] > ps[i]; break; }
            if (ge) {
                uint64_t borrow = 0;
                for (int i = 0; i < 5; ++i) {
                    unsigned __int128 t = (unsigned __int128)v[i] - ps[i] - borrow;
                    v[i] = (uint64_t)t;
                    borrow = (uint64_t)(t >> 64) & 1;
                }
            }
        }
        std::memcpy(out + 4 * k, v, 32);
    }
    return JB_OK;
}

// The serial tail of a round of the resident kernel: `count` values, each the 17 u64 lanes of a block-summed
// unreduced accumulator sum_y a_y b_y over Montgomery operands (lane w = sum of the 32-bit limbs of weight 2^(32 w),
// < 2^64). V = sum_w lane_w 2^(32 w) < 2^577 = lo + h0 2^256 + h1 2^512; the field value is V R^-1 mod p =
// REDC(lo) + h0 + h1 R, each term one word-serial Montgomery product with the wide operand as the multiplier.
int jb_wide_lanes_reduce_host(const uint64_t* lanes, size_t count, uint64_t* out) {
    if (!lanes || !out) return JB_ERR_INVALID;
    static const HostFr raw_one{{1, 0, 0, 0}};
    static const HostFr r1{{HostFr::R1[0], HostFr::R1[1], HostFr::R1[2], HostFr::R1[3]}};
    static const HostFr r2{{HostFr::R2[0], HostFr::R2[1], HostFr::R2[2], HostFr::R2[3]}};
    for (size_t k = 0; k < count; ++k) {
        const uint64_t* lane = lanes + 17 * k;
        uint32_t w[20];
        unsigned __int128 carry = 0;
        for (int i = 0; i < 17; ++i) {
            carry += lane[i];
            w[i] = (uint32_t)carry;
            carry >>= 32;
        }
        for (int i = 17; i < 20; ++i) {
            w[i] = (uint32_t)carry;
            carry >>= 32;
        }
        HostFr lo, h0, h1;
        for (int i = 0; i < 4; ++i) {
            lo.l[i] = (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32);
            h0.l[i] = (uint64_t)w[8 + 2 * i] | ((uint64_t)w[8 + 2 * i + 1] << 32);
        }
        h1 = HostFr{{(uint64_t)w[16] | ((uint64_t)w[17] << 32), (uint64_t)w[18] | ((uint64_t)w[19] << 32), 0, 0}};
        const HostFr v = raw_one * lo + r1 * h0 + r2 * h1;
        v.store(out + 4 * k);
    }
    return JB_OK;
}

// lanes of one member's round (as the resident kernel publishes them) -> K canonical values
static int resident_values(int D, const uint64_t* lanes, uint64_t* vals) {
    return D == 1 ? jb_lanes_reduce_host(lanes, 1, vals) : jb_wide_lanes_reduce_host(lanes, (size_t)D, vals);
}

int jb_partials_finalize(jb_ctx* c, const void* device_lanes, size_t count, uint64_t* out) {
    if (!c || !device_lanes || !out || count == 0 || count * 64 > JB_SMALL_BYTES) return JB_ERR_INVALID;
    Guard g(c);
    int st = c->check(cudaMemcpyAsync(c->h_small, device_lanes, count * 64, cudaMemcpyDeviceToHost, c->stream),
                      "partials D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "partials sync");
    if (st != JB_OK) return st;
    return jb_lanes_reduce_host(c->h_small, count, out);
}


// Copies table j of a member (its current, possibly partly bound, contents) into caller device memory.
int jb_member_export_table(jb_member* mem, size_t j, void* device_dst, size_t cap_elems, size_t* len_out) {
    if (!mem || !device_dst) return JB_ERR_INVALID;
    jb_ctx* c = mem->ctx;
    Guard g(c, true);
    before_launch(mem);  // the host's view of the tables (buffer parity, length) is exact at a round boundary
    if (mem->kind == MemberKind::Booleanity)
        return c->fail(JB_ERR_INVALID, "export_table: a booleanity member keeps its tables to itself");
    if (j >= (size_t)mem->ntables()) return c->fail(JB_ERR_INVALID, "export_table: table index out of range");
    if (mem->kind == MemberKind::ReadWrite && mem->rw->cycles)
        return c->fail(JB_ERR_INVALID, "export_table: a read-write member in its cycle rounds has no tables");
    if (!mem->src.empty() && mem->src[j].type != JB_SOURCE_TABLE)
        return c->fail(JB_ERR_INVALID, "export_table: the source is not bound yet (a column, not a field table)");
    if (cap_elems < mem->len) return c->fail(JB_ERR_INVALID, "export_table: destination too small");
    if (len_out) *len_out = mem->len;
    return c->check(cudaMemcpyAsync(device_dst, mem->tables[j].buf, mem->len * 32, cudaMemcpyDeviceToDevice, c->stream),
                    "export_table D2D");
}

int jb_member_finish_rounds(jb_member* mem, const uint64_t bind[4]) {
    if (!mem || !bind) return JB_ERR_INVALID;
    jb_ctx* c = mem->ctx;
    if (mem->sharded && !mem->gathered) {
        if (!mem->tail) return c->fail(JB_ERR_INVALID, "finish_rounds: sharded member has not reached its tail");
        return jb_member_finish_rounds(mem->tail, bind);
    }
    Guard g(c, true);
    if (mem->len < 2) return c->fail(JB_ERR_INVALID, "finish_rounds: member already fully bound");
    if (!canonical_fr(bind)) return c->fail(JB_ERR_INVALID, "finish_rounds: challenge limbs not canonical");
    if (mem->kind == MemberKind::ReadWrite && mem->rw->cycles) {  // K = 1: the last cycle variable is the member's last
        if (mem->len != 2) return c->fail(JB_ERR_INVALID, "finish_rounds: rounds remain");
        eq_absorb_bind(mem, 0, bind);
        return rw_bind_cycle(mem, bind);
    }
    if (mem->kind == MemberKind::Booleanity) {  // the last variable: a cycle one, or the last address one when T = 1
        if (mem->len != 2) return c->fail(JB_ERR_INVALID, "finish_rounds: rounds remain");
        const BoolState& bl = *mem->bl;
        eq_absorb_coord(mem, bl.T == 1 ? bool_addr_coord(bl, bl.log_k - 1)
                                       : mem->eq_w.data() + 4 * (mem->order == JB_LOW_TO_HIGH ? 0 : mem->eq_n - 1), bind);
        before_launch(mem);
        const int st = bool_finish(mem, bind);
        if (st == JB_OK) mem->len = 1;
        return st;
    }
    // (the address rounds of a read-write member that binds every cycle variable first have no eq factor)
    if (mem->eq && (mem->kind != MemberKind::ReadWrite || mem->rw->p < mem->eq_n)) {
        size_t var = 0;
        for (size_t l = mem->len; l > 2; l >>= 1) ++var;  // unbound variables besides the one being bound
        // LowToHigh binds w[var] (the most significant unbound one is w[0]); HighToLow binds w[n - 1 - var]
        eq_absorb_bind(mem, mem->order == JB_LOW_TO_HIGH ? var : mem->eq_n - 1 - var, bind);
    }
    // right after a round answered from lookahead its challenge is still pending: the run ends (and binds it) first
    if (mem->run && mem->pend) resident_end(mem->run, false);
    if (mem->run) {
        // the terminal bind is one more mailbox command; a fully bound member gets its values back with the
        // acknowledgement (has_final), so nothing is read from the device afterwards
        const int st = resident_member_final(mem, bind);
        // (a kernel found lost before the command was posted leaves the bind to the launches below)
        if (st != JB_OK || mem->len < 2) return st;
    }
    before_launch(mem);
    if (!mem->src.empty()) {  // len = 2: the sources are bound straight from their columns
        int st = mem->kind == MemberKind::Product ? product_finish(mem, bind) : sources_finish(mem, bind);
        if (st != JB_OK) return st;
    } else {
        for (int j = 0; j < mem->ntables(); ++j) {
            int st = bind_table(c, mem->tables[j], bind, mem->order);
            if (st != JB_OK) return st;
        }
    }
    mem->len /= 2;
    return JB_OK;
}

// Where table j's single entry lies once the member is fully bound.
static const uint64_t* final_entry(const jb_member* mem, int j) {
    return mem->kind == MemberKind::Booleanity ? bool_final_entry(mem, j) : mem->tables[j].buf;
}

int jb_member_final_evals(jb_member* mem, uint64_t* out) {
    if (!mem || !out) return JB_ERR_INVALID;
    jb_ctx* c = mem->ctx;
    if (mem->sharded && !mem->gathered) {
        if (!mem->tail) return c->fail(JB_ERR_INVALID, "NotFullyBound (sharded member before its tail)");
        return jb_member_final_evals(mem->tail, out);
    }
    Guard g(c, true);
    const int T = mem->ntables();
    if (mem->has_final) {
        std::memcpy(out, mem->final_vals, (size_t)T * 32);
        return JB_OK;
    }
    if (mem->len != 1) {
        char buf[96];
        size_t remaining = mem->pend ? (size_t)-1 : 0;  // (a pending challenge is a round already bound)
        for (size_t l = mem->len; l > 1; l >>= 1) ++remaining;
        std::snprintf(buf, sizeof buf, "NotFullyBound { remaining: %zu }", remaining);
        return c->fail(JB_ERR_INVALID, buf);
    }
    before_launch(mem);
    for (int j = 0; j < T; ++j) {
        int st = c->check(cudaMemcpyAsync(c->h_small + 4 * j, final_entry(mem, j), 32, cudaMemcpyDeviceToHost, c->stream),
                          "final evals D2H");
        if (st != JB_OK) return st;
    }
    int st = c->check(cudaStreamSynchronize(c->stream), "final evals sync");
    if (st != JB_OK) return st;
    std::memcpy(out, c->h_small, (size_t)T * 32);
    return JB_OK;
}

void jb_member_destroy(jb_member* mem) {
    if (!mem) return;
    if (mem->tail) jb_member_destroy(mem->tail);
    Guard g(mem->ctx, true);
    if (mem->run) resident_end(mem->run, false);
    if (mem->eq_tabs) mem->ctx->dev_free(mem->eq_tabs);
    switch (mem->kind) {
        case MemberKind::Expr:
        case MemberKind::Product: sources_release(mem); break;
        case MemberKind::ReadWrite: rw_release(mem); delete mem->rw; break;
        case MemberKind::Booleanity: bool_release(mem); delete mem->bl; break;
        default: break;
    }
    for (auto& t : mem->tables) mem->ctx->release(t);
    delete mem;
}

// ---- device RoundScheduler (crates/jolt-sumcheck/src/prover.rs:106-120; BuildRoundScheduler,
//      crates/jolt-kernels/src/backend.rs:64-70) ------------------------------------------------------------
// "Order and transport are free": a batch round costs ONE host round trip whatever the member count.
//   * homogeneous batches (same shape and order, <= RES_MAX_MEMBERS members) are served by ONE resident kernel:
//     a single mailbox command carries every member's action and the shared challenge, the kernel answers
//     with every member's round sums;
//   * otherwise every active member's pass is enqueued before the first wait (one result slot per member;
//     short members through their own small resident kernels), then the results are collected - in chunks of
//     JB_RESULT_SLOTS - 1 members when more are active.
struct jb_scheduler {
    jb_ctx* ctx;
    std::vector<jb_member*> members;
    bool homogeneous = false;
    bool run_failed = false;  // a resident batch could not be started: stay on the overlapped launches
};

int jb_scheduler_create(jb_ctx* c, jb_member** members, size_t n, jb_scheduler** out) {
    if (!c || !members || !out || n == 0) return JB_ERR_INVALID;
    Guard g(c, true);
    jb_scheduler* s = new (std::nothrow) jb_scheduler();
    if (!s) return JB_ERR_OOM;
    s->ctx = c;
    s->homogeneous = n <= (size_t)RES_MAX_MEMBERS;
    for (size_t i = 0; i < n; ++i) {
        jb_member* m = members[i];
        if (!m || m->ctx != c) {
            delete s;
            return c->fail(JB_ERR_INVALID, "scheduler: members must belong to the scheduler's context");
        }
        for (size_t k = 0; k < i; ++k)
            if (members[k] == m) {
                delete s;
                return c->fail(JB_ERR_INVALID, "scheduler: duplicate member");
            }
        if (m->m + (eq_rounds(m) ? 1 : 0) + 1 > JB_MAX_EVALS) {  // out_evals holds JB_MAX_EVALS elements per work item
            delete s;
            return c->fail(JB_ERR_UNSUPPORTED, "scheduler: a member of degree >= 8");
        }
        s->members.push_back(m);
        if (!resident_kind(m) || m->sharded || m->m != members[0]->m || m->terms != members[0]->terms ||
            m->order != members[0]->order)
            s->homogeneous = false;
    }
    *out = s;
    return JB_OK;
}

void jb_scheduler_destroy(jb_scheduler* s) { delete s; }

// starts the batch's resident kernel over every member that still has rounds to prove
static int scheduler_begin_run(jb_scheduler* s) {
    jb_ctx* c = s->ctx;
    std::vector<jb_member*> live;
    for (auto* m : s->members) {
        if (m->run) return JB_ERR_UNSUPPORTED;  // already served by another run
        if (m->len >= 2) {
            if (!resident_eligible(m)) return JB_ERR_UNSUPPORTED;
            live.push_back(m);
        }
    }
    if (live.empty()) return JB_ERR_UNSUPPORTED;
    return resident_begin(c, live.data(), (int)live.size());
}

static int overlapped_rounds(jb_scheduler* s, const jb_round_work* work, size_t n_work, uint64_t* out_evals);

int jb_scheduler_prove_round(jb_scheduler* s, const jb_round_work* work, size_t n_work, uint64_t* out_evals) {
    if (!s || (n_work && (!work || !out_evals))) return JB_ERR_INVALID;
    jb_ctx* c = s->ctx;
    // sharded members synchronise across ranks inside their own round: no overlap to win, run them in order
    for (size_t i = 0; i < n_work; ++i) {
        if (work[i].member >= s->members.size()) return c->fail(JB_ERR_INVALID, "scheduler: member index out of range");
        if (s->members[work[i].member]->sharded) {
            for (size_t k = 0; k < n_work; ++k) {
                const jb_round_work& w = work[k];
                int st = jb_member_prove_round(s->members[w.member], w.has_bind ? w.bind : nullptr, w.round,
                                               w.has_claim ? w.claim : nullptr, out_evals + k * JB_MAX_EVALS * 4);
                if (st != JB_OK) return st;
            }
            return JB_OK;
        }
    }
    Guard g(c, true);
    const uint64_t* shared_bind = nullptr;
    bool all_skip1 = !c->verify_rounds, same_bind = true;
    for (size_t i = 0; i < n_work; ++i) {
        const jb_round_work& w = work[i];
        jb_member* m = s->members[w.member];
        for (size_t k = 0; k < i; ++k)
            if (work[k].member == w.member) return c->fail(JB_ERR_INVALID, "scheduler: a member appears twice in one round");
        const int st = check_round_args(m, w.has_bind ? w.bind : nullptr, w.round);
        if (st != JB_OK) return st;
        if (w.has_claim && !canonical_fr(w.claim)) return c->fail(JB_ERR_INVALID, "prove_round: claim limbs not canonical");
        if (m->len < (w.has_bind ? 4u : 2u)) return c->fail(JB_ERR_INVALID, "prove_round: member has no round left");
        if (!w.has_claim) all_skip1 = false;
        if (w.has_bind) {
            if (shared_bind && std::memcmp(shared_bind, w.bind, 32) != 0) same_bind = false;
            shared_bind = w.bind;
        }
    }
    // ---- one resident kernel for the whole batch -------------------------------------------------------
    if (s->homogeneous && !s->run_failed && all_skip1 && same_bind && c->use_tail && n_work) {
        ResidentRun* run = s->members[work[0].member]->run;
        bool ok = true;
        if (!run) {
            int st = scheduler_begin_run(s);
            if (st == JB_OK) run = s->members[work[0].member]->run;
            else if (st == JB_ERR_UNSUPPORTED) ok = false;
            else return st;
        }
        for (size_t i = 0; ok && i < n_work; ++i) ok = s->members[work[i].member]->run == run;
        if (ok && run) {
            RunItem items[RES_MAX_MEMBERS];
            for (size_t i = 0; i < n_work; ++i)
                items[i] = RunItem{s->members[work[i].member], work[i].has_bind ? work[i].bind : nullptr, work[i].claim,
                                   work[i].round, out_evals + i * JB_MAX_EVALS * 4};
            int st = run_round(c, run, items, (int)n_work, shared_bind, false);
            if (st != JB_OK && s->members[work[0].member]->run) resident_end(s->members[work[0].member]->run, true);
            return st;
        }
        s->run_failed = true;
    }
    // ---- overlapped: enqueue every member's pass, then collect -----------------------------------------
    // Slot 0 serves in-place rounds, so at most JB_RESULT_SLOTS - 1 launched passes can be in flight: larger batches
    // run in chunks of that many members, each chunk enqueued (into slots 1..) and collected before the next.
    c->quiesce_resident(false);
    for (size_t base = 0; base < n_work; base += JB_RESULT_SLOTS - 1) {
        const size_t n_chunk = std::min(n_work - base, (size_t)JB_RESULT_SLOTS - 1);
        int st = overlapped_rounds(s, work + base, n_chunk, out_evals + base * JB_MAX_EVALS * 4);
        if (st != JB_OK) return st;
    }
    return JB_OK;
}

// one chunk of the overlapped path: every member's pass is enqueued (member i of the chunk reports into result
// slot i + 1), then the results are collected
static int overlapped_rounds(jb_scheduler* s, const jb_round_work* work, size_t n_work, uint64_t* out_evals) {
    jb_ctx* c = s->ctx;
    enum { VIA_LAUNCH = 0, VIA_RUN = 1 };
    int via[JB_RESULT_SLOTS];
    uint64_t seqs[JB_RESULT_SLOTS];
    bool skip[JB_RESULT_SLOTS];
    for (size_t i = 0; i < n_work; ++i) {
        const jb_round_work& w = work[i];
        jb_member* m = s->members[w.member];
        const uint64_t* bind = w.has_bind ? w.bind : nullptr;
        skip[i] = w.has_claim && !c->verify_rounds;
        via[i] = VIA_LAUNCH;
        if (eq_rounds(m)) {  // the Gruen member needs host work between its launch and its result: run it in place
            int st = eq_prove_round(m, bind, w.round, w.has_claim ? w.claim : nullptr, out_evals + i * JB_MAX_EVALS * 4);
            if (st != JB_OK) return st;
            m->rounds_done++;
            via[i] = -1;
            continue;
        }
        const size_t len_after = bind ? m->len / 2 : m->len;
        if (skip[i] && len_after <= RES_SMALL_LEN && (m->run || resident_eligible(m))) {
            // short member: its own small resident kernel (a few blocks), one mailbox command
            if (!m->run) {
                jb_member* one[1] = {m};
                int st = resident_begin(c, one, 1, len_after, false);
                if (st != JB_OK && st != JB_ERR_UNSUPPORTED) return st;
            }
            if (m->run && resident_run_size(m->run) == 1) {
                unsigned actions[RES_MAX_MEMBERS] = {0};
                actions[m->run_idx] = bind ? RES_ACT_BIND_EVAL : RES_ACT_EVAL;
                int st = JB_OK;
                while (st == JB_OK && resident_inflight(m->run) > 0) st = resident_consume(m->run, nullptr, nullptr);
                if (st == JB_OK) st = resident_post(m->run, actions, bind, false);
                if (st == JB_RES_LOST) st = resident_recover(m->run);  // back to launches (below)
                else if (st != JB_OK) return st;
                else {
                    m->look_ok = false;
                    via[i] = VIA_RUN;
                    continue;
                }
                if (st != JB_OK) return st;
            }
        }
        if (m->run) resident_end(m->run, true);
        int st = member_round(m, bind, skip[i], nullptr, nullptr, (int)i + 1, &seqs[i]);
        if (st != JB_OK) return st;
    }
    for (size_t i = 0; i < n_work; ++i) {
        if (via[i] < 0) continue;
        const jb_round_work& w = work[i];
        jb_member* m = s->members[w.member];
        int st;
        if (via[i] == VIA_RUN) {
            uint64_t out[RES_MAX_MEMBERS * RES_SLOT_U64];
            ResConsumed info[RES_MAX_MEMBERS];
            st = resident_consume(m->run, out, info);
            if (st == JB_RES_LOST) {  // recover (replays this round's bind), then an eval-only launch
                st = resident_recover(m->run);
                if (st == JB_OK) st = launched_round(m, nullptr, true, w.claim, w.round, out_evals + i * JB_MAX_EVALS * 4);
            } else if (st == JB_OK) {
                uint64_t vals[JB_MAX_EVALS * 4];
                answer_values(m, info[0], out, vals);
                st = assemble_evals(c, m->m, true, vals, w.claim, w.round, out_evals + i * JB_MAX_EVALS * 4);
            }
        } else {
            st = wait_round_result(c, (int)i + 1, seqs[i]);
            uint64_t vals[JB_MAX_ROUND_EVALS * 4];
            if (st == JB_OK)
                st = assemble_evals(c, m->m, skip[i], slot_values(c->h_result + (i + 1) * JB_SLOT_U64, m->m, skip[i], vals),
                                    w.has_claim ? w.claim : nullptr, w.round, out_evals + i * JB_MAX_EVALS * 4);
        }
        if (st != JB_OK) return st;
        m->rounds_done++;
    }
    return JB_OK;
}

int jb_scheduler_finish_rounds(jb_scheduler* s, const jb_finish_work* work, size_t n_work) {
    if (!s || (n_work && !work)) return JB_ERR_INVALID;
    jb_ctx* c = s->ctx;
    {
        Guard g(c, true);
        // every finishing member of one resident run takes its terminal bind in ONE command
        ResidentRun* run = nullptr;
        bool one_run = n_work > 0;
        for (size_t i = 0; i < n_work && one_run; ++i) {
            if (work[i].member >= s->members.size()) return c->fail(JB_ERR_INVALID, "scheduler: member index out of range");
            jb_member* m = s->members[work[i].member];
            if (!m->run || m->eq || m->sharded || m->len != 2 || !canonical_fr(work[i].bind)) one_run = false;
            else if (!run) run = m->run;
            else if (m->run != run) one_run = false;
            if (one_run && std::memcmp(work[0].bind, work[i].bind, 32) != 0) one_run = false;
        }
        if (one_run && run) {
            unsigned actions[RES_MAX_MEMBERS] = {0};
            for (size_t i = 0; i < n_work; ++i) actions[s->members[work[i].member]->run_idx] = RES_ACT_FINAL;
            int st = resident_round(run, actions, work[0].bind, false, nullptr);
            return st == JB_RES_LOST ? resident_recover(run) : st;
        }
    }
    for (size_t i = 0; i < n_work; ++i) {
        if (work[i].member >= s->members.size()) return c->fail(JB_ERR_INVALID, "scheduler: member index out of range");
        int st = jb_member_finish_rounds(s->members[work[i].member], work[i].bind);
        if (st != JB_OK) return st;
    }
    return JB_OK;
}

}  // extern "C"
