// Booleanity member (jb_member_create_booleanity): Shout's booleanity check on the RA polynomials,
//   sum_k sum_j scale eq(r_addr, k) eq(r_cycle, j) sum_i c_i (ra_i(k, j)^2 - ra_i(k, j)),   ra_i(k, j) = [addr_i(j) = k],
// over the K x T matrix from the address columns, in O(d T + d K) memory.
//
// Address phase (log K rounds). G_i[k] = sum_{j: addr_i(j) = k} eq(r_cycle, j) is the pushforward and Q_i starts equal
// to it. ra_i is one-hot, so once some address variables are bound to r' every cycle contributes one product of eq
// factors, and its square carries the squared factors:
//   sum_j eq(r_cycle, j) ra_i(r', X, k_rest, j)^2 = (1 - X)^2 Q_i[lo] + X^2 Q_i[hi]
// when Q binds by the squared rule (1 - r)^2 lo + r^2 hi, while G binds linearly. Weighted by eq over the address
// coordinates after the current one (the current one's factor is the host's, as for every split-eq member), a round's
// inner polynomial is
//   q(X) = sum_pairs eq_rest sum_i c_i [(1 - X)^2 Q_i[lo] + X^2 Q_i[hi] - ((1 - X) G_i[lo] + X G_i[hi])],
// so q(0) = sum eq_rest c_i (Q_lo - G_lo) and q(inf) = sum eq_rest c_i (Q_lo + Q_hi). One launch per round binds the
// previous variable into the other buffer and evaluates the current one, one thread per (table, pair).
//
// Cycle phase (log T rounds). With rho the bound address point what remains is eq(r_addr, rho) - already in the
// member's eq scalar - times sum_j eq(r_cycle, j) sum_i c_i (H_i(j)^2 - H_i(j)), H_i(j) = F[addr_i(j)] with one
// F = eq(rho, .) for all d polynomials. Rounds 0 and 1 gather H from the columns (F staged in shared memory up to
// SRC_SMEM_K entries, read through L2 beyond); round 1 binds them into d field tables of T / 2 entries. Every later
// round is one pass over all d tables: per pair and table the bind, then lo^2 - lo and (hi - lo)^2, weighted by c_i
// and the split eq.
#include <cuda_runtime.h>

#include "columns.cuh"
#include "member.hpp"
#include "sources.cuh"

using namespace jb;
using namespace jbi;

namespace {

constexpr int BL_BLOCK = 256;

struct BoolCoef {
    Fr c[BOOL_MAX_POLYS];
};

// The bind of an address round: G under s (linear), Q as (1 - r)^2 lo + r^2 hi.
struct AddrBind {
    BindScalar s;
    Fr r2, omr2;
};

// Where a cycle pass reads and writes: the d columns (d x T addresses) with F, or the field tables in at stride s_in;
// the bound tables go to out at stride s_out.
struct CycleSrc {
    const void* cols;
    int kind;
    uint32_t K;
    size_t T;
    const uint64_t* F;
    int f_smem;  // F is staged in dynamic shared memory
    const uint64_t* in;
    size_t s_in;
    uint64_t* out;
    size_t s_out;
};

__device__ __forceinline__ Fr gather(const CycleSrc& cs, size_t i, size_t j, const uint4* fs) {
    const size_t bytes = cs.kind == SK_U8 ? 1 : 2;
    const uint32_t a = ld_address(static_cast<const uint8_t*>(cs.cols) + i * cs.T * bytes, j, cs.kind);
    if (a >= cs.K) return Fr::zero();  // none (creation refused any other a >= K)
    return cs.f_smem ? elem_from<Fr>(fs[2 * a], fs[2 * a + 1]) : ld_elem<Fr>(cs.F, a);
}

// An address round over the d tables of G and Q, packed at the table length (2P after the bind): G_0 .. G_{d-1} then
// Q_0 .. Q_{d-1}. BIND: the tables of length 4P in gq_in are bound into gq_out first.
template <int ORDER, bool BIND>
__global__ void __launch_bounds__(BL_BLOCK) bool_addr_kernel(const uint64_t* gq_in, uint64_t* gq_out, int d, size_t P,
                                                             const uint64_t* eq_rest, const __grid_constant__ BoolCoef cf,
                                                             AddrBind ab, RoundOut out) {
    __shared__ uint32_t smem[BL_BLOCK / 32 * 2 * 8];
    Fr acc[2] = {Fr::zero(), Fr::zero()};
    const size_t len = 2 * P, in_len = BIND ? 2 * len : len, n = (size_t)d * P;
    const uint64_t* q_in = gq_in + (size_t)d * in_len * 4;
    uint64_t* q_out = gq_out + (size_t)d * len * 4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const size_t i = e / P, y = e - i * P;
        const size_t il = ORDER == ORDER_HIGH_TO_LOW ? y : 2 * y, ih = ORDER == ORDER_HIGH_TO_LOW ? y + P : 2 * y + 1;
        const uint64_t* gi = gq_in + i * in_len * 4;
        const uint64_t* qi = q_in + i * in_len * 4;
        Fr gl, ql, qh;  // (q uses G only through G_lo)
        if (BIND) {
            // entry k of the bound table from the pair (k, k + len) HighToLow, (2k, 2k + 1) LowToHigh
            auto lo = [&](size_t k) { return ORDER == ORDER_HIGH_TO_LOW ? k : 2 * k; };
            auto hi = [&](size_t k) { return ORDER == ORDER_HIGH_TO_LOW ? k + len : 2 * k + 1; };
            gl = bind_pair<false>(ld_elem<Fr>(gi, lo(il)), ld_elem<Fr>(gi, hi(il)), ab.s);
            const Fr gh = bind_pair<false>(ld_elem<Fr>(gi, lo(ih)), ld_elem<Fr>(gi, hi(ih)), ab.s);
            ql = fp_add(fp_mul(ab.omr2, ld_elem<Fr>(qi, lo(il))), fp_mul(ab.r2, ld_elem<Fr>(qi, hi(il))));
            qh = fp_add(fp_mul(ab.omr2, ld_elem<Fr>(qi, lo(ih))), fp_mul(ab.r2, ld_elem<Fr>(qi, hi(ih))));
            uint64_t* go = gq_out + i * len * 4;
            uint64_t* qo = q_out + i * len * 4;
            st_elem(go, il, gl);
            st_elem(go, ih, gh);
            st_elem(qo, il, ql);
            st_elem(qo, ih, qh);
        } else {
            gl = ld_elem<Fr>(gi, il);
            ql = ld_elem<Fr>(qi, il);
            qh = ld_elem<Fr>(qi, ih);
        }
        const Fr w = fp_mul(ld_elem<Fr>(eq_rest, y), cf.c[i]);
        acc[0] = fp_add(acc[0], fp_mul(w, fp_sub(ql, gl)));
        acc[1] = fp_add(acc[1], fp_mul(w, fp_add(ql, qh)));
    }
    block_sum<2>(acc, smem);
    round_epilogue<2>(acc, smem, out);
}

// A cycle round over `P` pairs (after the bind, if any) of all d tables. COLS: the tables are the columns gathered
// through F (round 0 without, round 1 with the bind into cs.out); else the field tables cs.in, bound into cs.out (in
// place HighToLow). q(0) = sum_y w_y sum_i c_i (lo^2 - lo), q(inf) = sum_y w_y sum_i c_i (hi - lo)^2.
template <int ORDER, bool COLS, bool BIND, bool HI4>
__global__ void __launch_bounds__(BL_BLOCK) bool_cycle_kernel(const __grid_constant__ CycleSrc cs, int d, size_t P,
                                                              BindScalar s, EqWeights eqw,
                                                              const __grid_constant__ BoolCoef cf, RoundOut out) {
    extern __shared__ uint4 fs[];
    __shared__ uint32_t smem[BL_BLOCK / 32 * 2 * 8];
    if (COLS && cs.f_smem) {
        for (uint32_t k = threadIdx.x; k < 2 * cs.K; k += blockDim.x) fs[k] = reinterpret_cast<const uint4*>(cs.F)[k];
        __syncthreads();
    }
    Fr acc[2] = {Fr::zero(), Fr::zero()};
    const size_t mask = ((size_t)1 << eqw.in_bits) - 1;
    for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < P; y += (size_t)gridDim.x * blockDim.x) {
        // the entries of the pair: HighToLow y, y + P [, y + 2P, y + 3P]; LowToHigh 2y, 2y + 1 [4y .. 4y + 3]
        const size_t i0 = ORDER == ORDER_HIGH_TO_LOW ? y : (BIND ? 4 : 2) * y;
        const size_t i1 = ORDER == ORDER_HIGH_TO_LOW ? (BIND ? y + 2 * P : y + P) : i0 + 1;
        const size_t i2 = ORDER == ORDER_HIGH_TO_LOW ? y + P : i0 + 2;
        const size_t i3 = ORDER == ORDER_HIGH_TO_LOW ? y + 3 * P : i0 + 3;
        const size_t o0 = ORDER == ORDER_HIGH_TO_LOW ? y : 2 * y;
        const size_t o1 = ORDER == ORDER_HIGH_TO_LOW ? y + P : 2 * y + 1;
        Fr a0 = Fr::zero(), ai = Fr::zero();
        for (int i = 0; i < d; ++i) {
            Fr lo, hi;
            if (COLS) {
                if (BIND) {
                    lo = bind_pair<HI4>(gather(cs, i, i0, fs), gather(cs, i, i1, fs), s);
                    hi = bind_pair<HI4>(gather(cs, i, i2, fs), gather(cs, i, i3, fs), s);
                } else {
                    lo = gather(cs, i, i0, fs);
                    hi = gather(cs, i, i1, fs);
                }
            } else {
                const uint64_t* t = cs.in + (size_t)i * cs.s_in * 4;
                if (ORDER == ORDER_HIGH_TO_LOW) {  // (in place)
                    lo = bind_pair<HI4>(ld_elem_rw<Fr>(t, i0), ld_elem_rw<Fr>(t, i1), s);
                    hi = bind_pair<HI4>(ld_elem_rw<Fr>(t, i2), ld_elem_rw<Fr>(t, i3), s);
                } else {
                    lo = bind_pair<HI4>(ld_elem<Fr>(t, i0), ld_elem<Fr>(t, i1), s);
                    hi = bind_pair<HI4>(ld_elem<Fr>(t, i2), ld_elem<Fr>(t, i3), s);
                }
            }
            if (BIND) {
                uint64_t* o = cs.out + (size_t)i * cs.s_out * 4;
                st_elem(o, o0, lo);
                st_elem(o, o1, hi);
            }
            a0 = fp_add(a0, fp_mul(cf.c[i], fp_sub(fp_sqr(lo), lo)));
            ai = fp_add(ai, fp_mul(cf.c[i], fp_sqr(fp_sub(hi, lo))));
        }
        const Fr wt = fp_mul(ld_elem<Fr>(eqw.e_out, y >> eqw.in_bits), ld_elem<Fr>(eqw.e_in, y & mask));
        acc[0] = fp_add(acc[0], fp_mul(wt, a0));
        acc[1] = fp_add(acc[1], fp_mul(wt, ai));
    }
    block_sum<2>(acc, smem);
    round_epilogue<2>(acc, smem, out);
}

// The terminal bind: two entries left per table, the pair (0, 1) in either order, into entry 0 of out_i. COLS: the
// columns through F (unstaged); else the tables in at stride s_in.
template <bool COLS>
__global__ void __launch_bounds__(32) bool_final_kernel(const __grid_constant__ CycleSrc cs, int d, BindScalar s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d) return;
    Fr lo, hi;
    if (COLS) {
        lo = gather(cs, i, 0, nullptr);
        hi = gather(cs, i, 1, nullptr);
    } else {
        lo = ld_elem_rw<Fr>(cs.in + (size_t)i * cs.s_in * 4, 0);
        hi = ld_elem_rw<Fr>(cs.in + (size_t)i * cs.s_in * 4, 1);
    }
    st_elem(cs.out + (size_t)i * cs.s_out * 4, 0, bind_pair<false>(lo, hi, s));
}

Fr dev_fr(const uint64_t* l) {
    Fr x;
    for (int w = 0; w < 4; ++w) {
        x.v[2 * w] = (uint32_t)l[w];
        x.v[2 * w + 1] = (uint32_t)(l[w] >> 32);
    }
    return x;
}

BoolCoef coefs(const BoolState& bl) {
    BoolCoef cf;
    std::memset(&cf, 0, sizeof cf);
    for (int i = 0; i < bl.d; ++i) cf.c[i] = dev_fr(bl.coeff[i]);
    return cf;
}

CycleSrc cycle_src(const BoolState& bl) {
    CycleSrc cs;
    std::memset(&cs, 0, sizeof cs);
    cs.cols = bl.cols;
    cs.kind = bl.kind;
    cs.K = (uint32_t)bl.K;
    cs.T = bl.T;
    cs.F = bl.F;
    return cs;
}

template <int ORDER, bool COLS, bool BIND, bool HI4>
int launch_cycle(jb_ctx* c, const CycleSrc& cs, int d, size_t P, const BindScalar& s, const EqWeights& eqw,
                 const BoolCoef& cf, RoundOut ro) {
    const size_t smem = cs.f_smem ? (size_t)cs.K * 32 : 0;
    return launch_round(c, bool_cycle_kernel<ORDER, COLS, BIND, HI4>, BL_BLOCK, smem, 8, P, 2, BIND ? 0 : 2, 2,
                        "bool_cycle_kernel launch", ro, cs, d, P, s, eqw, cf);
}

template <int ORDER>
int dispatch_cycle(jb_ctx* c, const CycleSrc& cs, bool cols, bool bind, bool hi4, int d, size_t P, const BindScalar& s,
                   const EqWeights& eqw, const BoolCoef& cf, RoundOut ro) {
    if (cols && !bind) return launch_cycle<ORDER, true, false, false>(c, cs, d, P, s, eqw, cf, ro);
    if (cols) return hi4 ? launch_cycle<ORDER, true, true, true>(c, cs, d, P, s, eqw, cf, ro)
                         : launch_cycle<ORDER, true, true, false>(c, cs, d, P, s, eqw, cf, ro);
    return hi4 ? launch_cycle<ORDER, false, true, true>(c, cs, d, P, s, eqw, cf, ro)
               : launch_cycle<ORDER, false, true, false>(c, cs, d, P, s, eqw, cf, ro);
}

void free_address_tables(jb_ctx* c, BoolState& bl) {
    c->dev_free(bl.gq[0]);
    c->dev_free(bl.gq[1]);
    c->dev_free(bl.eq_rest);
    bl.gq[0] = bl.gq[1] = bl.eq_rest = nullptr;
    bl.klen = 0;
}

}  // namespace

const uint64_t* bool_addr_coord(const BoolState& bl, size_t m) {
    return bl.r_addr.data() + 4 * (bl.order == JB_HIGH_TO_LOW ? m : bl.log_k - 1 - m);
}

void bool_release(jb_member* mem) {
    BoolState* bl = mem->bl;
    if (!bl) return;
    jb_ctx* c = mem->ctx;
    free_address_tables(c, *bl);
    c->dev_free(bl->F);
    c->dev_free(bl->cols);
    c->dev_free(bl->h[0]);
    c->dev_free(bl->h[1]);
    bl->F = nullptr;
    bl->cols = nullptr;
    bl->h[0] = bl->h[1] = nullptr;
}

int bool_create(jb_ctx* c, const void* const* columns, size_t count, int kind, int on_device, size_t T, size_t K,
                const uint64_t* coeffs, const uint64_t* r_addr, const uint64_t* r_cycle, const uint64_t* scale,
                int order, jb_member** out) {
    const char* what = "booleanity";
    if (!columns || !coeffs || !out) return c->fail(JB_ERR_INVALID, "booleanity: null pointer");
    if (count == 0) return c->fail(JB_ERR_INVALID, "booleanity: no columns");
    if (count > (size_t)BOOL_MAX_POLYS) return c->fail(JB_ERR_UNSUPPORTED, "booleanity: at most JB_BOOL_MAX_POLYS columns");
    if (order != JB_HIGH_TO_LOW && order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "booleanity: unknown binding order");
    if (!pow2(K) || K > ((size_t)1 << 16)) return c->fail(JB_ERR_INVALID, "booleanity: K must be a power of two in [1, 2^16]");
    int st = check_one_hot_columns(c, what, kind, T, K, on_device, columns, count);
    if (st != JB_OK) return st;
    if (K * T < 2) return c->fail(JB_ERR_INVALID, "booleanity: K * T must be at least 2");
    const size_t log_k = (size_t)log2_of(K), log_t = (size_t)log2_of(T);
    if ((log_k && !r_addr) || (log_t && !r_cycle)) return c->fail(JB_ERR_INVALID, "booleanity: null point");
    for (size_t i = 0; i < count; ++i)
        if (!canonical_fr(coeffs + 4 * i)) return c->fail(JB_ERR_INVALID, "booleanity: coefficient limbs not canonical");
    for (size_t i = 0; i < log_k; ++i)
        if (!canonical_fr(r_addr + 4 * i)) return c->fail(JB_ERR_INVALID, "booleanity: r_addr limbs not canonical");
    for (size_t i = 0; i < log_t; ++i)
        if (!canonical_fr(r_cycle + 4 * i)) return c->fail(JB_ERR_INVALID, "booleanity: r_cycle limbs not canonical");
    if (scale && !canonical_fr(scale)) return c->fail(JB_ERR_INVALID, "booleanity: scale not canonical");

    // everything the rounds need is allocated here
    jb_member* mem = new_member(c, MemberKind::Booleanity, 2, 1, order, K * T);
    if (!mem) return JB_ERR_OOM;
    BoolState* bl = new (std::nothrow) BoolState();
    if (!bl) {
        delete mem;
        return JB_ERR_OOM;
    }
    mem->bl = bl;
    bl->d = (int)count;
    bl->kind = kind;
    bl->order = order;
    bl->T = T;
    bl->K = K;
    bl->log_k = log_k;
    bl->log_t = log_t;
    std::memcpy(bl->coeff, coeffs, count * 32);
    bl->r_addr.assign(r_addr, r_addr + 4 * log_k);
    bl->rho.reserve(log_k);
    bl->hlen = T;
    const size_t bytes = (size_t)small_kind_bytes(kind), d = count;
    bl->h_stride[0] = std::max<size_t>(T / 2, 1);
    bl->h_stride[1] = std::max<size_t>(T / 4, 1);
    st = c->dev_alloc(&bl->cols, d * T * bytes);
    for (size_t i = 0; i < d && st == JB_OK; ++i)
        st = c->check(cudaMemcpyAsync(static_cast<uint8_t*>(bl->cols) + i * T * bytes, columns[i], T * bytes,
                                      on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream),
                      "booleanity: column copy");
    if (st == JB_OK) st = c->dev_alloc((void**)&bl->F, K * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&bl->h[0], d * bl->h_stride[0] * 32);
    if (st == JB_OK && order == JB_LOW_TO_HIGH) st = c->dev_alloc((void**)&bl->h[1], d * bl->h_stride[1] * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&bl->gq[0], 2 * d * K * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&bl->gq[1], 2 * d * (K / 2) * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&bl->eq_rest, (K - 1) * 32);
    // eq over the address coordinates after round m's: HighToLow r_addr[m + 1 ..), LowToHigh r_addr[.. log_k - 1 - m)
    for (size_t m = 0; m < log_k && st == JB_OK; ++m)
        st = eq_build(c, order == JB_HIGH_TO_LOW ? r_addr + 4 * (m + 1) : r_addr, log_k - 1 - m, nullptr,
                      bl->eq_rest + 4 * (K - (K >> m)));
    // G from the pushforward (which also finds an address >= K that is not none), Q = G
    if (st == JB_OK) {
        const void* dcols[BOOL_MAX_POLYS];
        uint64_t* g[BOOL_MAX_POLYS];
        for (size_t i = 0; i < d; ++i) {
            dcols[i] = static_cast<const uint8_t*>(bl->cols) + i * T * bytes;
            g[i] = bl->gq[0] + i * K * 4;
        }
        st = one_hot_pushforward_into(c, dcols, d, kind, T, K, r_cycle, g);
    }
    if (st == JB_OK)
        st = c->check(cudaMemcpyAsync(bl->gq[0] + d * K * 4, bl->gq[0], d * K * 32, cudaMemcpyDeviceToDevice, c->stream),
                      "booleanity: Q copy");
    bl->klen = K;
    if (st == JB_OK && log_k == 0) st = bool_begin_cycles(mem, nullptr);
    // (the borrowed columns have been read: the pushforward waited for the device)
    if (st != JB_OK) {  // (the caller holds the context lock: no jb_member_destroy here)
        bool_release(mem);
        delete bl;
        delete mem;
        return st;
    }
    *out = mem;
    return JB_OK;
}

int bool_address_pass(jb_member* mem, const uint64_t* bind, size_t m, RoundOut ro) {
    jb_ctx* c = mem->ctx;
    BoolState& bl = *mem->bl;
    AddrBind ab;
    std::memset(&ab, 0, sizeof ab);
    size_t len = bl.klen;
    if (bind) {
        bool hi4;
        ab.s = make_scalar(bind, &hi4);
        const HostFr r = HostFr::from_limbs(bind), omr = HostFr::one() - r;
        uint64_t l[4];
        (r * r).store(l);
        ab.r2 = dev_fr(l);
        (omr * omr).store(l);
        ab.omr2 = dev_fr(l);
        len /= 2;
    }
    const size_t P = len / 2;
    const uint64_t* eq_rest = bl.eq_rest + 4 * (bl.K - (bl.K >> m));
    const uint64_t* in = bl.gq[bl.gq_cur];
    uint64_t* out = bl.gq[bl.gq_cur ^ 1];
    const size_t items = (size_t)bl.d * P;
    const BoolCoef cf = coefs(bl);
    int st;
#define JB_BOOL_ADDR(O, B)                                                                                             \
    launch_round(c, bool_addr_kernel<O, B>, BL_BLOCK, 0, 8, items, 2, B ? 0 : 2, 2, "bool_addr_kernel launch", ro, in,  \
                 out, bl.d, P, eq_rest, cf, ab)
    if (mem->order == JB_HIGH_TO_LOW) st = bind ? JB_BOOL_ADDR(ORDER_HIGH_TO_LOW, true) : JB_BOOL_ADDR(ORDER_HIGH_TO_LOW, false);
    else st = bind ? JB_BOOL_ADDR(ORDER_LOW_TO_HIGH, true) : JB_BOOL_ADDR(ORDER_LOW_TO_HIGH, false);
#undef JB_BOOL_ADDR
    if (st != JB_OK || !bind) return st;
    bl.rho.insert(bl.rho.end(), bind, bind + 4);
    bl.gq_cur ^= 1;
    bl.klen = len;
    mem->len /= 2;
    return JB_OK;
}

int bool_begin_cycles(jb_member* mem, const uint64_t* last) {
    jb_ctx* c = mem->ctx;
    BoolState& bl = *mem->bl;
    if (last) {
        bl.rho.insert(bl.rho.end(), last, last + 4);
        mem->len /= 2;
    }
    // rho in binding order -> the address point MSB first (LowToHigh bound the LSB first)
    std::vector<uint64_t> pt(4 * bl.log_k);
    for (size_t m = 0; m < bl.log_k; ++m) {
        const size_t at = mem->order == JB_HIGH_TO_LOW ? m : bl.log_k - 1 - m;
        std::memcpy(pt.data() + 4 * at, bl.rho.data() + 4 * m, 32);
    }
    const int st = eq_build(c, pt.data(), bl.log_k, nullptr, bl.F);
    free_address_tables(c, bl);  // (stream-ordered: after the last pass has read them)
    return st;
}

int bool_cycle_pass(jb_member* mem, const uint64_t* bind, const EqWeights& eqw, RoundOut ro) {
    jb_ctx* c = mem->ctx;
    BoolState& bl = *mem->bl;
    bool hi4 = false;
    BindScalar s;
    std::memset(&s, 0, sizeof s);
    size_t len = bl.hlen;
    if (bind) {
        s = make_scalar(bind, &hi4);
        len /= 2;
    }
    const size_t P = len / 2;
    const bool cols = bl.cols != nullptr;
    const bool l2h = mem->order == JB_LOW_TO_HIGH;
    CycleSrc cs = cycle_src(bl);
    int next = bl.h_cur;
    if (cols) {
        cs.f_smem = bl.K <= SRC_SMEM_K ? 1 : 0;
        next = 0;
    } else {
        cs.in = bl.h[bl.h_cur];
        cs.s_in = bl.h_stride[bl.h_cur];
        next = l2h ? bl.h_cur ^ 1 : bl.h_cur;
    }
    cs.out = bl.h[next];
    cs.s_out = bl.h_stride[next];
    const BoolCoef cf = coefs(bl);
    const int st = l2h ? dispatch_cycle<ORDER_LOW_TO_HIGH>(c, cs, cols, bind != nullptr, hi4, bl.d, P, s, eqw, cf, ro)
                       : dispatch_cycle<ORDER_HIGH_TO_LOW>(c, cs, cols, bind != nullptr, hi4, bl.d, P, s, eqw, cf, ro);
    if (st != JB_OK || !bind) return st;
    if (cols) {
        c->dev_free(bl.cols);  // (stream-ordered: freed after the pass has read them)
        bl.cols = nullptr;
    }
    bl.h_cur = next;
    bl.hlen = len;
    mem->len /= 2;
    return JB_OK;
}

int bool_finish(jb_member* mem, const uint64_t r[4]) {
    jb_ctx* c = mem->ctx;
    BoolState& bl = *mem->bl;
    bool hi4;
    const BindScalar s = make_scalar(r, &hi4);
    CycleSrc cs = cycle_src(bl);
    int next = 0;
    if (bl.klen) {  // T = 1: G (packed at length 2) holds ra_i(rho, 0) once its last variable is bound
        cs.in = bl.gq[bl.gq_cur];
        cs.s_in = 2;
    } else if (!bl.cols) {
        cs.in = bl.h[bl.h_cur];
        cs.s_in = bl.h_stride[bl.h_cur];
        next = mem->order == JB_LOW_TO_HIGH ? bl.h_cur ^ 1 : bl.h_cur;
    }
    cs.out = bl.h[next];
    cs.s_out = bl.h_stride[next];
    if (bl.cols && !bl.klen) bool_final_kernel<true><<<1, 32, 0, c->stream>>>(cs, bl.d, s);
    else bool_final_kernel<false><<<1, 32, 0, c->stream>>>(cs, bl.d, s);
    c->launches++;
    const int st = c->check(cudaGetLastError(), "bool_final_kernel launch");
    if (st != JB_OK) return st;
    if (bl.klen) free_address_tables(c, bl);
    c->dev_free(bl.cols);
    bl.cols = nullptr;
    bl.h_cur = next;
    bl.hlen = 1;
    return JB_OK;
}

const uint64_t* bool_final_entry(const jb_member* mem, int i) {
    const BoolState& bl = *mem->bl;
    return bl.h[bl.h_cur] + (size_t)i * bl.h_stride[bl.h_cur] * 4;
}
