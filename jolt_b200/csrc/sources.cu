// The source pass of expression members over sources (jb_member_create_expr_sources): rounds 0 and 1 of a member
// some of whose tables are still witness columns in their own format -
//   * COMPACT: primitive integers (small_scalar.cuh), value F::from(v) (promote_small);
//   * ONE_HOT: an address column, value eq(r_addr, addr[j]) gathered from the source's K-entry eq table (staged in
//     shared memory for K <= SRC_SMEM_K, read through L2 beyond), 0 for the none value;
//   * TABLE: a field table, loaded as expr_round_kernel loads it.
// Round 0 reads the sources; round 1 reads them again, binds them into the len/2 field tables the member allocated
// at creation and sweeps the bound pairs. The sweep itself (points, monomials, split-eq weight) is expr_sweep, the
// one expr_round_kernel runs, so both passes publish the same values: a bound compact or one-hot entry is
// bind_pair(F(lo), F(hi)), exactly the entry jb_table_upload_small / a gathered table would hold after its bind.
#include <cuda_runtime.h>

#include <algorithm>

#include "member.hpp"
#include "small_scalar.cuh"

using namespace jb;
using namespace jbi;

namespace {

constexpr uint32_t SRC_SMEM_K = 256;  // a one-hot source's eq table is staged in shared memory up to 8 KiB
constexpr uint32_t SRC_NO_SMEM = 0xffffffffu;
// the largest dynamic shared memory of a launch: the columns and block-sum scratch of 8 tables, 8 staged eq tables
constexpr size_t SRC_SMEM_MAX = expr_smem_bytes(EXPR_MAX_TABLES) + (size_t)EXPR_MAX_TABLES * SRC_SMEM_K * 32;

// What the pass reads for each table j of the member. The type of a table is uniform over the grid.
struct SourceParams {
    const void* values[EXPR_MAX_TABLES];  // COMPACT / ONE_HOT column
    const uint64_t* eq[EXPR_MAX_TABLES];  // ONE_HOT: eq(r_addr, .) in global memory
    uint32_t K[EXPR_MAX_TABLES];
    uint32_t smem[EXPR_MAX_TABLES];       // ONE_HOT: word offset of the staged eq table in dynamic shared memory
    uint8_t type[EXPR_MAX_TABLES];        // JB_SOURCE_*
    uint8_t kind[EXPR_MAX_TABLES];
};

// Entry i of the compact or one-hot source j.
__device__ __forceinline__ Fr src_value(const SourceParams& sp, int j, size_t i, const uint32_t* dsm) {
    if (sp.type[j] == JB_SOURCE_COMPACT) {
        uint32_t mag[4];
        const bool neg = ld_small(sp.values[j], i, sp.kind[j], mag);
        return promote_small(mag, neg);
    }
    const bool u8 = sp.kind[j] == SK_U8;
    const uint32_t a = u8 ? (uint32_t)static_cast<const uint8_t*>(sp.values[j])[i]
                          : (uint32_t)static_cast<const uint16_t*>(sp.values[j])[i];
    if (a == (u8 ? 0xffu : 0xffffu) || a >= sp.K[j]) return Fr::zero();  // none (creation refused other a >= K)
    if (sp.smem[j] != SRC_NO_SMEM) {
        const uint4* s = reinterpret_cast<const uint4*>(dsm + sp.smem[j]);
        return elem_from<Fr>(s[2 * a], s[2 * a + 1]);
    }
    return ld_elem<Fr>(sp.eq[j], a);
}

// expr_round_kernel with step 1 loading each table by its source type (same launch shape, columns and budget).
// BIND (round 1): a source table is bound from its column into tp.out[j] (the member's len/2 buffer); a field
// table is bound as in expr_round_kernel (in place HighToLow, ping-pong LowToHigh).
template <int ORDER, bool BIND, bool HI4, bool WEIGHTED>
__global__ void __launch_bounds__(EXPR_BLOCK, 4)
    source_round_kernel(const __grid_constant__ TablePtrs tp, size_t pairs, BindScalar s,
                        const __grid_constant__ ExprParams ex, const __grid_constant__ SourceParams sp, RoundOut out) {
    extern __shared__ uint32_t dsm[];
    uint32_t* col = dsm + threadIdx.x;
    uint32_t* red = dsm + (size_t)ex.ntables * 16 * EXPR_BLOCK;
    for (int j = 0; j < ex.ntables; ++j)
        if (sp.type[j] == JB_SOURCE_ONE_HOT && sp.smem[j] != SRC_NO_SMEM)
            for (uint32_t i = threadIdx.x; i < 2 * sp.K[j]; i += blockDim.x)
                reinterpret_cast<uint4*>(dsm + sp.smem[j])[i] = reinterpret_cast<const uint4*>(sp.eq[j])[i];
    __syncthreads();
    Fr acc[EXPR_MAX_POINTS];
#pragma unroll
    for (int e = 0; e < EXPR_MAX_POINTS; ++e) acc[e] = Fr::zero();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < pairs; y += stride) {
        const size_t yn = y + stride;
        if (yn < pairs) {
            for (int j = 0; j < ex.ntables; ++j) {
                if (sp.type[j] != JB_SOURCE_TABLE) continue;  // (a column entry is 1-24 bytes: the lines are shared)
                if (ORDER == ORDER_HIGH_TO_LOW) {
                    prefetch_l2(tp.in[j], yn);
                    prefetch_l2(tp.in[j], yn + pairs);
                    if (BIND) {
                        prefetch_l2(tp.in[j], yn + 2 * pairs);
                        prefetch_l2(tp.in[j], yn + 3 * pairs);
                    }
                } else {
                    prefetch_l2(tp.in[j], (BIND ? 4 : 2) * yn);
                }
            }
        }
        // the entries of the pair: HighToLow y, y + P [, y + 2P, y + 3P]; LowToHigh 2y, 2y + 1 [4y .. 4y + 3]
        const size_t i0 = ORDER == ORDER_HIGH_TO_LOW ? y : (BIND ? 4 : 2) * y;
        const size_t i1 = ORDER == ORDER_HIGH_TO_LOW ? (BIND ? y + 2 * pairs : y + pairs) : i0 + 1;
        const size_t i2 = ORDER == ORDER_HIGH_TO_LOW ? y + pairs : i0 + 2;
        const size_t i3 = ORDER == ORDER_HIGH_TO_LOW ? y + 3 * pairs : i0 + 3;
        const size_t o0 = ORDER == ORDER_HIGH_TO_LOW ? y : 2 * y;
        const size_t o1 = ORDER == ORDER_HIGH_TO_LOW ? y + pairs : 2 * y + 1;
        for (int j = 0; j < ex.ntables; ++j) {
            Fr lo, hi;
            if (sp.type[j] == JB_SOURCE_TABLE) {
                const uint64_t* in = tp.in[j];
                if (BIND) {
                    if (ORDER == ORDER_HIGH_TO_LOW) {
                        lo = bind_pair<HI4>(ld_elem_rw<Fr>(in, i0), ld_elem_rw<Fr>(in, i1), s);
                        hi = bind_pair<HI4>(ld_elem_rw<Fr>(in, i2), ld_elem_rw<Fr>(in, i3), s);
                    } else {
                        lo = bind_pair<HI4>(ld_elem<Fr>(in, i0), ld_elem<Fr>(in, i1), s);
                        hi = bind_pair<HI4>(ld_elem<Fr>(in, i2), ld_elem<Fr>(in, i3), s);
                    }
                } else if (ORDER == ORDER_HIGH_TO_LOW) {
                    lo = ld_elem_rw<Fr>(in, i0);
                    hi = ld_elem_rw<Fr>(in, i1);
                } else {
                    lo = ld_elem<Fr>(in, i0);
                    hi = ld_elem<Fr>(in, i1);
                }
            } else if (BIND) {
                lo = bind_pair<HI4>(src_value(sp, j, i0, dsm), src_value(sp, j, i1, dsm), s);
                hi = bind_pair<HI4>(src_value(sp, j, i2, dsm), src_value(sp, j, i3, dsm), s);
            } else {
                lo = src_value(sp, j, i0, dsm);
                hi = src_value(sp, j, i1, dsm);
            }
            if (BIND) {
                st_elem(tp.out[j], o0, lo);
                st_elem(tp.out[j], o1, hi);
            }
            expr_st(col, 16 * j, lo);
            expr_st(col, 16 * j + 8, fp_sub(hi, lo));
        }
        expr_sweep<WEIGHTED>(col, ex, tp, y, acc);
    }
    block_sum<EXPR_MAX_POINTS>(acc, red);
    round_epilogue<EXPR_MAX_POINTS>(acc, red, out);
}

// The terminal bind of a member whose sources are unbound: out_j[i] = lo + s (hi - lo) for every compact / one-hot
// source (the field tables are bound by bind_table).
template <int ORDER>
__global__ void __launch_bounds__(256) source_bind_kernel(const __grid_constant__ SourceParams sp, int ntables,
                                                          const __grid_constant__ TablePtrs tp, size_t half,
                                                          BindScalar s) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x)
        for (int j = 0; j < ntables; ++j) {
            if (sp.type[j] == JB_SOURCE_TABLE) continue;
            const size_t il = ORDER == ORDER_HIGH_TO_LOW ? i : 2 * i, ih = ORDER == ORDER_HIGH_TO_LOW ? i + half : 2 * i + 1;
            st_elem(tp.out[j], i, bind_pair<false>(src_value(sp, j, il, nullptr), src_value(sp, j, ih, nullptr), s));
        }
}

// Flags an address >= K that is not the none value.
template <class A>
__global__ void __launch_bounds__(256) check_addresses_kernel(const A* addr, size_t n, uint32_t K, unsigned int* bad) {
    const uint32_t none = (uint32_t)(A)~(A)0;
    bool b = false;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t a = addr[i];
        b |= a != none && a >= K;
    }
    if (b) atomicOr(bad, 1u);
}

// Shared memory of a launch: the expression columns and scratch, then the staged eq tables (offsets into sp.smem).
size_t fill_params(const jb_member* mem, bool staged, SourceParams& sp) {
    std::memset(&sp, 0, sizeof sp);
    const int T = mem->ntables();
    size_t words = expr_smem_bytes(T) / 4;
    for (int j = 0; j < T; ++j) {
        const SourceCol& sc = mem->src[j];
        sp.type[j] = (uint8_t)sc.type;
        sp.kind[j] = (uint8_t)sc.kind;
        sp.values[j] = sc.values;
        sp.eq[j] = sc.eq;
        sp.K[j] = sc.K;
        sp.smem[j] = SRC_NO_SMEM;
        if (staged && sc.type == JB_SOURCE_ONE_HOT && sc.K <= SRC_SMEM_K) {
            sp.smem[j] = (uint32_t)words;
            words += (size_t)sc.K * 8;
        }
    }
    return words * 4;
}

template <int ORDER, bool BIND, bool HI4, bool WEIGHTED>
int launch_sources(jb_ctx* c, const TablePtrs& tp, size_t pairs, const BindScalar& s, const ExprParams& ex,
                   const SourceParams& sp, size_t smem, RoundOut out) {
    auto kernel = source_round_kernel<ORDER, BIND, HI4, WEIGHTED>;
    static const bool attr = [&] {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SRC_SMEM_MAX);
        return true;
    }();
    (void)attr;
    // (two launches per member: the occupancy query is not worth caching by shared-memory size)
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, EXPR_BLOCK, smem) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    size_t need = (pairs + EXPR_BLOCK - 1) / EXPR_BLOCK;
    size_t resident = (size_t)c->sm_count * per_sm;
    size_t grid = need < resident ? need : resident;
    if (grid < 1) grid = 1;
    int st = c->ensure_partial(grid * EXPR_MAX_POINTS);
    if (st != JB_OK) return st;
    out.partial = c->d_partial;
    int tix = c->timing_begin(BIND ? 0 : 2, pairs, ex.D);
    const unsigned block = pairs <= 32 ? 32u : (unsigned)EXPR_BLOCK;
    kernel<<<(unsigned)grid, block, smem, c->stream>>>(tp, pairs, s, ex, sp, out);
    c->timing_end(tix);
    c->launches++;
    return c->check(cudaGetLastError(), "source_round_kernel launch");
}

template <int ORDER, bool WEIGHTED>
int dispatch_sources2(jb_ctx* c, const TablePtrs& tp, size_t pairs, bool bind, bool hi4, const BindScalar& s,
                      const ExprParams& ex, const SourceParams& sp, size_t smem, const RoundOut& out) {
    if (!bind) return launch_sources<ORDER, false, false, WEIGHTED>(c, tp, pairs, s, ex, sp, smem, out);
    return hi4 ? launch_sources<ORDER, true, true, WEIGHTED>(c, tp, pairs, s, ex, sp, smem, out)
               : launch_sources<ORDER, true, false, WEIGHTED>(c, tp, pairs, s, ex, sp, smem, out);
}

}  // namespace

int sources_round(jb_ctx* c, const jb_member* mem, bool weighted, const TablePtrs& tp, size_t pairs, bool bind,
                  const BindScalar& s, const ExprParams& ex, RoundOut out) {
    SourceParams sp;
    const size_t smem = fill_params(mem, true, sp);
    const bool hi4 = (s.w[0] | s.w[1] | s.w[2] | s.w[3]) == 0;  // the 125-bit challenge [0, 0, lo, hi] (make_scalar)
    if (mem->order == JB_LOW_TO_HIGH)
        return weighted ? dispatch_sources2<ORDER_LOW_TO_HIGH, true>(c, tp, pairs, bind, hi4, s, ex, sp, smem, out)
                        : dispatch_sources2<ORDER_LOW_TO_HIGH, false>(c, tp, pairs, bind, hi4, s, ex, sp, smem, out);
    return weighted ? dispatch_sources2<ORDER_HIGH_TO_LOW, true>(c, tp, pairs, bind, hi4, s, ex, sp, smem, out)
                    : dispatch_sources2<ORDER_HIGH_TO_LOW, false>(c, tp, pairs, bind, hi4, s, ex, sp, smem, out);
}

int sources_finish(jb_member* mem, const uint64_t r[4]) {
    jb_ctx* c = mem->ctx;
    const size_t half = mem->len / 2;
    SourceParams sp;
    fill_params(mem, false, sp);
    TablePtrs tp;
    std::memset(&tp, 0, sizeof tp);
    for (int j = 0; j < mem->ntables(); ++j) {
        if (mem->src[j].type == JB_SOURCE_TABLE) {
            int st = bind_table(c, mem->tables[j], r, mem->order);
            if (st != JB_OK) return st;
        } else {
            tp.out[j] = mem->tables[j].buf;
        }
    }
    bool hi4;
    const BindScalar s = make_scalar(r, &hi4);
    const unsigned grid = (unsigned)std::min<size_t>((half + 255) / 256, (size_t)c->sm_count * 4);
    if (mem->order == JB_LOW_TO_HIGH)
        source_bind_kernel<ORDER_LOW_TO_HIGH><<<grid, 256, 0, c->stream>>>(sp, mem->ntables(), tp, half, s);
    else
        source_bind_kernel<ORDER_HIGH_TO_LOW><<<grid, 256, 0, c->stream>>>(sp, mem->ntables(), tp, half, s);
    c->launches++;
    int st = c->check(cudaGetLastError(), "source_bind_kernel launch");
    if (st != JB_OK) return st;
    for (int j = 0; j < mem->ntables(); ++j) mem->tables[j].len = half;
    sources_release(mem);
    return JB_OK;
}

void sources_release(jb_member* mem) {
    for (SourceCol& sc : mem->src) {
        mem->ctx->dev_free(sc.values);
        mem->ctx->dev_free(sc.eq);
    }
    mem->src.clear();
}

int sources_copy_column(jb_ctx* c, const void* values, size_t bytes, int on_device, void** out) {
    int st = c->dev_alloc(out, bytes);
    if (st != JB_OK) return st;
    return c->check(cudaMemcpyAsync(*out, values, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                                    c->stream),
                    "expr sources: column copy");
}

int sources_one_hot_eq(jb_ctx* c, SourceCol& sc, size_t len, const uint64_t* r_addr, size_t log_k, unsigned int* d_flag) {
    int st = c->dev_alloc((void**)&sc.eq, (size_t)sc.K * 32);
    if (st == JB_OK) st = eq_build(c, r_addr, log_k, nullptr, sc.eq);
    if (st != JB_OK) return st;
    const unsigned grid = (unsigned)std::min<size_t>((len + 255) / 256, (size_t)c->sm_count * 8);
    if (sc.kind == SK_U8)
        check_addresses_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const uint8_t*>(sc.values), len, sc.K, d_flag);
    else
        check_addresses_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const uint16_t*>(sc.values), len, sc.K, d_flag);
    c->launches++;
    return c->check(cudaGetLastError(), "check_addresses_kernel launch");
}
