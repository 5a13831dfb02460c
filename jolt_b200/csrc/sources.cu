// The source pass of expression members over sources (jb_member_create_expr_sources): rounds 0 and 1 of a member
// some of whose tables are still witness columns in their own format -
//   * COMPACT: primitive integers (small_scalar.cuh), value F::from(v) (promote_small);
//   * ONE_HOT: an address column (columns.cuh), value eq(r_addr, addr[j]) gathered from the source's K-entry eq table
//     (staged in shared memory for K <= SRC_SMEM_K, read through L2 beyond), 0 for the none value;
//   * TABLE: a field table, loaded as expr_round_kernel loads it.
// Round 0 reads the sources; round 1 reads them again, binds them into the len/2 field tables the member allocated
// at creation and sweeps the bound pairs. The sweep itself (points, monomials, split-eq weight) is expr_sweep, the
// one expr_round_kernel runs, so both passes publish the same values: a bound compact or one-hot entry is
// bind_pair(F(lo), F(hi)), exactly the entry jb_table_upload_small / a gathered table would hold after its bind.
#include <cuda_runtime.h>

#include <algorithm>

#include "columns.cuh"
#include "member.hpp"
#include "sources.cuh"

using namespace jb;
using namespace jbi;

namespace {

// the largest dynamic shared memory of a launch: the columns and block-sum scratch of 8 tables, 8 staged eq tables
constexpr size_t SRC_SMEM_MAX = expr_smem_bytes(EXPR_MAX_TABLES) + (size_t)EXPR_MAX_TABLES * SRC_SMEM_K * 32;

// What the pass reads for each table j of the member. The type of a table is uniform over the grid.
struct SourceParams {
    static constexpr int ADDRESS_WIDEST = SK_U16;  // expression members over sources: u8 / u16 addresses
    const void* values[EXPR_MAX_TABLES];  // COMPACT / ONE_HOT column
    const uint64_t* eq[EXPR_MAX_TABLES];  // ONE_HOT: eq(r_addr, .) in global memory
    uint32_t K[EXPR_MAX_TABLES];
    uint32_t smem[EXPR_MAX_TABLES];       // ONE_HOT: word offset of the staged eq table in dynamic shared memory
    uint8_t type[EXPR_MAX_TABLES];        // JB_SOURCE_*
    uint8_t kind[EXPR_MAX_TABLES];
};

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

// Flags an address >= K that is not the none value. U8: a u8 column; else `kind` (SK_U16 / SK_U32) at run time.
template <bool U8>
__global__ void __launch_bounds__(256) check_addresses_kernel(const void* addr, size_t n, int kind, uint32_t K,
                                                              unsigned int* bad) {
    bool b = false;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t a = ld_address<SK_U32>(addr, i, U8 ? SK_U8 : kind);
        b |= a != NO_ADDRESS && a >= K;
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
                   const SourceParams& sp, size_t smem, const RoundOut& out) {
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
    return launch_round(c, kernel, EXPR_BLOCK, smem, per_sm, pairs, EXPR_MAX_POINTS, BIND ? 0 : 2, ex.D,
                        "source_round_kernel launch", out, tp, pairs, s, ex, sp);
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
    SourceParams sp;
    fill_params(mem, false, sp);
    TablePtrs tp;
    std::memset(&tp, 0, sizeof tp);
    return finish_sources(mem, r, sp, tp);
}

void sources_release(jb_member* mem) {
    for (SourceCol& sc : mem->src) {
        mem->ctx->dev_free(sc.values);
        mem->ctx->dev_free(sc.eq);
    }
    mem->src.clear();
}

int sources_one_hot_eq(jb_ctx* c, SourceCol& sc, size_t len, const uint64_t* r_addr, size_t log_k, unsigned int* d_flag) {
    int st = c->dev_alloc((void**)&sc.eq, (size_t)sc.K * 32);
    if (st == JB_OK) st = eq_build(c, r_addr, log_k, nullptr, sc.eq);
    if (st != JB_OK) return st;
    const unsigned grid = launch_grid(c, len, 256, 8);
    if (sc.kind == SK_U8)
        check_addresses_kernel<true><<<grid, 256, 0, c->stream>>>(sc.values, len, sc.kind, sc.K, d_flag);
    else
        check_addresses_kernel<false><<<grid, 256, 0, c->stream>>>(sc.values, len, sc.kind, sc.K, d_flag);
    c->launches++;
    return c->check(cudaGetLastError(), "check_addresses_kernel launch");
}
