// The per-entry load of a member's source before its bind and the terminal bind from the columns, shared by the
// passes that read sources in their own format (sources.cu, product.cu). A pass's parameter struct SP carries, per
// table j: values[j] (the COMPACT / ONE_HOT column), eq[j] (ONE_HOT: eq(r_addr, .) in global memory), K[j], smem[j] (ONE_HOT: word offset of the eq
// table staged in dynamic shared memory, or SRC_NO_SMEM), type[j] (JB_SOURCE_*) and kind[j], and SP::ADDRESS_WIDEST,
// the widest address kind its one-hot sources may have (columns.cuh): SK_U16 for the expression pass, whose source
// pass sits at the register budget, SK_U32 for the product pass, so product members reach RAM-sized K.
#pragma once
#include <cstring>

#include "columns.cuh"
#include "member.hpp"
#include "poly_kernels.cuh"

namespace jb {

constexpr uint32_t SRC_SMEM_K = 256;  // a one-hot source's eq table may be staged in shared memory up to 8 KiB
constexpr uint32_t SRC_NO_SMEM = 0xffffffffu;

// Entry i of the compact or one-hot source j.
template <class SP>
__device__ __forceinline__ Fr src_value(const SP& sp, int j, size_t i, const uint32_t* dsm) {
    if (sp.type[j] == JB_SOURCE_COMPACT) {
        uint32_t mag[4];
        const bool neg = ld_small(sp.values[j], i, sp.kind[j], mag);
        return promote_small(mag, neg);
    }
    const uint32_t a = ld_address<SP::ADDRESS_WIDEST>(sp.values[j], i, sp.kind[j]);
    if (a >= sp.K[j]) return Fr::zero();  // none (NO_ADDRESS; creation refused any other a >= K)
    if (sp.smem[j] != SRC_NO_SMEM) {
        const uint4* s = reinterpret_cast<const uint4*>(dsm + sp.smem[j]);
        return elem_from<Fr>(s[2 * a], s[2 * a + 1]);
    }
    return ld_elem<Fr>(sp.eq[j], a);
}

// The terminal bind of a member whose sources are unbound: tp.out_j[i] = lo + s (hi - lo) for every compact / one-hot
// source j < ntables (the field tables are bound by bind_table).
template <class SP, class TP, int ORDER>
__global__ void __launch_bounds__(256) source_bind_kernel(const __grid_constant__ SP sp, int ntables,
                                                          const __grid_constant__ TP tp, size_t half, BindScalar s) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x)
        for (int j = 0; j < ntables; ++j) {
            if (sp.type[j] == JB_SOURCE_TABLE) continue;
            const size_t il = ORDER == ORDER_HIGH_TO_LOW ? i : 2 * i, ih = ORDER == ORDER_HIGH_TO_LOW ? i + half : 2 * i + 1;
            st_elem(tp.out[j], i, bind_pair<false>(src_value(sp, j, il, nullptr), src_value(sp, j, ih, nullptr), s));
        }
}

// The terminal bind (len = 2) of a member whose sources are still unbound, whatever pass structs SP / TP carry them (sp
// filled from mem->src with nothing staged; tp's out pointers are set here): every field table through bind_table, every
// column through source_bind_kernel, then the columns are released.
template <class SP, class TP>
int finish_sources(jb_member* mem, const uint64_t r[4], const SP& sp, TP& tp) {
    jb_ctx* c = mem->ctx;
    const size_t half = mem->len / 2;
    const int T = mem->ntables();
    for (int j = 0; j < T; ++j) {
        if (mem->src[j].type == JB_SOURCE_TABLE) {
            int st = jbi::bind_table(c, mem->tables[j], r, mem->order);
            if (st != JB_OK) return st;
        } else {
            tp.out[j] = mem->tables[j].buf;
        }
    }
    bool hi4;
    const BindScalar s = jbi::make_scalar(r, &hi4);
    const unsigned grid = launch_grid(c, half, 256, 4);
    if (mem->order == JB_LOW_TO_HIGH)
        source_bind_kernel<SP, TP, ORDER_LOW_TO_HIGH><<<grid, 256, 0, c->stream>>>(sp, T, tp, half, s);
    else
        source_bind_kernel<SP, TP, ORDER_HIGH_TO_LOW><<<grid, 256, 0, c->stream>>>(sp, T, tp, half, s);
    c->launches++;
    int st = c->check(cudaGetLastError(), "source_bind_kernel launch");
    if (st != JB_OK) return st;
    for (int j = 0; j < T; ++j) mem->tables[j].len = half;
    sources_release(mem);
    return JB_OK;
}

}  // namespace jb
