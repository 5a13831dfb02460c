// A/B variant of the eval-only sweep (degree 2, s(1) from the claim): evaluation blocks are STAGED INTO SHARED
// MEMORY by the TMA unit - cp.async.bulk (1-D bulk copies, SASS UBLKCP) issued by a producer warp and tracked by
// mbarriers - instead of being loaded by every thread with 128-bit LDGs. BASELINE.json's north_star names "TMA
// staging of evaluation blocks into shared memory"; r01 argued against it without building it. This builds it so the
// choice is a measurement (tools/tma_ab.py):
//   * 8 compute warps + 1 producer warp; a ring of STAGES tiles of TILE = 256 pair indices (one per compute thread);
//     a tile holds, per table, the TILE pairs' lo and hi elements (LowToHigh: one contiguous 16 KiB run;
//     HighToLow: two 8 KiB runs);
//   * producer: wait empty[s] -> arrive.expect_tx(full[s], bytes) -> cp.async.bulk ... mbarrier::complete_tx::bytes;
//   * compute: wait full[s] -> LDS the thread's operands -> the same two wide products as fused_pass -> arrive
//     empty[s]. No landing registers for global loads, no software pipelining, no L2 prefetch instructions.
// The block reduction and the round epilogue are fused_pass's.
#pragma once
#include "bulk_copy.cuh"
#include "poly_kernels.cuh"

namespace jb {

constexpr int TMA_TILE = 256;
constexpr int TMA_STAGES = 2;
constexpr int TMA_THREADS = 256 + 32;

__device__ __forceinline__ Fr lds_elem(const uint8_t* p) {
    Fr r;
    const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + 16);
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}

struct TmaShape {
    static constexpr size_t tile_bytes = (size_t)2 * TMA_TILE * 64;          // two tables, lo + hi per pair
    static constexpr size_t acc_words = (size_t)2 * 17 * 256;                 // K = 2 wide accumulators per thread
    static constexpr size_t smem_bytes = TMA_STAGES * tile_bytes + (acc_words + 8 * 2 * 8) * 4 + 2 * TMA_STAGES * 8 + 128;
};

template <int ORDER>
__global__ void __launch_bounds__(TMA_THREADS, 2) eval2_tma_kernel(TablePtrs tp, size_t pairs, RoundOut out) {
    constexpr int K = 2;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    uint8_t* tiles = smem_raw;                                                     // [stage][table][TILE * 64]
    uint32_t* wacc = reinterpret_cast<uint32_t*>(smem_raw + TMA_STAGES * TmaShape::tile_bytes);
    uint32_t* red = wacc + TmaShape::acc_words;
    uint64_t* full = reinterpret_cast<uint64_t*>(red + 8 * K * 8);
    uint64_t* empty = full + TMA_STAGES;
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int s = 0; s < TMA_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 256);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < 256) {
#pragma unroll
        for (int e = 0; e < K; ++e)
#pragma unroll
            for (int w = 0; w < 17; ++w) wacc[(e * 17 + w) * 256 + tid] = 0;
    }
    __syncthreads();
    const size_t ntiles = (pairs + TMA_TILE - 1) / TMA_TILE;
    if (tid >= 256) {
        // ---- producer warp: one lane drives the TMA unit -----------------------------------------------------
        if (tid == 256) {
            unsigned it = 0;
            for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
                const int s = it % TMA_STAGES;
                const unsigned phase = (it / TMA_STAGES) & 1;
                mbar_wait(&empty[s], phase ^ 1);
                const size_t y0 = t * TMA_TILE;
                const unsigned valid = (unsigned)(pairs - y0 < (size_t)TMA_TILE ? pairs - y0 : (size_t)TMA_TILE);
                mbar_expect_tx(&full[s], valid * 64 * 2);
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    uint8_t* dst = tiles + (size_t)s * TmaShape::tile_bytes + (size_t)j * TMA_TILE * 64;
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(tp.in[j]);
                    if (ORDER == ORDER_LOW_TO_HIGH) {
                        bulk_g2s(dst, src + y0 * 64, valid * 64, &full[s]);
                    } else {
                        bulk_g2s(dst, src + y0 * 32, valid * 32, &full[s]);
                        bulk_g2s(dst + TMA_TILE * 32, src + (y0 + pairs) * 32, valid * 32, &full[s]);
                    }
                }
            }
        }
    } else {
        // ---- compute warps ------------------------------------------------------------------------------------
        unsigned it = 0;
        for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
            const int s = it % TMA_STAGES;
            const unsigned phase = (it / TMA_STAGES) & 1;
            mbar_wait(&full[s], phase);
            const size_t y = t * TMA_TILE + tid;
            if (y < pairs) {
                Fr lo[2], hi[2];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const uint8_t* base = tiles + (size_t)s * TmaShape::tile_bytes + (size_t)j * TMA_TILE * 64;
                    if (ORDER == ORDER_LOW_TO_HIGH) {
                        lo[j] = lds_elem(base + tid * 64);
                        hi[j] = lds_elem(base + tid * 64 + 32);
                    } else {
                        lo[j] = lds_elem(base + tid * 32);
                        hi[j] = lds_elem(base + TMA_TILE * 32 + tid * 32);
                    }
                }
                mul_wide_acc_smem(wacc + (0 * 17) * 256 + tid, 256, lo[0].v, lo[1].v);
                const Fr d0 = fp_sub_lazy(hi[0], lo[0]), d1 = fp_sub_lazy(hi[1], lo[1]);
                mul_wide_acc_smem(wacc + (1 * 17) * 256 + tid, 256, d0.v, d1.v);
            }
            mbar_arrive(&empty[s]);
        }
    }
    // ---- block reduction (as fused_pass) + round epilogue -------------------------------------------------------
    __syncthreads();
    Fr acc[K];
    uint64_t* colsum = reinterpret_cast<uint64_t*>(red);
    const int lane = tid & 31, warp = tid >> 5;
    if (warp < 8) {
        for (int c = warp; c < K * 17; c += 8) {
            uint64_t sacc = 0;
            for (int t2 = lane; t2 < 256; t2 += 32) sacc += wacc[c * 256 + t2];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) sacc += __shfl_down_sync(0xffffffffu, sacc, off);
            if (lane == 0) colsum[c] = sacc;
        }
    }
    __syncthreads();
    if (warp == 0) {
        Fr mine = Fr::zero();
        if (lane < K) {
            uint32_t Tw[17];
            uint64_t carry = 0;
#pragma unroll
            for (int w = 0; w < 17; ++w) {
                const uint64_t t2 = colsum[lane * 17 + w] + carry;
                Tw[w] = (uint32_t)t2;
                carry = t2 >> 32;
            }
            mine = reduce_wide17<FrParams>(Tw, 1);
        }
#pragma unroll
        for (int e = 0; e < K; ++e)
#pragma unroll
            for (int w = 0; w < 8; ++w) acc[e].v[w] = __shfl_sync(0xffffffffu, mine.v[w], e);
    }
    __syncthreads();
    round_epilogue<K>(acc, red, out);
}

}  // namespace jb
