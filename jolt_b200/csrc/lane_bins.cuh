// Exact field sums in bins of 8 u64 lanes, one lane per 32-bit limb: adding a canonical element adds each limb (< 2^32)
// into its lane with an integer atomic, so a lane holds up to 2^32 - 1 additions, and the result is independent of
// their order (bit-exact and deterministic whatever the schedule). bins_to_fr_kernel turns bins into field elements.
// Internal to the translation units that include it.
#pragma once
#include "field.cuh"

namespace {

using namespace jb;

constexpr int BINS_BLOCK = 256;

// Warp-aggregated bin update: every thread with emit adds its field value `v` (8 canonical limbs) to bin `key`.
__device__ __forceinline__ void pf_flush(bool emit, uint32_t key, const Fr& v, unsigned long long* bins, int lane) {
    const unsigned m = __ballot_sync(0xffffffffu, emit);
    if (!emit) return;
    const unsigned peers = __match_any_sync(m, key);
    const int leader = __ffs(peers) - 1;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const uint32_t lo = __reduce_add_sync(peers, v.v[w] & 0xffffu);
        const uint32_t hi = __reduce_add_sync(peers, v.v[w] >> 16);
        if (lane == leader) atomicAdd(bins + (size_t)key * 8 + w, (unsigned long long)lo + ((unsigned long long)hi << 16));
    }
}

// n bins of 8 u64 limb-sum lanes -> canonical Montgomery elements (the lanes hold sums of Montgomery values, so the
// integer they encode is reduced mod p, not Montgomery-reduced): V = lo + top 2^256, V mod p = (lo mod p) + top R.
__global__ void __launch_bounds__(BINS_BLOCK) bins_to_fr_kernel(const unsigned long long* lanes, size_t n, uint64_t* out) {
    for (size_t i = (size_t)blockIdx.x * BINS_BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * BINS_BLOCK) {
        Fr lo, top = Fr::zero();
        unsigned long long carry = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const unsigned long long v = lanes[i * 8 + w];
            const unsigned long long s = (v & 0xffffffffull) + (carry & 0xffffffffull);
            lo.v[w] = (uint32_t)s;
            carry = (v >> 32) + (carry >> 32) + (s >> 32);
        }
        top.v[0] = (uint32_t)carry;
        top.v[1] = (uint32_t)(carry >> 32);
#pragma unroll
        for (int k = 0; k < 5; ++k) cond_sub_p<FrParams>(lo.v);  // lo < 2^256 < 6p
        st_elem(out, i, fp_add(lo, fp_mul(top, Fr::r2())));  // top < 2^64 < p: montmul(top, R^2) = top R mod p
    }
}

}  // namespace
