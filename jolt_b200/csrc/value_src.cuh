// Weighted value loaders of the row-walking kernels (mle_eval.cu, vmp.cu): A += e * v(i) UNREDUCED into a 17-word
// register accumulator, for a field table (a 256 x 256 product) and a compact column of KIND (a 256 x 32w product of the
// magnitude). Compact values are plain integers, so sum e~ v comes out as R * sum e v, not in the R^2 domain of the
// field product. Internal to the translation units that include it.
#pragma once
#include "field.cuh"
#include "small_scalar.cuh"

namespace {

using namespace jb;

struct FieldSrc {
    static constexpr int SMEM_U4 = 1;
    __device__ void init(uint4*) const {}
    __device__ __forceinline__ void acc(uint32_t (&A)[17], const Fr& e, const void* p, size_t i, const uint4*) const {
        const Fr v = ld_elem<Fr>(static_cast<const uint64_t*>(p), i);
        mul_wide_acc_reg(A, e.v, v.v);
    }
};

template <int KIND>
struct SmallSrc {
    static constexpr int SMEM_U4 = 1;
    // 32-bit words of the magnitude
    static constexpr int BW = KIND <= SK_U32 ? 1 : (KIND == SK_U64 || KIND == SK_I64 || KIND == SK_S64) ? 2 : 4;
    __device__ void init(uint4*) const {}
    __device__ __forceinline__ void acc(uint32_t (&A)[17], const Fr& e, const void* p, size_t i, const uint4*) const {
        uint32_t mag[4];
        const bool neg = ld_small(p, i, KIND, mag);
        if (neg) {  // (p - e~) |v|: the Montgomery form of -e times |v|, still an exact non-negative integer product
            uint32_t ne[8];
            const uint32_t pm[8] = {FrParams::P(0), FrParams::P(1), FrParams::P(2), FrParams::P(3),
                                    FrParams::P(4), FrParams::P(5), FrParams::P(6), FrParams::P(7)};
            sub8(ne, pm, e.v);
            mul_wide_acc_bw<BW>(A, ne, mag);
        } else {
            mul_wide_acc_bw<BW>(A, e.v, mag);
        }
    }
};

}  // namespace
