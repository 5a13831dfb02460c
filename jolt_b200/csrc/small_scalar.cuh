// Small-scalar encodings shared by the compact-table kernels (compact.cu) and the small-scalar MSM
// (msm.cu). The reference keeps most witness columns as primitive integers - `Polynomial<T>` with
// T in {bool, u8, u16, u32, u64, u128, i64, i128} (crates/jolt-poly/src/dense.rs:22-142), legacy
// MultilinearPolynomial::{U8Scalars .. I128Scalars} (crates/jolt-prover-legacy/src/msm/mod.rs:27-79) -
// and promotes with Ring::from_u64 / from_i64 / from_u128 / from_i128
// (crates/jolt-field/src/bn254/mod.rs:265-298): value mod r, negatives as r - |v|.
#pragma once
#include "field.cuh"

namespace jb {

// numeric values of jb_scalar_kind (include/jolt_b200.h)
constexpr int SK_FR = 0, SK_U8 = 1, SK_U16 = 2, SK_U32 = 3, SK_U64 = 4, SK_U128 = 5, SK_I64 = 6, SK_I128 = 7;
// sign-magnitude integers: jolt_field::signed::{S64, S128} = SignedBigInt<1>, SignedBigInt<2>
// (crates/jolt-field/src/signed.rs:25-32; legacy msm_s64 / msm_s128, crates/jolt-prover-legacy/src/msm/mod.rs:140-158;
// MultilinearPolynomial::S128Scalars, poly/multilinear_polynomial.rs:33). Records of N u64 magnitude limbs followed by
// one sign byte (is_positive), padded to a multiple of 8: jb_s64 = 16 bytes, jb_s128 = 24 bytes (include/jolt_b200.h).
// "Zero is not canonicalized" (signed.rs:16-17): -0 is 0.
constexpr int SK_S64 = 8, SK_S128 = 9;
constexpr int SK_LAST = SK_S128;

__host__ __device__ inline int small_kind_bytes(int kind) {
    switch (kind) {
        case SK_U8: return 1;
        case SK_U16: return 2;
        case SK_U32: return 4;
        case SK_U64: case SK_I64: return 8;
        case SK_U128: case SK_I128: return 16;
        case SK_S64: return 16;   // record stride (8 magnitude + 1 sign + 7 padding)
        case SK_S128: return 24;  // (16 magnitude + 1 sign + 7 padding)
        default: return 0;
    }
}

// bits of the magnitude (|i64::MIN| = 2^63 needs 64 bits, |i128::MIN| = 2^127 needs 128)
__host__ __device__ inline int small_kind_bits(int kind) {
    switch (kind) {
        case SK_U8: return 8;
        case SK_U16: return 16;
        case SK_U32: return 32;
        case SK_U64: case SK_I64: case SK_S64: return 64;
        case SK_U128: case SK_I128: case SK_S128: return 128;
        default: return 254;
    }
}

// values[i] as sign + magnitude: mag = |v| in four little-endian 32-bit words; returns v < 0.
__device__ __forceinline__ bool ld_small(const void* values, size_t i, int kind, uint32_t mag[4]) {
    uint64_t lo = 0, hi = 0;
    bool neg = false;
    switch (kind) {
        case SK_U8: lo = ((const uint8_t*)values)[i]; break;
        case SK_U16: lo = ((const uint16_t*)values)[i]; break;
        case SK_U32: lo = ((const uint32_t*)values)[i]; break;
        case SK_U64: lo = ((const uint64_t*)values)[i]; break;
        case SK_U128:
            lo = ((const uint64_t*)values)[2 * i];
            hi = ((const uint64_t*)values)[2 * i + 1];
            break;
        case SK_I64: {
            const uint64_t v = ((const uint64_t*)values)[i];
            neg = (v >> 63) != 0;
            lo = neg ? (0ull - v) : v;  // unsigned_abs
            break;
        }
        case SK_I128: {
            lo = ((const uint64_t*)values)[2 * i];
            hi = ((const uint64_t*)values)[2 * i + 1];
            neg = (hi >> 63) != 0;
            if (neg) {  // two's-complement negate over 128 bits
                lo = ~lo + 1ull;
                hi = ~hi + (lo == 0 ? 1ull : 0ull);
            }
            break;
        }
        case SK_S64: {
            lo = ((const uint64_t*)values)[2 * i];
            neg = (((const uint64_t*)values)[2 * i + 1] & 0xffull) == 0;  // is_positive == false
            break;
        }
        case SK_S128: {
            lo = ((const uint64_t*)values)[3 * i];
            hi = ((const uint64_t*)values)[3 * i + 1];
            neg = (((const uint64_t*)values)[3 * i + 2] & 0xffull) == 0;
            break;
        }
        default: break;
    }
    if ((lo | hi) == 0) neg = false;  // -0 (representable by the sign-magnitude kinds) is 0
    mag[0] = (uint32_t)lo;
    mag[1] = (uint32_t)(lo >> 32);
    mag[2] = (uint32_t)hi;
    mag[3] = (uint32_t)(hi >> 32);
    return neg;
}

// F::from(v) of a value as ld_small returns it (canonical Montgomery form)
__device__ __forceinline__ Fr promote_small(const uint32_t mag[4], bool neg) {
    Fr k = Fr::zero();
#pragma unroll
    for (int j = 0; j < 4; ++j) k.v[j] = mag[j];
    Fr m = fp_to_mont(k);  // |v| < 2^128 < r: already canonical as an integer
    return neg ? fp_neg(m) : m;
}

}  // namespace jb
