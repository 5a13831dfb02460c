// BN254 Fr / Fq Montgomery arithmetic for sm_90a, one element per thread, 8 x u32 limbs in
// registers (memory layout = the reference's 4 x u64 little-endian Montgomery limbs,
// crates/jolt-field/src/bn254/mod.rs:33-42; R = 2^256).
//
// Multiplication is word-serial Montgomery (CIOS) with the partial products split into an
// "even" and an "odd" column accumulator so that every a[j]*b_i lo/hi pair lands in adjacent
// limbs of ONE carry chain; ptxas fuses each mad.lo.cc/madc.hi.cc pair on the same operands
// into a single IMAD.WIDE.U32 (+carry), i.e. 8 wide IMADs per 8x1 row instead of 16.
// Frame: T = sum X[k] 2^(32k) + sum Y[k] 2^(32(k+1)).  After the reduction row X[0] == 0 and the
// frame shifts one limb: X' = Y, Y'[k] = X[k+2], X'[0] += X[1]  (pure register renaming).
//
// Both moduli have two spare bits (p < 2^254, 4p < R), so the un-subtracted product of
// operands < 2p stays < 2p ("lazy" variants below); public results are always fully reduced.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace jb {

struct FrParams {
    __host__ __device__ static constexpr uint32_t P(int i) {
        constexpr uint32_t t[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u,
                                      0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return t[i];
    }
    static constexpr uint32_t INV = 0xefffffffu;  // -p^-1 mod 2^32
    // R mod p (Montgomery one)
    __host__ __device__ static constexpr uint32_t ONE(int i) {
        constexpr uint32_t t[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u,
                                        0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return t[i];
    }
    // R^2 mod p
    __host__ __device__ static constexpr uint32_t R2(int i) {
        constexpr uint32_t t[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u,
                                       0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
        return t[i];
    }
};

struct FqParams {
    __host__ __device__ static constexpr uint32_t P(int i) {
        constexpr uint32_t t[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u,
                                      0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return t[i];
    }
    static constexpr uint32_t INV = 0xe4866389u;
    __host__ __device__ static constexpr uint32_t ONE(int i) {
        constexpr uint32_t t[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u,
                                        0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return t[i];
    }
    __host__ __device__ static constexpr uint32_t R2(int i) {
        constexpr uint32_t t[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u,
                                       0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
        return t[i];
    }
};

template <class PR>
struct Fp {
    uint32_t v[8];

    __device__ __forceinline__ static Fp zero() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.v[i] = 0;
        return r;
    }
    __device__ __forceinline__ static Fp one() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.v[i] = PR::ONE(i);
        return r;
    }
    __device__ __forceinline__ static Fp r2() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.v[i] = PR::R2(i);
        return r;
    }
    __device__ __forceinline__ bool is_zero() const {
        return (v[0] | v[1] | v[2] | v[3] | v[4] | v[5] | v[6] | v[7]) == 0;
    }
    __device__ __forceinline__ bool operator==(const Fp& o) const {
        uint32_t d = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) d |= v[i] ^ o.v[i];
        return d == 0;
    }
};

// ---- carry-chain primitives (each chain is ONE asm statement: the CC flag never crosses
// statements, so the compiler cannot schedule a flag-clobbering instruction in between) ------

// r = a + b (8 limbs), returns nothing: caller guarantees no carry out (operands < 2^255).
template <class PR>
__device__ __forceinline__ void add8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    asm("add.cc.u32 %0, %8, %16;\n\t"
        "addc.cc.u32 %1, %9, %17;\n\t"
        "addc.cc.u32 %2, %10, %18;\n\t"
        "addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t"
        "addc.cc.u32 %5, %13, %21;\n\t"
        "addc.cc.u32 %6, %14, %22;\n\t"
        "addc.u32 %7, %15, %23;"
        : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
          "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
}

// r = a - b (8 limbs); returns the borrow (0 or 0xffffffff).
__device__ __forceinline__ uint32_t sub8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]),
          "=r"(borrow)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
          "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
    return borrow;
}

// x in [0, 2p) -> [0, p)
template <class PR>
__device__ __forceinline__ void cond_sub_p(uint32_t* x) {
    uint32_t t[8];
    const uint32_t p[8] = {PR::P(0), PR::P(1), PR::P(2), PR::P(3), PR::P(4), PR::P(5), PR::P(6), PR::P(7)};
    uint32_t borrow = sub8(t, x, p);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = borrow ? x[i] : t[i];
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_add(const Fp<PR>& a, const Fp<PR>& b) {
    Fp<PR> r;
    add8<PR>(r.v, a.v, b.v);
    cond_sub_p<PR>(r.v);
    return r;
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_sub(const Fp<PR>& a, const Fp<PR>& b) {
    Fp<PR> r;
    uint32_t borrow = sub8(r.v, a.v, b.v);
    uint32_t pm[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) pm[i] = PR::P(i) & borrow;
    add8<PR>(r.v, r.v, pm);  // wraps mod 2^256 exactly when borrow was set
    return r;
}

// a - b + p in (0, 2p): no data-dependent select ("lazy" difference, feeds fp_mul_lazy).
template <class PR>
__device__ __forceinline__ Fp<PR> fp_sub_lazy(const Fp<PR>& a, const Fp<PR>& b) {
    Fp<PR> r;
    uint32_t t[8];
    const uint32_t p[8] = {PR::P(0), PR::P(1), PR::P(2), PR::P(3), PR::P(4), PR::P(5), PR::P(6), PR::P(7)};
    add8<PR>(t, a.v, p);
    sub8(r.v, t, b.v);
    return r;
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_neg(const Fp<PR>& a) {
    Fp<PR> r;
    const uint32_t p[8] = {PR::P(0), PR::P(1), PR::P(2), PR::P(3), PR::P(4), PR::P(5), PR::P(6), PR::P(7)};
    sub8(r.v, p, a.v);
    bool z = a.is_zero();
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = z ? 0u : r.v[i];
    return r;
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_dbl(const Fp<PR>& a) {
    return fp_add(a, a);
}

// ---- multiplication rows ---------------------------------------------------------------------

// First row: X = a_even * b, Y = a_odd * b   (no addends).
__device__ __forceinline__ void row_first(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t b) {
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
        asm("mul.lo.u32 %0, %2, %3;\n\tmul.hi.u32 %1, %2, %3;" : "=r"(X[j]), "=r"(X[j + 1]) : "r"(a[j]), "r"(b));
        asm("mul.lo.u32 %0, %2, %3;\n\tmul.hi.u32 %1, %2, %3;" : "=r"(Y[j]), "=r"(Y[j + 1]) : "r"(a[j + 1]), "r"(b));
    }
}

// X[0..7] += a_even * b (one chain), carry out added into Y[7].
__device__ __forceinline__ void row_even(uint32_t* X, uint32_t* Y, uint32_t a0, uint32_t a2, uint32_t a4,
                                         uint32_t a6, uint32_t b) {
    asm("mad.lo.cc.u32 %0, %9, %13, %0;\n\t"
        "madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
        "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
        "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
        "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
        "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(X[0]), "+r"(X[1]), "+r"(X[2]), "+r"(X[3]), "+r"(X[4]), "+r"(X[5]), "+r"(X[6]), "+r"(X[7]),
          "+r"(Y[7])
        : "r"(a0), "r"(a2), "r"(a4), "r"(a6), "r"(b));
}

// Y[0..7] += a_odd * b (one chain). No carry out by the T < 2^288 bound.
__device__ __forceinline__ void row_odd(uint32_t* Y, uint32_t a1, uint32_t a3, uint32_t a5, uint32_t a7,
                                        uint32_t b) {
    asm("mad.lo.cc.u32 %0, %8, %12, %0;\n\t"
        "madc.hi.cc.u32 %1, %8, %12, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t"
        "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "madc.lo.cc.u32 %4, %10, %12, %4;\n\t"
        "madc.hi.cc.u32 %5, %10, %12, %5;\n\t"
        "madc.lo.cc.u32 %6, %11, %12, %6;\n\t"
        "madc.hi.u32 %7, %11, %12, %7;"
        : "+r"(Y[0]), "+r"(Y[1]), "+r"(Y[2]), "+r"(Y[3]), "+r"(Y[4]), "+r"(Y[5]), "+r"(Y[6]), "+r"(Y[7])
        : "r"(a1), "r"(a3), "r"(a5), "r"(a7), "r"(b));
}

// Frame shift fused with the odd product row:
//   Xn = Y (caller renames), Xn[0] += X[1] (carry into Yn[0]),
//   Yn[k] = X[k+2] + (a_odd * b)[k]   (X[8] = X[9] = 0).
__device__ __forceinline__ void row_shift_odd(uint32_t* Yn, uint32_t& Xn0, const uint32_t* X, uint32_t a1,
                                              uint32_t a3, uint32_t a5, uint32_t a7, uint32_t b) {
    asm("add.cc.u32 %8, %8, %9;\n\t"
        "madc.lo.cc.u32 %0, %16, %20, %10;\n\t"
        "madc.hi.cc.u32 %1, %16, %20, %11;\n\t"
        "madc.lo.cc.u32 %2, %17, %20, %12;\n\t"
        "madc.hi.cc.u32 %3, %17, %20, %13;\n\t"
        "madc.lo.cc.u32 %4, %18, %20, %14;\n\t"
        "madc.hi.cc.u32 %5, %18, %20, %15;\n\t"
        "madc.lo.cc.u32 %6, %19, %20, 0;\n\t"
        "madc.hi.u32 %7, %19, %20, 0;"
        : "=r"(Yn[0]), "=r"(Yn[1]), "=r"(Yn[2]), "=r"(Yn[3]), "=r"(Yn[4]), "=r"(Yn[5]), "=r"(Yn[6]), "=r"(Yn[7]),
          "+r"(Xn0)
        : "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]), "r"(X[7]), "r"(a1), "r"(a3), "r"(a5),
          "r"(a7), "r"(b));
}

// One full word-step after the first: shift frame, add a*b_i, add m*p. On exit X[0] == 0.
template <class PR>
__device__ __forceinline__ void mont_step(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
    uint32_t Yn[8];
    // new X is the old Y; new Y is built from old X[2..7] plus the odd products
    row_shift_odd(Yn, Y[0], X, a[1], a[3], a[5], a[7], bi);
#pragma unroll
    for (int k = 0; k < 8; ++k) { X[k] = Y[k]; Y[k] = Yn[k]; }
    row_even(X, Y, a[0], a[2], a[4], a[6], bi);
    uint32_t m = X[0] * PR::INV;
    row_even(X, Y, PR::P(0), PR::P(2), PR::P(4), PR::P(6), m);
    row_odd(Y, PR::P(1), PR::P(3), PR::P(5), PR::P(7), m);
}

template <class PR>
__device__ __forceinline__ void mont_first(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t b0) {
    row_first(X, Y, a, b0);
    uint32_t m = X[0] * PR::INV;
    row_even(X, Y, PR::P(0), PR::P(2), PR::P(4), PR::P(6), m);
    row_odd(Y, PR::P(1), PR::P(3), PR::P(5), PR::P(7), m);
}

// out = (X >> 32) + (Y << 0 in the shifted frame): out[k] = X[k+1] + Y[k]; result < 2p.
__device__ __forceinline__ void mont_merge(uint32_t* out, const uint32_t* X, const uint32_t* Y) {
    asm("add.cc.u32 %0, %8, %15;\n\t"
        "addc.cc.u32 %1, %9, %16;\n\t"
        "addc.cc.u32 %2, %10, %17;\n\t"
        "addc.cc.u32 %3, %11, %18;\n\t"
        "addc.cc.u32 %4, %12, %19;\n\t"
        "addc.cc.u32 %5, %13, %20;\n\t"
        "addc.cc.u32 %6, %14, %21;\n\t"
        "addc.u32 %7, 0, %22;"
        : "=r"(out[0]), "=r"(out[1]), "=r"(out[2]), "=r"(out[3]), "=r"(out[4]), "=r"(out[5]), "=r"(out[6]),
          "=r"(out[7])
        : "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]), "r"(X[7]), "r"(Y[0]), "r"(Y[1]),
          "r"(Y[2]), "r"(Y[3]), "r"(Y[4]), "r"(Y[5]), "r"(Y[6]), "r"(Y[7]));
}

// Montgomery product, result in [0, 2p) for operands in [0, 2p).
template <class PR>
__device__ __forceinline__ Fp<PR> fp_mul_lazy(const Fp<PR>& a, const Fp<PR>& b) {
    uint32_t X[8], Y[8];
    mont_first<PR>(X, Y, a.v, b.v[0]);
#pragma unroll
    for (int i = 1; i < 8; ++i) mont_step<PR>(X, Y, a.v, b.v[i]);
    Fp<PR> r;
    mont_merge(r.v, X, Y);
    return r;
}

// Fully reduced Montgomery product.
template <class PR>
__device__ __forceinline__ Fp<PR> fp_mul(const Fp<PR>& a, const Fp<PR>& b) {
    Fp<PR> r = fp_mul_lazy(a, b);
    cond_sub_p<PR>(r.v);
    return r;
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_sqr(const Fp<PR>& a) {
    return fp_mul(a, a);
}

// Product with a multiplier whose four LOW 32-bit words are zero - the reference's 125-bit
// sumcheck challenge, Montgomery limbs [0, 0, lo, hi] (crates/jolt-field/src/bn254/mod.rs:254;
// legacy mul_by_hi_2limbs, crates/jolt-prover-legacy/src/field/challenge/macros.rs:274-283).
// The four zero rows of the word-serial product are identities, so only rows 4..7 run:
// montmul(a, [0,0,lo,hi]) == a * (lo + hi 2^64) * 2^-128.  `hi4` = words 4..7 of the multiplier.
template <class PR>
__device__ __forceinline__ Fp<PR> fp_mul_hi4_lazy(const Fp<PR>& a, const uint32_t* hi4) {
    uint32_t X[8], Y[8];
    mont_first<PR>(X, Y, a.v, hi4[0]);
#pragma unroll
    for (int i = 1; i < 4; ++i) mont_step<PR>(X, Y, a.v, hi4[i]);
    Fp<PR> r;
    mont_merge(r.v, X, Y);
    return r;
}

template <class PR>
__device__ __forceinline__ Fp<PR> fp_mul_hi4(const Fp<PR>& a, const uint32_t* hi4) {
    Fp<PR> r = fp_mul_hi4_lazy(a, hi4);
    cond_sub_p<PR>(r.v);
    return r;
}

// Montgomery -> canonical integer limbs (multiply by 1) and back (multiply by R^2).
template <class PR>
__device__ __forceinline__ Fp<PR> fp_from_mont(const Fp<PR>& a) {
    Fp<PR> one_raw = Fp<PR>::zero();
    one_raw.v[0] = 1;
    return fp_mul(a, one_raw);
}
template <class PR>
__device__ __forceinline__ Fp<PR> fp_to_mont(const Fp<PR>& a) {
    return fp_mul(a, Fp<PR>::r2());
}

// ---- deferred-reduction accumulation (the GPU counterpart of the reference's WideAccumulator,
// crates/jolt-field/src/bn254/mont.rs:565-602): acc += a * b as a plain 512-bit integer product of the
// Montgomery limbs, E collecting the lo/hi pairs that start at even limb positions and O (weight
// shifted by one limb) those that start at odd positions - every row is two 4-pair carry chains; ONE
// Montgomery reduction at the end turns the sum of products into the field sum.

// r[0..7] += (a0,a1,a2,a3) * b as four adjacent lo/hi pairs in one carry chain; the carry out is
// added into `top` (the word above r[7]).
__device__ __forceinline__ void chain8_top(uint32_t* r, uint32_t& top, uint32_t a0, uint32_t a1, uint32_t a2,
                                           uint32_t a3, uint32_t b) {
    asm("mad.lo.cc.u32 %0, %9, %13, %0;\n\t"
        "madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
        "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
        "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
        "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
        "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]), "+r"(top)
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b));
}
// Shared-memory form: the 544-bit accumulator lives at acc[k * stride] (k = 0..16; one column per
// thread, so accesses are conflict-free) and is only in registers while a product is merged - this
// is what lets the fused round kernel run at three blocks per SM. Operands may be lazy (< 2p):
// 17 words hold > 2^30 such products.
__device__ __forceinline__ void mul_wide_acc_smem(uint32_t* acc, int stride, const uint32_t* a, const uint32_t* b) {
    uint32_t E[17], O[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
        chain8_top(E + i, E[i + 8], a[0], a[2], a[4], a[6], b[i]);
        chain8_top(O + i, O[i + 8], a[1], a[3], a[5], a[7], b[i]);
        chain8_top(O + i, O[i + 8], a[0], a[2], a[4], a[6], b[i + 1]);
        chain8_top(E + i + 2, E[i + 10], a[1], a[3], a[5], a[7], b[i + 1]);
    }
    uint32_t A[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) A[k] = acc[k * stride];
    asm("add.cc.u32 %0, %0, %17;\n\t"
        "addc.cc.u32 %1, %1, %18;\n\t"
        "addc.cc.u32 %2, %2, %19;\n\t"
        "addc.cc.u32 %3, %3, %20;\n\t"
        "addc.cc.u32 %4, %4, %21;\n\t"
        "addc.cc.u32 %5, %5, %22;\n\t"
        "addc.cc.u32 %6, %6, %23;\n\t"
        "addc.cc.u32 %7, %7, %24;\n\t"
        "addc.cc.u32 %8, %8, %25;\n\t"
        "addc.cc.u32 %9, %9, %26;\n\t"
        "addc.cc.u32 %10, %10, %27;\n\t"
        "addc.cc.u32 %11, %11, %28;\n\t"
        "addc.cc.u32 %12, %12, %29;\n\t"
        "addc.cc.u32 %13, %13, %30;\n\t"
        "addc.cc.u32 %14, %14, %31;\n\t"
        "addc.cc.u32 %15, %15, %32;\n\t"
        "addc.u32 %16, %16, 0;"
        : "+r"(A[0]), "+r"(A[1]), "+r"(A[2]), "+r"(A[3]), "+r"(A[4]), "+r"(A[5]), "+r"(A[6]), "+r"(A[7]),
          "+r"(A[8]), "+r"(A[9]), "+r"(A[10]), "+r"(A[11]), "+r"(A[12]), "+r"(A[13]), "+r"(A[14]), "+r"(A[15]),
          "+r"(A[16])
        : "r"(E[0]), "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]),
          "r"(E[9]), "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E[15]));
    asm("add.cc.u32 %0, %0, %16;\n\t"
        "addc.cc.u32 %1, %1, %17;\n\t"
        "addc.cc.u32 %2, %2, %18;\n\t"
        "addc.cc.u32 %3, %3, %19;\n\t"
        "addc.cc.u32 %4, %4, %20;\n\t"
        "addc.cc.u32 %5, %5, %21;\n\t"
        "addc.cc.u32 %6, %6, %22;\n\t"
        "addc.cc.u32 %7, %7, %23;\n\t"
        "addc.cc.u32 %8, %8, %24;\n\t"
        "addc.cc.u32 %9, %9, %25;\n\t"
        "addc.cc.u32 %10, %10, %26;\n\t"
        "addc.cc.u32 %11, %11, %27;\n\t"
        "addc.cc.u32 %12, %12, %28;\n\t"
        "addc.cc.u32 %13, %13, %29;\n\t"
        "addc.cc.u32 %14, %14, %30;\n\t"
        "addc.u32 %15, %15, 0;"
        : "+r"(A[1]), "+r"(A[2]), "+r"(A[3]), "+r"(A[4]), "+r"(A[5]), "+r"(A[6]), "+r"(A[7]), "+r"(A[8]),
          "+r"(A[9]), "+r"(A[10]), "+r"(A[11]), "+r"(A[12]), "+r"(A[13]), "+r"(A[14]), "+r"(A[15]), "+r"(A[16])
        : "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]), "r"(O[6]), "r"(O[7]), "r"(O[8]),
          "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]));
#pragma unroll
    for (int k = 0; k < 17; ++k) acc[k * stride] = A[k];
}

// Register form: A[0..16] += a * b (plain 512-bit product of the limbs; operands may be lazy, < 2p).
__device__ __forceinline__ void mul_wide_acc_reg(uint32_t (&A)[17], const uint32_t* a, const uint32_t* b) {
    uint32_t E[17], O[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
        chain8_top(E + i, E[i + 8], a[0], a[2], a[4], a[6], b[i]);
        chain8_top(O + i, O[i + 8], a[1], a[3], a[5], a[7], b[i]);
        chain8_top(O + i, O[i + 8], a[0], a[2], a[4], a[6], b[i + 1]);
        chain8_top(E + i + 2, E[i + 10], a[1], a[3], a[5], a[7], b[i + 1]);
    }
    asm("add.cc.u32 %0, %0, %17;\n\t"
        "addc.cc.u32 %1, %1, %18;\n\t"
        "addc.cc.u32 %2, %2, %19;\n\t"
        "addc.cc.u32 %3, %3, %20;\n\t"
        "addc.cc.u32 %4, %4, %21;\n\t"
        "addc.cc.u32 %5, %5, %22;\n\t"
        "addc.cc.u32 %6, %6, %23;\n\t"
        "addc.cc.u32 %7, %7, %24;\n\t"
        "addc.cc.u32 %8, %8, %25;\n\t"
        "addc.cc.u32 %9, %9, %26;\n\t"
        "addc.cc.u32 %10, %10, %27;\n\t"
        "addc.cc.u32 %11, %11, %28;\n\t"
        "addc.cc.u32 %12, %12, %29;\n\t"
        "addc.cc.u32 %13, %13, %30;\n\t"
        "addc.cc.u32 %14, %14, %31;\n\t"
        "addc.cc.u32 %15, %15, %32;\n\t"
        "addc.u32 %16, %16, 0;"
        : "+r"(A[0]), "+r"(A[1]), "+r"(A[2]), "+r"(A[3]), "+r"(A[4]), "+r"(A[5]), "+r"(A[6]), "+r"(A[7]),
          "+r"(A[8]), "+r"(A[9]), "+r"(A[10]), "+r"(A[11]), "+r"(A[12]), "+r"(A[13]), "+r"(A[14]), "+r"(A[15]),
          "+r"(A[16])
        : "r"(E[0]), "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]),
          "r"(E[9]), "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E[15]));
    asm("add.cc.u32 %0, %0, %16;\n\t"
        "addc.cc.u32 %1, %1, %17;\n\t"
        "addc.cc.u32 %2, %2, %18;\n\t"
        "addc.cc.u32 %3, %3, %19;\n\t"
        "addc.cc.u32 %4, %4, %20;\n\t"
        "addc.cc.u32 %5, %5, %21;\n\t"
        "addc.cc.u32 %6, %6, %22;\n\t"
        "addc.cc.u32 %7, %7, %23;\n\t"
        "addc.cc.u32 %8, %8, %24;\n\t"
        "addc.cc.u32 %9, %9, %25;\n\t"
        "addc.cc.u32 %10, %10, %26;\n\t"
        "addc.cc.u32 %11, %11, %27;\n\t"
        "addc.cc.u32 %12, %12, %28;\n\t"
        "addc.cc.u32 %13, %13, %29;\n\t"
        "addc.cc.u32 %14, %14, %30;\n\t"
        "addc.u32 %15, %15, 0;"
        : "+r"(A[1]), "+r"(A[2]), "+r"(A[3]), "+r"(A[4]), "+r"(A[5]), "+r"(A[6]), "+r"(A[7]), "+r"(A[8]),
          "+r"(A[9]), "+r"(A[10]), "+r"(A[11]), "+r"(A[12]), "+r"(A[13]), "+r"(A[14]), "+r"(A[15]), "+r"(A[16])
        : "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]), "r"(O[6]), "r"(O[7]), "r"(O[8]),
          "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]));
}

// A[0..16] += a * b for a multiplier of BW 32-bit words (BW = 8: the full product of mul_wide_acc_reg). The partial
// products are laid out as in mul_wide_acc_reg (E: pairs at even limb positions, O: shifted by one limb).
template <int BW>
__device__ __forceinline__ void mul_wide_acc_bw(uint32_t (&A)[17], const uint32_t* a, const uint32_t* b) {
    if (BW == 8) {
        mul_wide_acc_reg(A, a, b);
        return;
    }
    uint32_t E[17], O[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < BW; ++i) {
        if ((i & 1) == 0) {
            chain8_top(E + i, E[i + 8], a[0], a[2], a[4], a[6], b[i]);
            chain8_top(O + i, O[i + 8], a[1], a[3], a[5], a[7], b[i]);
        } else {
            chain8_top(O + i - 1, O[i + 7], a[0], a[2], a[4], a[6], b[i]);
            chain8_top(E + i + 1, E[i + 9], a[1], a[3], a[5], a[7], b[i]);
        }
    }
    uint64_t carry = 0;
#pragma unroll
    for (int k = 0; k < 17; ++k) {
        const uint64_t t = (uint64_t)A[k] + E[k] + (k ? O[k - 1] : 0u) + carry;
        A[k] = (uint32_t)t;
        carry = t >> 32;
    }
}

// 544-bit accumulator (17 words at acc[k * stride]) -> canonical acc * R^-1 mod p. It sits on the latency path of
// every sumcheck round (one lane per value reduces the block's column sums), so it is three Montgomery products on
// the fast IMAD.WIDE rows instead of a word-serial 64-bit loop: with acc = lo + hi R + top R^2 (R = 2^256),
//   acc R^-1 = REDC(lo) + hi + top R  (mod p),   REDC(lo) = montmul(1, lo),  hi mod p = montmul(R mod p, hi),
//   top R mod p = montmul(R^2 mod p, top).
// The wide operand is always the MULTIPLIER (consumed one 32-bit word per row, any value allowed); the multiplicand
// is a constant < p, which is what the row bounds of mont_step assume. Each product is < 2p, the sum < 5p + 1 < 2^256.
template <class PR>
__device__ __forceinline__ Fp<PR> reduce_wide17(const uint32_t* acc, int stride) {
    Fp<PR> lo, hi, top = Fp<PR>::zero(), one_raw = Fp<PR>::zero();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        lo.v[k] = acc[k * stride];
        hi.v[k] = acc[(8 + k) * stride];
    }
    top.v[0] = acc[16 * stride];
    one_raw.v[0] = 1;
    Fp<PR> r = fp_mul_lazy(one_raw, lo);
    const Fp<PR> h = fp_mul_lazy(Fp<PR>::one(), hi);
    const Fp<PR> t = fp_mul_lazy(Fp<PR>::r2(), top);
    add8<PR>(r.v, r.v, h.v);
    add8<PR>(r.v, r.v, t.v);
#pragma unroll
    for (int it = 0; it < 5; ++it) cond_sub_p<PR>(r.v);
    return r;
}

using Fr = Fp<FrParams>;
using Fq = Fp<FqParams>;

// ---- global memory access of one element (32 B, naturally aligned) ---------------------------
// sm_90's widest LDG/STG is 128 bits: an element is two 16 B requests to the same 32 B sector, so a warp
// still covers 1 KiB contiguous -> fully coalesced 32 B sectors. Only the read-only load is inline PTX (for
// its L1::no_allocate hint); the others are plain vector accesses the compiler may schedule freely.
template <class F>
__device__ __forceinline__ F ld_elem(const uint64_t* base, size_t idx) {
    F r;
    const uint32_t* p = reinterpret_cast<const uint32_t*>(base) + idx * 8;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p));
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
        : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]) : "l"(p + 4));
    return r;
}

// Software prefetch of the 128-byte line holding element idx into L2 (no register cost): issued one
// grid-stride iteration ahead so the demand load that follows finds the line on chip.
__device__ __forceinline__ void prefetch_l2(const uint64_t* base, size_t idx) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const uint32_t*>(base) + idx * 8));
}

template <class F>
__device__ __forceinline__ F elem_from(const uint4& a, const uint4& b) {
    F r;
    r.v[0] = a.x, r.v[1] = a.y, r.v[2] = a.z, r.v[3] = a.w;
    r.v[4] = b.x, r.v[5] = b.y, r.v[6] = b.z, r.v[7] = b.w;
    return r;
}

// coherent variant for buffers written earlier in the same kernel / aliased in-place updates
template <class F>
__device__ __forceinline__ F ld_elem_rw(const uint64_t* base, size_t idx) {
    const uint4* p = reinterpret_cast<const uint4*>(base) + idx * 2;
    return elem_from<F>(p[0], p[1]);
}

template <class F>
__device__ __forceinline__ void st_elem(uint64_t* base, size_t idx, const F& x) {
    uint4* p = reinterpret_cast<uint4*>(base) + idx * 2;
    p[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
    p[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}

// Streaming store (evict-first): for tables that are written once and not read again by the same kernel.
template <class F>
__device__ __forceinline__ void st_elem_cs(uint64_t* base, size_t idx, const F& x) {
    uint4* p = reinterpret_cast<uint4*>(base) + idx * 2;
    __stcs(p, make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]));
    __stcs(p + 1, make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]));
}

}  // namespace jb
