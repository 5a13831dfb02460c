// Random linear combinations for batched openings (jb_table_linear_combination): the prover's joint polynomial
// P = sum_i c_i p_i over committed polynomials in their own formats - field tables, compact integer columns and
// one-hot address columns - formed in one pass on the device, so P can go straight to jb_hyperkzg_open.
//
// A thread owns one output x and walks every term, accumulating UNREDUCED into a 17-word register accumulator in the
// R^2 domain; one reduce_wide17 (a Montgomery reduction, R^-1) per output gives canonical P~[x] = P[x] R:
//   * field table:   mul_wide_acc_reg(c~, f~)      = c f R^2        (a 256 x 256 product)
//   * compact value: (c R)~ |v|                    = c v R^2        (a 256 x 32w product, w = 1, 2 or 4 words);
//                    a negative value uses p - (c R)~ (the trick SmallSrc in mle_eval.cu uses); both precomputed
//   * one-hot entry: c~ added into words 8..16     = c~ 2^256 = c R^2 when the entry is hot, nothing otherwise
// Bound: every contribution is < p^2 < 2^508 (field), < 2^254 2^128 (compact) or < 2^254 2^256 = 2^510 (one-hot), so
// the sum of fewer than 2^34 terms stays below 2^544 - the entry point refuses count >= 2^32.
//
// The terms are a device array of descriptors, staged through shared memory LC_GROUP at a time; every thread of the
// grid walks the same term sequence, so the type switch is uniform (source_round_kernel relies on the same property).
// A call with count <= LC_GROUP stages its descriptors once per block; a longer one restages each group per tile.
// Either way there is one pass: P is written once and each term is read once. A term shorter than len is the prefix of
// the index range and contributes nothing beyond its length. A one-hot term at x reads addr[j] (cycle-major
// x = j K + k, address-major x = k T + j) and compares it with k; a bad address raises the call's flag, and the entry
// point then discards the output (columns.cuh decides the column formats and their checks). Integer arithmetic only:
// bit-exact and deterministic.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "lc_terms.cuh"

using namespace jb;
using namespace jbi;
using Guard = CtxGuard;

namespace {

constexpr int LC_BLOCK = 256;
constexpr int LC_GROUP = 32;  // descriptors staged in shared memory at a time (32 x 104 B = 3.25 KiB)

__device__ __forceinline__ void add_hi(uint32_t (&A)[17], const uint32_t* c) {
    uint64_t carry = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t t = (uint64_t)A[8 + k] + c[k] + carry;
        A[8 + k] = (uint32_t)t;
        carry = t >> 32;
    }
    A[16] += (uint32_t)carry;
}

// A += c_t p_t(x) for x < len_t
__device__ __forceinline__ void lc_term(uint32_t (&A)[17], const LcTerm& t, size_t x, unsigned int* bad) {
    if (x >= t.len) return;
    uint32_t c[8];
    if (t.type == JB_LC_TABLE) {
#pragma unroll
        for (int k = 0; k < 8; ++k) c[k] = t.c[k];
        const Fr f = ld_elem<Fr>(static_cast<const uint64_t*>(t.ptr), x);
        mul_wide_acc_reg(A, c, f.v);
    } else if (t.type == JB_LC_COMPACT) {
        uint32_t mag[4];
        const bool neg = ld_small(t.ptr, x, (int)t.kind, mag);
#pragma unroll
        for (int k = 0; k < 8; ++k) c[k] = neg ? t.nc[k] : t.c[k];
        const int bits = small_kind_bits((int)t.kind);
        if (bits <= 32) mul_wide_acc_bw<1>(A, c, mag);
        else if (bits <= 64) mul_wide_acc_bw<2>(A, c, mag);
        else mul_wide_acc_bw<4>(A, c, mag);
    } else {
        const size_t j = t.layout == JB_ONE_HOT_CYCLE_MAJOR ? x >> t.log_k : x & (((size_t)1 << t.log_t) - 1);
        const uint32_t k = t.layout == JB_ONE_HOT_CYCLE_MAJOR ? (uint32_t)(x & ((1u << t.log_k) - 1))
                                                              : (uint32_t)(x >> t.log_t);
        const uint32_t a = ld_address(t.ptr, j, (int)t.kind);
        if (a == NO_ADDRESS) return;
        if (a == k) {
#pragma unroll
            for (int w = 0; w < 8; ++w) c[w] = t.c[w];
            add_hi(A, c);
        } else if (a >> t.log_k) {
            atomicOr(bad, 1u);
        }
    }
}

// Tiles of LC_BLOCK outputs, grid-strided; the trip count is uniform over a block (the tile base is), so the block
// can restage descriptors between tiles.
__global__ void __launch_bounds__(LC_BLOCK, 2)
    lincomb_kernel(const LcTerm* terms, size_t count, size_t len, uint64_t* out, unsigned int* bad) {
    __shared__ LcTerm s_terms[LC_GROUP];
    const size_t stride = (size_t)gridDim.x * LC_BLOCK;
    const bool once = count <= LC_GROUP;
    bool staged = false;
    for (size_t base = (size_t)blockIdx.x * LC_BLOCK; base < len; base += stride) {
        const size_t x = base + threadIdx.x;
        uint32_t A[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) A[k] = 0;
        for (size_t g = 0; g < count; g += LC_GROUP) {
            const int n = count - g < LC_GROUP ? (int)(count - g) : LC_GROUP;
            if (!once || !staged) {
                __syncthreads();  // the previous group is consumed
                const uint64_t* src = reinterpret_cast<const uint64_t*>(terms + g);
                uint64_t* dst = reinterpret_cast<uint64_t*>(s_terms);
                for (int i = threadIdx.x; i < n * (int)(sizeof(LcTerm) / 8); i += LC_BLOCK) dst[i] = src[i];
                __syncthreads();
                staged = true;
            }
            if (x < len)
                for (int t = 0; t < n; ++t) lc_term(A, s_terms[t], x, bad);
        }
        if (x < len) st_elem(out, x, reduce_wide17<FrParams>(A, 1));
    }
}

}  // namespace

extern "C" {

int jb_table_linear_combination(jb_ctx* c, const jb_lc_term* terms, size_t count, size_t len, jb_table* out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!terms || !out) return c->fail(JB_ERR_INVALID, "linear_combination: null pointer");
    if (count == 0) return c->fail(JB_ERR_INVALID, "linear_combination: no terms");
    if (!pow2(len)) return c->fail(JB_ERR_INVALID, "linear_combination: the length must be a power of two");
    if (count >= ((size_t)1 << 32)) return c->fail(JB_ERR_UNSUPPORTED, "linear_combination: at most 2^32 - 1 terms");
    Guard g(c);
    std::vector<LcTerm> desc;
    int st = check_terms(c, terms, count, len, desc);
    if (st != JB_OK) return st;
    Scratch scratch(c);
    st = load_columns(scratch, terms, count, desc);
    LcTerm* d_terms = nullptr;
    unsigned int* d_bad = nullptr;
    Table t;
    if (st == JB_OK) st = scratch.alloc(count * sizeof(LcTerm), &d_terms);
    if (st == JB_OK) st = scratch.alloc(sizeof(unsigned int), &d_bad);
    if (st == JB_OK) st = c->dev_alloc((void**)&t.buf, len * 32);
    if (st == JB_OK)
        st = c->check(cudaMemcpyAsync(d_terms, desc.data(), count * sizeof(LcTerm), cudaMemcpyHostToDevice, c->stream),
                      "linear_combination terms H2D");
    if (st == JB_OK) st = c->check(cudaMemsetAsync(d_bad, 0, sizeof(unsigned int), c->stream), "linear_combination flag");
    if (st == JB_OK) {
        lincomb_kernel<<<launch_grid(c, len, LC_BLOCK, 8), LC_BLOCK, 0, c->stream>>>(d_terms, count, len, t.buf, d_bad);
        c->launches++;
        st = c->check(cudaGetLastError(), "lincomb_kernel launch");
    }
    unsigned int bad = 0;
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, c->stream), "linear_combination flag D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "linear_combination sync");
    if (st == JB_OK && bad) st = fail_bad_address(c);
    t.cap = t.len = len;
    return c->hand_over(st, t, out);
}

}  // extern "C"
