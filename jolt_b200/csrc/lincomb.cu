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
// x = j K + k, address-major x = k T + j) and compares it with k; an address >= K that is not the none value raises
// the call's flag, and the entry point then discards the output. Integer arithmetic only: bit-exact and deterministic.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "member.hpp"
#include "small_scalar.cuh"

using namespace jb;
using namespace jbi;
using Guard = CtxGuard;

namespace {

constexpr int LC_BLOCK = 256;
constexpr int LC_GROUP = 32;  // descriptors staged in shared memory at a time (32 x 104 B = 3.25 KiB)

struct LcTerm {
    const void* ptr;  // TABLE: entries; COMPACT: values; ONE_HOT: addresses
    uint64_t len;     // entries of the term: a prefix of the output (ONE_HOT: K T)
    uint32_t c[8];    // TABLE / ONE_HOT: c~; COMPACT: (c R)~
    uint32_t nc[8];   // COMPACT: p - (c R)~, for negative values
    uint32_t type, kind, layout;
    uint32_t log_k, log_t, pad;
};
static_assert(sizeof(LcTerm) % 8 == 0, "LcTerm is staged as u64 words");

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
        const bool u8 = t.kind == SK_U8;
        const uint32_t a = u8 ? (uint32_t)static_cast<const uint8_t*>(t.ptr)[j] : (uint32_t)static_cast<const uint16_t*>(t.ptr)[j];
        if (a == (u8 ? 0xffu : 0xffffu)) return;  // none
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

bool pow2(size_t x) { return x != 0 && (x & (x - 1)) == 0; }
uint32_t log2_of(size_t x) {
    uint32_t l = 0;
    while (x >> (l + 1)) ++l;
    return l;
}

// The checks of one term that need no allocation; fills its descriptor except the column pointer of a host column.
int check_term(jb_ctx* c, const jb_lc_term& in, size_t len, LcTerm& t) {
    std::memset(&t, 0, sizeof t);
    if (!canonical_fr(in.coeff)) return c->fail(JB_ERR_INVALID, "linear_combination: coefficient limbs not canonical");
    t.type = (uint32_t)in.type;
    HostFr cf = HostFr::from_limbs(in.coeff);
    if (in.type == JB_LC_TABLE) {
        Table* tab = c->find(in.table);
        if (!tab) return c->fail(JB_ERR_INVALID, "unknown table handle");
        if (!pow2(tab->len)) return c->fail(JB_ERR_INVALID, "linear_combination: a table's length is not a power of two");
        t.ptr = tab->buf;
        t.len = tab->len;
    } else if (in.type == JB_LC_COMPACT) {
        if (in.kind < SK_U8 || in.kind > SK_LAST) return c->fail(JB_ERR_INVALID, "linear_combination: unknown scalar kind");
        if (in.on_device != 0 && in.on_device != 1) return c->fail(JB_ERR_INVALID, "linear_combination: on_device must be 0 or 1");
        if (!pow2(in.len)) return c->fail(JB_ERR_INVALID, "linear_combination: a compact length is not a power of two");
        if (!in.values) return c->fail(JB_ERR_INVALID, "linear_combination: null column");
        if (in.on_device && ((uintptr_t)in.values % (size_t)std::min(8, small_kind_bytes(in.kind))))
            return c->fail(JB_ERR_INVALID, "linear_combination: misaligned device column");
        t.kind = (uint32_t)in.kind;
        t.len = in.len;
        const HostFr r2{{HostFr::R2[0], HostFr::R2[1], HostFr::R2[2], HostFr::R2[3]}};
        cf = cf * r2;  // (c R)~: times a plain integer |v| it is c v R^2
        uint64_t neg[4];
        std::memcpy(neg, HostFr::P, 32);
        uint64_t borrow = 0;
        for (int k = 0; k < 4; ++k) {  // p - (c R)~ (= p for c = 0: still a multiple of p)
            const unsigned __int128 d = (unsigned __int128)neg[k] - cf.l[k] - borrow;
            neg[k] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
        for (int k = 0; k < 4; ++k) {
            t.nc[2 * k] = (uint32_t)neg[k];
            t.nc[2 * k + 1] = (uint32_t)(neg[k] >> 32);
        }
    } else if (in.type == JB_LC_ONE_HOT) {
        if (in.kind != SK_U8 && in.kind != SK_U16)
            return c->fail(JB_ERR_INVALID, "one-hot: addresses must be JB_SCALAR_U8 or JB_SCALAR_U16");
        if (in.layout != JB_ONE_HOT_CYCLE_MAJOR && in.layout != JB_ONE_HOT_ADDRESS_MAJOR)
            return c->fail(JB_ERR_INVALID, "linear_combination: unknown one-hot layout");
        if (!pow2(in.len) || !pow2(in.K)) return c->fail(JB_ERR_INVALID, "one-hot: K and T must be powers of two");
        if (in.on_device != 0 && in.on_device != 1) return c->fail(JB_ERR_INVALID, "linear_combination: on_device must be 0 or 1");
        if (in.len >= ((size_t)1 << 31)) return c->fail(JB_ERR_UNSUPPORTED, "one-hot: T must be < 2^31");
        if (in.K > ((size_t)1 << 16)) return c->fail(JB_ERR_UNSUPPORTED, "one-hot: K must be <= 2^16");
        if (!in.values) return c->fail(JB_ERR_INVALID, "linear_combination: null column");
        if (in.on_device && ((uintptr_t)in.values % (size_t)small_kind_bytes(in.kind)))
            return c->fail(JB_ERR_INVALID, "one-hot: misaligned device column");
        t.kind = (uint32_t)in.kind;
        t.layout = (uint32_t)in.layout;
        t.log_k = log2_of(in.K);
        t.log_t = log2_of(in.len);
        t.len = in.K * in.len;
    } else {
        return c->fail(JB_ERR_INVALID, "linear_combination: unknown term type");
    }
    if (t.len > len) return c->fail(JB_ERR_INVALID, "linear_combination: a term is longer than the output");
    for (int k = 0; k < 4; ++k) {
        t.c[2 * k] = (uint32_t)cf.l[k];
        t.c[2 * k + 1] = (uint32_t)(cf.l[k] >> 32);
    }
    return JB_OK;
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
    std::vector<LcTerm> desc(count);
    for (size_t i = 0; i < count; ++i) {
        const int st = check_term(c, terms[i], len, desc[i]);
        if (st != JB_OK) return st;
    }
    Columns cols(c);
    int st = JB_OK;
    for (size_t i = 0; i < count && st == JB_OK; ++i) {
        const jb_lc_term& in = terms[i];
        if (in.type == JB_LC_TABLE) continue;
        const size_t bytes = in.len * (size_t)small_kind_bytes(in.kind);
        st = cols.get(in.values, bytes, in.on_device, &desc[i].ptr);
    }
    LcTerm* d_terms = nullptr;
    unsigned int* d_bad = nullptr;
    Table t;
    if (st == JB_OK) st = c->dev_alloc((void**)&d_terms, count * sizeof(LcTerm));
    if (st == JB_OK) st = c->dev_alloc((void**)&d_bad, sizeof(unsigned int));
    if (st == JB_OK) st = c->dev_alloc((void**)&t.buf, len * 32);
    if (st == JB_OK)
        st = c->check(cudaMemcpyAsync(d_terms, desc.data(), count * sizeof(LcTerm), cudaMemcpyHostToDevice, c->stream),
                      "linear_combination terms H2D");
    if (st == JB_OK) st = c->check(cudaMemsetAsync(d_bad, 0, sizeof(unsigned int), c->stream), "linear_combination flag");
    if (st == JB_OK) {
        const size_t tiles = (len + LC_BLOCK - 1) / LC_BLOCK;
        const unsigned grid = (unsigned)std::min<size_t>(tiles, (size_t)c->sm_count * 8);
        lincomb_kernel<<<grid, LC_BLOCK, 0, c->stream>>>(d_terms, count, len, t.buf, d_bad);
        c->launches++;
        st = c->check(cudaGetLastError(), "lincomb_kernel launch");
    }
    unsigned int bad = 0;
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, c->stream), "linear_combination flag D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "linear_combination sync");
    if (st == JB_OK && bad) st = c->fail(JB_ERR_INVALID, "one-hot: an address >= K that is not the none value");
    c->dev_free(d_terms);
    c->dev_free(d_bad);
    if (st != JB_OK) {
        c->dev_free(t.buf);
        return st;
    }
    t.cap = t.len = len;
    *out = c->next_id++;
    c->tables[*out] = t;
    return JB_OK;
}

}  // extern "C"
