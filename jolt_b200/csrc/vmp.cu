// Dory's vector-matrix product of a batched polynomial (jb_lc_vector_matrix_product): v = L^T M for the joint
// polynomial P = sum_i c_i p_i of jb_table_linear_combination laid out as R rows of W columns (flat index x = row W +
// col, the rows of the tier-1 commitments), straight from the terms in their own formats. P is never formed.
//
// One output representation: W bins of 8 u64 lanes of 32-bit limb sums (lane_bins.cuh), zeroed, to which every kernel
// adds canonical field values with integer atomics; bins_to_fr_kernel turns them into the output table. Exact and
// order-free, so the result is bit-exact and deterministic whatever the schedule.
//
// vmp_gather_kernel: the grid is (column tiles) x (row slices) and a thread owns one column of one slice. Per term it
// walks its rows, accumulating UNREDUCED into a 17-word register accumulator, reduces once and adds fp_mul(sum, c~) to
// a running total; at the end it adds the total to its column's bin (8 atomics, none for a zero total). A warp reads 32
// consecutive entries of one row (1 KiB of a field table) and L[row] is a broadcast.
//   * field table:    sum L~ f~ = R^2 sum L f  -> reduced R sum L f,      times c~      = (c sum L f)~
//   * compact column: sum L~ |v| = R sum L v   -> reduced sum L v (plain), times (c R)~ = (c sum L v)~
//                     (a negative value uses p - L~: value_src.cuh's SmallSrc)
//   * one-hot, address-major (x = k T + j): with W <= T the column is j mod W and the row addr_j T/W + j/W, so the
//     thread walks the cycles j = col + m W of its slice and adds L~[row] (field additions, no products); with W > T
//     the column (q T + j) has at most one hot row, addr_j / (W/T) when addr_j = q mod W/T, so one thread per column
//     reads one address (in the first slice only).
// vmp_scatter_kernel: one-hot, cycle-major (x = j K + k). The column depends on the address, so each hot cycle adds
// L~[x / W] into bin x mod W. A thread walks the cycles j = l + h S (S a multiple of W/K, so with W >= K its column
// is (l mod W/K) K + addr_j and runs of one address merge) and keeps a run per column; runs are flushed as c~ times
// their sum with pf_flush (warp-aggregated, safe for skewed columns). With W < K the column is addr_j mod W.
//
// Bounds. The accumulator: a thread adds at most R < 2^32 products < 2^508 per term, below 2^544. The lanes: a
// column's bin takes one addition per gather slice (at most R) and at most R per cycle-major term (a column holds R
// entries of each term), so count R <= 2^32 - 1 additions of values < 2^32 stay below 2^64 - the entry point refuses
// count R >= 2^32. An address >= K that is not the none value raises the call's flag (columns.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "lane_bins.cuh"
#include "lc_terms.cuh"
#include "value_src.cuh"

using Guard = CtxGuard;

namespace {

constexpr int VMP_BLOCK = 256;
constexpr int VMP_GROUP = 32;     // gather descriptors staged in shared memory at a time
constexpr int VMP_SCATTER_LOG_S = 10;  // at least 2^10 cycle lanes per scatter launch row (when T allows)

__device__ __forceinline__ Fr coeff_of(const LcTerm& t) {
    Fr c;
#pragma unroll
    for (int k = 0; k < 8; ++k) c.v[k] = t.c[k];
    return c;
}

// sum over rows [h0, h1) of L~[row] v(row W + col), reduced once
template <class Src>
__device__ __forceinline__ Fr row_sum(const Src& src, const void* p, const uint64_t* left, int log_w, size_t col,
                                      size_t h0, size_t h1) {
    uint32_t A[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) A[k] = 0;
#pragma unroll 2
    for (size_t h = h0; h < h1; ++h) src.acc(A, ld_elem<Fr>(left, h), p, (h << log_w) + col, nullptr);
    return reduce_wide17<FrParams>(A, 1);
}

__device__ __forceinline__ Fr small_row_sum(int kind, const void* p, const uint64_t* left, int log_w, size_t col,
                                         size_t h0, size_t h1) {
    switch (kind) {
        case SK_U8: return row_sum(SmallSrc<SK_U8>{}, p, left, log_w, col, h0, h1);
        case SK_U16: return row_sum(SmallSrc<SK_U16>{}, p, left, log_w, col, h0, h1);
        case SK_U32: return row_sum(SmallSrc<SK_U32>{}, p, left, log_w, col, h0, h1);
        case SK_U64: return row_sum(SmallSrc<SK_U64>{}, p, left, log_w, col, h0, h1);
        case SK_U128: return row_sum(SmallSrc<SK_U128>{}, p, left, log_w, col, h0, h1);
        case SK_I64: return row_sum(SmallSrc<SK_I64>{}, p, left, log_w, col, h0, h1);
        case SK_I128: return row_sum(SmallSrc<SK_I128>{}, p, left, log_w, col, h0, h1);
        case SK_S64: return row_sum(SmallSrc<SK_S64>{}, p, left, log_w, col, h0, h1);
        default: return row_sum(SmallSrc<SK_S128>{}, p, left, log_w, col, h0, h1);
    }
}

// One address-major one-hot term at column col of slice `slice` of `slices`: sum of L~ over its hot entries.
__device__ __forceinline__ Fr one_hot_column(const LcTerm& t, const uint64_t* left, int log_w, size_t col,
                                             unsigned slice, unsigned slices, unsigned int* bad) {
    const uint32_t K = 1u << t.log_k;
    Fr s = Fr::zero();
    if ((uint32_t)log_w <= t.log_t) {
        const size_t per = (size_t)1 << (t.log_t - log_w);  // cycles of one column
        const size_t mps = (per + slices - 1) / slices;
        const size_t m0 = (size_t)slice * mps, m1 = min(per, m0 + mps);
        for (size_t m = m0; m < m1; ++m) {
            const uint32_t a = ld_address(t.ptr, (m << log_w) + col, (int)t.kind);
            if (a == NO_ADDRESS) continue;
            if (a >= K) {
                atomicOr(bad, 1u);
                continue;
            }
            s = fp_add(s, ld_elem<Fr>(left, ((size_t)a << (t.log_t - log_w)) + m));
        }
    } else if (slice == 0) {
        const int log_q = log_w - (int)t.log_t;  // W / T columns per address row
        const size_t j = col & (((size_t)1 << t.log_t) - 1), q = col >> t.log_t;
        const uint32_t a = ld_address(t.ptr, j, (int)t.kind);
        if (a != NO_ADDRESS && a >= K) atomicOr(bad, 1u);
        else if (a != NO_ADDRESS && (a & ((1u << log_q) - 1)) == q) s = ld_elem<Fr>(left, a >> log_q);
    }
    return s;
}

// grid: x = tiles of VMP_BLOCK columns, y = slices of rps rows. terms: the field, compact and address-major one-hot
// terms; every thread walks the same sequence, so the type switch is uniform.
__global__ void __launch_bounds__(VMP_BLOCK, 2)
    vmp_gather_kernel(const LcTerm* terms, size_t count, const uint64_t* left, int log_w, size_t rps,
                      unsigned long long* bins, unsigned int* bad) {
    __shared__ LcTerm s_terms[VMP_GROUP];
    const size_t W = (size_t)1 << log_w;
    const size_t col = (size_t)blockIdx.x * VMP_BLOCK + threadIdx.x;
    const size_t r0 = (size_t)blockIdx.y * rps;
    Fr total = Fr::zero();
    for (size_t g = 0; g < count; g += VMP_GROUP) {
        const int n = count - g < VMP_GROUP ? (int)(count - g) : VMP_GROUP;
        __syncthreads();  // the previous group is consumed
        const uint64_t* src = reinterpret_cast<const uint64_t*>(terms + g);
        uint64_t* dst = reinterpret_cast<uint64_t*>(s_terms);
        for (int i = threadIdx.x; i < n * (int)(sizeof(LcTerm) / 8); i += VMP_BLOCK) dst[i] = src[i];
        __syncthreads();
        if (col >= W) continue;
        for (int i = 0; i < n; ++i) {
            const LcTerm& t = s_terms[i];
            if (col >= t.len) continue;  // a term shorter than W covers part of row 0
            Fr s;
            if (t.type == JB_LC_ONE_HOT) {
                s = one_hot_column(t, left, log_w, col, blockIdx.y, gridDim.y, bad);
            } else {
                const size_t rows = max(t.len >> log_w, (uint64_t)1);
                const size_t h1 = min(rows, r0 + rps);
                if (r0 >= h1) continue;
                s = t.type == JB_LC_TABLE ? row_sum(FieldSrc{}, t.ptr, left, log_w, col, r0, h1)
                                          : small_row_sum((int)t.kind, t.ptr, left, log_w, col, r0, h1);
            }
            total = fp_add(total, fp_mul(s, coeff_of(t)));
        }
    }
    if (col < W && !total.is_zero()) {
#pragma unroll
        for (int w = 0; w < 8; ++w) atomicAdd(bins + col * 8 + w, (unsigned long long)total.v[w]);
    }
}

// One cycle-major one-hot term. grid: x = the S = 2^log_s cycle lanes in tiles of VMP_BLOCK, y = slices of hps steps
// of the T / S steps; cycle j = h S + l.
__global__ void __launch_bounds__(VMP_BLOCK)
    vmp_scatter_kernel(LcTerm t, const uint64_t* left, int log_w, int log_s, size_t hps, unsigned long long* bins,
                       unsigned int* bad) {
    const int lane = threadIdx.x & 31;
    const size_t S = (size_t)1 << log_s;
    const size_t l = (size_t)blockIdx.x * VMP_BLOCK + threadIdx.x;
    const uint32_t K = 1u << t.log_k;
    const size_t W = (size_t)1 << log_w;
    const size_t h0 = (size_t)blockIdx.y * hps, h1 = min((size_t)1 << (t.log_t - log_s), h0 + hps);
    const Fr c = coeff_of(t);
    uint32_t cur = NO_ADDRESS;  // the thread's run: column and the field sum of its L~
    Fr acc = Fr::zero();
    for (size_t h = h0; h < h1; ++h) {  // block-uniform trip count: the warp stays converged for pf_flush
        uint32_t key = NO_ADDRESS;
        Fr w;
        if (l < S) {
            const size_t j = (h << log_s) + l;
            const uint32_t a = ld_address(t.ptr, j, (int)t.kind);
            if (a < K) {
                const size_t x = (j << t.log_k) + a;
                key = (uint32_t)(x & (W - 1));
                w = ld_elem<Fr>(left, x >> log_w);
            } else if (a != NO_ADDRESS) {
                atomicOr(bad, 1u);
            }
        }
        const bool emit = key != NO_ADDRESS && cur != NO_ADDRESS && key != cur;
        Fr v;
        if (emit) v = fp_mul(acc, c);
        pf_flush(emit, cur, v, bins, lane);
        if (key != NO_ADDRESS) {
            acc = key == cur ? fp_add(acc, w) : w;
            cur = key;
        }
    }
    Fr v;
    if (cur != NO_ADDRESS) v = fp_mul(acc, c);
    pf_flush(cur != NO_ADDRESS, cur, v, bins, lane);
}

int launch_check(jb_ctx* c, const char* what) {
    c->launches++;
    return c->check(cudaGetLastError(), what);
}

}  // namespace

extern "C" {

int jb_lc_vector_matrix_product(jb_ctx* c, const jb_lc_term* terms, size_t count, size_t len, size_t row_width,
                                jb_table left, jb_table* out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!terms || !out) return c->fail(JB_ERR_INVALID, "vector_matrix_product: null pointer");
    if (count == 0) return c->fail(JB_ERR_INVALID, "vector_matrix_product: no terms");
    if (!pow2(len)) return c->fail(JB_ERR_INVALID, "vector_matrix_product: the length must be a power of two");
    if (count >= ((size_t)1 << 32)) return c->fail(JB_ERR_UNSUPPORTED, "vector_matrix_product: at most 2^32 - 1 terms");
    if (!pow2(row_width) || row_width > len)
        return c->fail(JB_ERR_INVALID, "vector_matrix_product: the row width must be a power of two <= the length");
    const size_t W = row_width, R = len / row_width;
    if (W >= ((size_t)1 << 32) || R >= ((size_t)1 << 32) || count * R >= ((size_t)1 << 32))
        return c->fail(JB_ERR_UNSUPPORTED, "vector_matrix_product: count x rows must be < 2^32 (lane bound)");
    const int log_w = log2_of(W);
    Guard g(c);
    std::vector<LcTerm> desc;
    int st = check_terms(c, terms, count, len, desc);
    if (st != JB_OK) return st;
    const Table* L = c->find(left);
    if (!L) return c->fail(JB_ERR_INVALID, "vector_matrix_product: unknown left table handle");
    if (L->len != R) return c->fail(JB_ERR_INVALID, "vector_matrix_product: the left table must have len / row_width entries");
    Scratch scratch(c);
    st = load_columns(scratch, terms, count, desc);
    std::vector<LcTerm> gather, scatter;
    size_t rows = 1;  // rows of the longest gather term
    for (const LcTerm& t : desc) {
        if (t.type == JB_LC_ONE_HOT && t.layout == JB_ONE_HOT_CYCLE_MAJOR) {
            scatter.push_back(t);
        } else {
            gather.push_back(t);
            rows = std::max<size_t>(rows, t.len >> log_w);
        }
    }
    LcTerm* d_terms = nullptr;
    unsigned long long* d_bins = nullptr;  // W bins of 8 lanes, then the bad-address flag
    if (st == JB_OK && !gather.empty()) st = scratch.alloc(gather.size() * sizeof(LcTerm), &d_terms);
    if (st == JB_OK) st = scratch.alloc((W * 8 + 1) * 8, &d_bins);
    unsigned int* d_bad = reinterpret_cast<unsigned int*>(d_bins + W * 8);
    if (st == JB_OK) st = c->check(cudaMemsetAsync(d_bins, 0, (W * 8 + 1) * 8, c->stream), "vector_matrix_product bins");
    if (st == JB_OK && !gather.empty()) {
        st = c->check(cudaMemcpyAsync(d_terms, gather.data(), gather.size() * sizeof(LcTerm), cudaMemcpyHostToDevice,
                                      c->stream),
                      "vector_matrix_product terms H2D");
        // about four waves of two blocks per SM over the column tiles, split into row slices
        const size_t gx = (W + VMP_BLOCK - 1) / VMP_BLOCK;
        size_t gy = std::max<size_t>(1, (size_t)c->sm_count * 8 / gx);
        gy = std::min<size_t>(std::min<size_t>(gy, rows), 65535);
        const size_t rps = (rows + gy - 1) / gy;
        gy = (rows + rps - 1) / rps;
        if (st == JB_OK) {
            vmp_gather_kernel<<<dim3((unsigned)gx, (unsigned)gy), VMP_BLOCK, 0, c->stream>>>(
                d_terms, gather.size(), L->buf, log_w, rps, d_bins, d_bad);
            st = launch_check(c, "vmp_gather_kernel launch");
        }
    }
    for (size_t i = 0; i < scatter.size() && st == JB_OK; ++i) {
        const LcTerm& t = scatter[i];
        const int log_s = std::min<int>((int)t.log_t, std::max(log_w - (int)t.log_k, VMP_SCATTER_LOG_S));
        const size_t S = (size_t)1 << log_s, steps = ((size_t)1 << t.log_t) >> log_s;
        const size_t gx = (S + VMP_BLOCK - 1) / VMP_BLOCK;
        size_t gy = std::max<size_t>(1, (size_t)c->sm_count * 8 / gx);
        gy = std::min<size_t>(std::min(gy, steps), 65535);
        const size_t hps = (steps + gy - 1) / gy;
        gy = (steps + hps - 1) / hps;
        vmp_scatter_kernel<<<dim3((unsigned)gx, (unsigned)gy), VMP_BLOCK, 0, c->stream>>>(t, L->buf, log_w, log_s, hps,
                                                                                          d_bins, d_bad);
        st = launch_check(c, "vmp_scatter_kernel launch");
    }
    unsigned int bad = 0;
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, c->stream), "vector_matrix_product flag D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "vector_matrix_product sync");
    if (st == JB_OK && bad) st = fail_bad_address(c);
    Table t;
    if (st == JB_OK) st = c->dev_alloc((void**)&t.buf, W * 32);
    if (st == JB_OK) {
        bins_to_fr_kernel<<<launch_grid(c, W, BINS_BLOCK, 8), BINS_BLOCK, 0, c->stream>>>(d_bins, W, t.buf);
        st = launch_check(c, "bins_to_fr_kernel launch");
    }
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "vector_matrix_product output sync");
    t.cap = t.len = W;
    return c->hand_over(st, t, out);
}

}  // extern "C"
