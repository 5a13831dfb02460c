// Expression pass: one round of a sumcheck member whose summand is a general polynomial in its tables,
//   sum_x [eq(w, x) *] sum_k c_k prod_{i < d_k} f_{table_k[i]}(x)        (T <= 8 tables, <= 16 monomials, d_k <= 6)
// the device half of the reference tier's NaiveSumcheckProver::prove_round (jolt-kernels/src/reference/naive.rs:241-316)
// for an Expr that is a weighted sum of monomials. A table may appear in several monomials and several times in one
// (ra * ra); each table is read, bound and stored ONCE per pair whatever its multiplicity.
#pragma once
#include "poly_kernels.cuh"

namespace jb {

constexpr int EXPR_MAX_TABLES = 8;
constexpr int EXPR_MAX_MONOMIALS = 16;
constexpr int EXPR_MAX_DEGREE = 6;
constexpr int EXPR_MAX_POINTS = EXPR_MAX_DEGREE + 1;  // s(0), s(1), s(2..D-1), s(inf)
constexpr int EXPR_INF = -1;                          // ExprParams::point value of t = infinity
constexpr int EXPR_BLOCK = 128;
enum : uint8_t { EXPR_COEFF_GENERAL = 0, EXPR_COEFF_ONE = 1, EXPR_COEFF_MINUS_ONE = 2 };

// The expression travels as a kernel parameter (nothing in __constant__ state: members of several contexts launch
// concurrently). `point` lists the evaluation points of the round in the kernel-value order assemble_evals consumes:
// 0, [1], 2, .., D-1, inf for D >= 2 and 0, [1] for D == 1 (D = the largest monomial degree); it is filled per round.
struct ExprParams {
    uint32_t coeff[EXPR_MAX_MONOMIALS][8];               // Montgomery words (used when kind == GENERAL)
    uint8_t table[EXPR_MAX_MONOMIALS][EXPR_MAX_DEGREE];  // first degree[k] used
    uint8_t degree[EXPR_MAX_MONOMIALS];
    uint8_t kind[EXPR_MAX_MONOMIALS];                    // EXPR_COEFF_*: +-1 coefficients cost no product
    int8_t point[EXPR_MAX_POINTS];
    int nmono, ntables, D, npoints;
};
static_assert(sizeof(ExprParams) < 1024, "the expression must stay a small kernel parameter");

// Dynamic shared memory of a block: every thread owns a column of T x 16 words - the current value lo + t D and the
// difference D of each table's bound pair - laid out [word][thread] like the fused pass's wide accumulators, so a
// warp's accesses to one word are 32 consecutive banks (the table index is uniform over the grid). Runtime table
// indices therefore address shared memory, never a per-thread array (no local memory). Then the block-sum scratch.
__host__ __device__ constexpr size_t expr_smem_bytes(int ntables) {
    return ((size_t)ntables * 16 * EXPR_BLOCK + (EXPR_BLOCK / 32) * EXPR_MAX_POINTS * 8) * 4;
}

__device__ __forceinline__ Fr expr_ld(const uint32_t* col, int word0) {
    Fr x;
#pragma unroll
    for (int w = 0; w < 8; ++w) x.v[w] = col[(word0 + w) * EXPR_BLOCK];
    return x;
}
__device__ __forceinline__ void expr_st(uint32_t* col, int word0, const Fr& x) {
#pragma unroll
    for (int w = 0; w < 8; ++w) col[(word0 + w) * EXPR_BLOCK] = x.v[w];
}

// Steps 2 and 3 of a pair y whose bound (lo_j, D_j) are in the thread's columns: the monomials at every point of
// the round, times the split-eq weight (WEIGHTED), added to acc. Shared by every pass that stages pairs this way.
template <bool WEIGHTED>
__device__ __forceinline__ void expr_sweep(uint32_t* col, const ExprParams& ex, const TablePtrs& tp, size_t y,
                                           Fr (&acc)[EXPR_MAX_POINTS]) {
    Fr wgt;
    if (WEIGHTED) {  // the split-eq weight of the pair, formed where it is used
        const size_t yo = y >> tp.in_bits;
        wgt = fp_mul(ld_elem<Fr>(tp.e_out, yo), ld_elem<Fr>(tp.e_in, y - (yo << tp.in_bits)));
    }
    int at = 0;  // the point the value words of the columns hold
#pragma unroll
    for (int e = 0; e < EXPR_MAX_POINTS; ++e) {
        if (e >= ex.npoints) break;
        const int t = ex.point[e];
        const bool inf = t == EXPR_INF;
        for (; !inf && at < t; ++at)
            for (int j = 0; j < ex.ntables; ++j) expr_st(col, 16 * j, fp_add(expr_ld(col, 16 * j), expr_ld(col, 16 * j + 8)));
        const int off = inf ? 8 : 0;
        Fr sum = Fr::zero();
        for (int k = 0; k < ex.nmono; ++k) {
            const int d = ex.degree[k];
            if (inf && d < ex.D) continue;
            Fr prod = expr_ld(col, 16 * ex.table[k][0] + off);
            for (int i = 1; i < d; ++i) prod = fp_mul(prod, expr_ld(col, 16 * ex.table[k][i] + off));
            const int kind = ex.kind[k];
            if (kind == EXPR_COEFF_ONE) {
                sum = fp_add(sum, prod);
            } else if (kind == EXPR_COEFF_MINUS_ONE) {
                sum = fp_sub(sum, prod);
            } else {
                Fr c;
#pragma unroll
                for (int w = 0; w < 8; ++w) c.v[w] = ex.coeff[k][w];
                sum = fp_add(sum, fp_mul(prod, c));
            }
        }
        if (WEIGHTED) sum = fp_mul(sum, wgt);
        acc[e] = fp_add(acc[e], sum);
    }
}

// One launch per round, one thread per pair index y (grid-stride). Binding and the table layouts are those of
// fused_pass (HighToLow in place, LowToHigh ping-pong; BIND / HI4 / the 125-bit challenge path). Per pair:
//   1. every table is bound once (BIND) or read, and (lo_j, D_j = hi_j - lo_j) goes to the thread's column;
//   2. for each point t the columns advance lo_j + t D_j in place, and s_y(t) = sum_k c_k prod_i v_{table_k[i]}(t);
//      at t = inf only the monomials of full degree D contribute, through prod_i D_{table_k[i]};
//   3. WEIGHTED (split-eq members): s_y(t) is multiplied by e_out[y >> in_bits] * e_in[y & mask].
// Per-thread sums are reduced field elements (exact, order-free); the block sums them (block_sum) and the last
// block folds the blocks and publishes (round_epilogue), so a round is one launch with no Montgomery reduction
// beyond the products themselves. Always EXPR_MAX_POINTS values are published; the host reads `npoints`.
template <int ORDER, bool BIND, bool HI4, bool WEIGHTED>
__global__ void __launch_bounds__(EXPR_BLOCK, 4) expr_round_kernel(const __grid_constant__ TablePtrs tp, size_t pairs,
                                                                   BindScalar s, const __grid_constant__ ExprParams ex,
                                                                   RoundOut out) {
    extern __shared__ uint32_t dsm[];
    uint32_t* col = dsm + threadIdx.x;
    uint32_t* red = dsm + (size_t)ex.ntables * 16 * EXPR_BLOCK;
    Fr acc[EXPR_MAX_POINTS];
#pragma unroll
    for (int e = 0; e < EXPR_MAX_POINTS; ++e) acc[e] = Fr::zero();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < pairs; y += stride) {
        const size_t yn = y + stride;
        if (yn < pairs) {
            for (int j = 0; j < ex.ntables; ++j) {
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
        for (int j = 0; j < ex.ntables; ++j) {
            const uint64_t* in = tp.in[j];
            Fr lo, hi;
            if (BIND) {
                uint64_t* o = tp.out[j];
                if (ORDER == ORDER_HIGH_TO_LOW) {
                    lo = bind_pair<HI4>(ld_elem_rw<Fr>(in, y), ld_elem_rw<Fr>(in, y + 2 * pairs), s);
                    hi = bind_pair<HI4>(ld_elem_rw<Fr>(in, y + pairs), ld_elem_rw<Fr>(in, y + 3 * pairs), s);
                    st_elem(o, y, lo);
                    st_elem(o, y + pairs, hi);
                } else {
                    lo = bind_pair<HI4>(ld_elem<Fr>(in, 4 * y), ld_elem<Fr>(in, 4 * y + 1), s);
                    hi = bind_pair<HI4>(ld_elem<Fr>(in, 4 * y + 2), ld_elem<Fr>(in, 4 * y + 3), s);
                    st_elem(o, 2 * y, lo);
                    st_elem(o, 2 * y + 1, hi);
                }
            } else if (ORDER == ORDER_HIGH_TO_LOW) {
                lo = ld_elem_rw<Fr>(in, y);
                hi = ld_elem_rw<Fr>(in, y + pairs);
            } else {
                lo = ld_elem<Fr>(in, 2 * y);
                hi = ld_elem<Fr>(in, 2 * y + 1);
            }
            expr_st(col, 16 * j, lo);
            expr_st(col, 16 * j + 8, fp_sub(hi, lo));
        }
        expr_sweep<WEIGHTED>(col, ex, tp, y, acc);
    }
    block_sum<EXPR_MAX_POINTS>(acc, red);
    round_epilogue<EXPR_MAX_POINTS>(acc, red, out);
}

}  // namespace jb
