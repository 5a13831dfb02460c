// Batched-affine bucket accumulation for the Pippenger MSM (msm.cu): the first L halvings of every bucket's point list
// are done with AFFINE additions that share one field inversion per block (Montgomery's trick), 5M + 1S + the inversion's
// share instead of the 8M + 2S of a mixed XYZZ addition - the device form of what the reference's arkworks backend and
// its one-hot path do on the CPU (batch_g1_additions_multi_affine, crates/jolt-crypto/src/ec/bn254/batch_addition.rs:53-150:
// "every level halves each working set by pairwise additions that share a batch inversion").
//
// Layout that makes every level a FLAT kernel (no per-level scan, no search): the bucket offsets are computed on counts
// padded to a multiple of 2^L, and the holes of the sorted index list hold a sentinel (identity). Then at every level
// l < L the pair p is (2p, 2p + 1) -> p over the whole array, pairs never straddle buckets, and bucket b's points after L
// levels are [offsets[b] >> L, offsets[b + 1] >> L). The remaining ceil(cnt / 2^L) points per bucket go through the XYZZ
// accumulation (msm_accumulate_kernel<DIRECT>), which also produces the XYZZ buckets the reduction expects.
//
// COMPLETE additions: unlike the reference's batch addition (whose precondition is "no equal / opposite points in a
// pair"), the pairs here are whatever the scalars make them, so a pair is classified first:
//   either operand the identity (a hole, or an earlier P + (-P))  -> the other operand, no inversion;
//   x1 != x2                                                     -> lambda = (y2 - y1) / (x2 - x1);
//   x1 == x2, y1 == y2                                           -> doubling, lambda = 3 x1^2 / (2 y1)   (y != 0: no 2-torsion);
//   x1 == x2, y1 == -y2                                          -> the identity (0, 0).
// One block = 256 threads x kp pairs (pair p = base + k * 256 + tid: coalesced) and ONE inversion:
//   phase 1  each thread multiplies its pairs' denominators along TWO interleaved chains (even / odd k: two independent
//            dependency chains per thread), parking the running prefixes in global scratch (32 B per pair, streaming);
//   scan     prefix and suffix products of the 256 thread totals (shared memory), one Fermat inversion of the block total;
//   phase 2  walking backwards, each thread peels 1 / d off its chains and finishes the additions.
// The inversion is a serial chain of ~380 products on one thread; kp is chosen so that a block holds several
// times that much work and two resident blocks per SM cover each other's inversion.
#pragma once
#include "ec.cuh"

namespace jb {

constexpr int BAL_BLOCK = 256;
constexpr uint32_t BAL_HOLE = 0x7fffffffu;  // sorted[] entry (sign bit ignored) of a padding hole

struct AffPt {
    Fq x, y;
    __device__ __forceinline__ bool is_inf() const { return x.is_zero() && y.is_zero(); }
};

template <bool GATHER>
__device__ __forceinline__ Fq bal_load_x(const uint64_t* in, const uint32_t* sorted, size_t idx, uint32_t& e) {
    if (GATHER) {
        e = sorted[idx];
        if ((e & BAL_HOLE) == BAL_HOLE) return Fq::zero();
        return ld_elem<Fq>(in, 2 * (size_t)(e & BAL_HOLE));
    }
    e = 0;
    return ld_elem_rw<Fq>(in, 2 * idx);
}
template <bool GATHER>
__device__ __forceinline__ Fq bal_load_y(const uint64_t* in, size_t idx, uint32_t e) {
    if (GATHER) {
        if ((e & BAL_HOLE) == BAL_HOLE) return Fq::zero();
        const Fq y = ld_elem<Fq>(in, 2 * (size_t)(e & BAL_HOLE) + 1);
        return (e >> 31) ? fp_neg(y) : y;
    }
    return ld_elem_rw<Fq>(in, 2 * idx + 1);
}

// 0: copy / identity result (no denominator), 1: chord, 2: tangent
__device__ __forceinline__ int bal_classify(const Fq& x1, const Fq& y1, const Fq& x2, const Fq& y2, Fq& d) {
    const bool inf1 = x1.is_zero() && y1.is_zero(), inf2 = x2.is_zero() && y2.is_zero();
    if (inf1 || inf2) return 0;
    d = fp_sub(x2, x1);
    if (!d.is_zero()) return 1;
    if (fp_sub(y2, y1).is_zero()) {
        d = fp_dbl(y1);
        return 2;
    }
    return 0;  // P + (-P)
}

__device__ __forceinline__ void bal_st_s(uint32_t* base, int tid, const Fq& v) {
#pragma unroll
    for (int w = 0; w < 8; ++w) base[w * BAL_BLOCK + tid] = v.v[w];
}
__device__ __forceinline__ Fq bal_ld_s(const uint32_t* base, int tid) {
    Fq r;
#pragma unroll
    for (int w = 0; w < 8; ++w) r.v[w] = base[w * BAL_BLOCK + tid];
    return r;
}

// in: GATHER ? the base table (affine, 8 limbs per point) read through sorted[] : the previous level's points.
// out[p] = in[2p] + in[2p + 1] for p < (*total_entries >> (lvl + 1)). prefix: 4 limbs of scratch per pair.
template <bool GATHER>
__global__ void __launch_bounds__(BAL_BLOCK, 2)
    msm_affine_level_kernel(const uint64_t* __restrict__ in, const uint32_t* __restrict__ sorted, uint64_t* __restrict__ out,
                            uint64_t* __restrict__ prefix, const unsigned int* __restrict__ total_entries, unsigned lvl,
                            unsigned kp) {
    __shared__ uint32_t s_a[8 * BAL_BLOCK], s_b[8 * BAL_BLOCK];
    __shared__ uint32_t s_inv[8];
    const int tid = threadIdx.x;
    const size_t npairs = (size_t)(*total_entries) >> (lvl + 1);
    const size_t p_base = (size_t)blockIdx.x * BAL_BLOCK * kp;
    if (p_base >= npairs) return;  // uniform over the block
    // ---- phase 1 -------------------------------------------------------------------------------------------
    Fq acc0 = Fq::one(), acc1 = Fq::one();
    for (unsigned k = 0; k < kp; ++k) {
        const size_t p = p_base + (size_t)k * BAL_BLOCK + tid;
        if (p >= npairs) break;
        uint32_t e1, e2;
        const Fq x1 = bal_load_x<GATHER>(in, sorted, 2 * p, e1), x2 = bal_load_x<GATHER>(in, sorted, 2 * p + 1, e2);
        Fq d = fp_sub(x2, x1);
        bool has = !d.is_zero() && !x1.is_zero() && !x2.is_zero();
        if (!has) {  // rare: equal x, or an x of zero (possibly the identity): classify with the y coordinates
            const Fq y1 = bal_load_y<GATHER>(in, 2 * p, e1), y2 = bal_load_y<GATHER>(in, 2 * p + 1, e2);
            has = bal_classify(x1, y1, x2, y2, d) != 0;
        }
        if (has) {
            Fq& acc = (k & 1) ? acc1 : acc0;
            st_elem(prefix, p, acc);
            acc = fp_mul(acc, d);
        }
    }
    // ---- prefix / suffix products of the thread totals, one inversion ---------------------------------------
    const Fq total = fp_mul(acc0, acc1);
    bal_st_s(s_a, tid, total);
    __syncthreads();
    Fq pre = total, suf = total;  // inclusive so far
    for (int off = 1; off < BAL_BLOCK; off <<= 1) {
        Fq l = Fq::one(), r = Fq::one();
        const bool hl = tid >= off, hr = tid + off < BAL_BLOCK;
        if (hl) l = bal_ld_s(s_a, tid - off);
        if (hr) r = bal_ld_s(off == 1 ? s_a : s_b, tid + off);
        __syncthreads();
        if (hl) pre = fp_mul(pre, l);
        if (hr) suf = fp_mul(suf, r);
        bal_st_s(s_a, tid, pre);
        bal_st_s(s_b, tid, suf);
        __syncthreads();
    }
    if (tid == BAL_BLOCK - 1) {
        const Fq inv = fq_inverse(pre);  // never zero: only non-zero denominators were multiplied in
#pragma unroll
        for (int w = 0; w < 8; ++w) s_inv[w] = inv.v[w];
    }
    __syncthreads();
    Fq rinv;
#pragma unroll
    for (int w = 0; w < 8; ++w) rinv.v[w] = s_inv[w];
    if (tid > 0) rinv = fp_mul(rinv, bal_ld_s(s_a, tid - 1));
    if (tid + 1 < BAL_BLOCK) rinv = fp_mul(rinv, bal_ld_s(s_b, tid + 1));
    // rinv = 1 / (acc0 * acc1): split it over the two chains
    Fq rinv0 = fp_mul(rinv, acc1), rinv1 = fp_mul(rinv, acc0);
    // ---- phase 2 -------------------------------------------------------------------------------------------
    for (int k = (int)kp - 1; k >= 0; --k) {
        const size_t p = p_base + (size_t)k * BAL_BLOCK + tid;
        if (p >= npairs) continue;
        uint32_t e1, e2;
        const Fq x1 = bal_load_x<GATHER>(in, sorted, 2 * p, e1), x2 = bal_load_x<GATHER>(in, sorted, 2 * p + 1, e2);
        const Fq y1 = bal_load_y<GATHER>(in, 2 * p, e1), y2 = bal_load_y<GATHER>(in, 2 * p + 1, e2);
        Fq d;
        const int type = bal_classify(x1, y1, x2, y2, d);
        Fq x3, y3;
        if (type == 0) {
            const bool inf1 = x1.is_zero() && y1.is_zero(), inf2 = x2.is_zero() && y2.is_zero();
            if (inf1 && !inf2) { x3 = x2; y3 = y2; }
            else if (inf2 && !inf1) { x3 = x1; y3 = y1; }
            else { x3 = Fq::zero(); y3 = Fq::zero(); }  // both the identity, or P + (-P)
        } else {
            Fq& rv = (k & 1) ? rinv1 : rinv0;
            const Fq inv = fp_mul(rv, ld_elem_rw<Fq>(prefix, p));
            rv = fp_mul(rv, d);
            Fq num;
            if (type == 1) num = fp_sub(y2, y1);
            else {
                const Fq xx = fp_sqr(x1);
                num = fp_add(fp_dbl(xx), xx);
            }
            const Fq lambda = fp_mul(num, inv);
            x3 = fp_sub(fp_sub(fp_sqr(lambda), x1), x2);
            y3 = fp_sub(fp_mul(lambda, fp_sub(x1, x3)), y1);
        }
        st_elem(out, 2 * p, x3);
        st_elem(out, 2 * p + 1, y3);
    }
}

}  // namespace jb
