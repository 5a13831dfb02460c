// Batch affine addition of G1 points: sums of index-selected bases, one sum per index set - the device form of
// batch_g1_additions_multi_affine (crates/jolt-crypto/src/ec/bn254/batch_addition.rs:53-150), which Dory's tier-1
// commitments use for one-hot / binary witness columns (crates/jolt-dory/src/streaming.rs:68,128,152,201): every
// level halves each working set by pairwise AFFINE additions (lambda = (y2 - y1) / (x2 - x1): 1M + 1S + 1M once the
// inverse is known) and all the pairs of a level share batch inversions (Montgomery's trick).
// Here: one launch per level; a block handles 2048 consecutive pairs (8 per thread) and ONE Fq inversion:
//   phase 1  every thread multiplies its pairs' denominators, keeping the running prefixes in shared memory;
//   scan     prefix and suffix products of the 256 per-thread totals (Hillis-Steele in shared memory), thread 0
//            inverts the block total (Fermat), so 1 / (own total) = inv_all * prefix * suffix;
//   phase 2  walking its pairs backwards, every thread peels off 1 / (x2 - x1) and finishes the addition.
// ~8.3 Fq products per addition (6 + the scan's 18 per thread over 8 pairs) against 10 for a mixed XYZZ addition,
// and the result is affine: it feeds the next level (or the caller) without a normalisation.
// Precondition (as in the reference): the two points of a pair have distinct x. Like ark_ff's batch_inversion the
// zero denominators are skipped (their "inverse" is 0), so a violating pair yields the same unchecked garbage the
// reference yields for that pair only.
#include "../../include/jolt_b200.h"

#include <cuda_runtime.h>

#include <vector>

#include "ctx.hpp"
#include "ec.cuh"

using namespace jb;
using Guard = CtxGuard;

namespace {

constexpr int BA_KP = 8;       // pairs per thread
constexpr int BA_BLOCK = 256;

__device__ __forceinline__ void st_s(uint32_t* base, int slot, int tid, const Fq& v) {
#pragma unroll
    for (int w = 0; w < 8; ++w) base[(slot * 8 + w) * BA_BLOCK + tid] = v.v[w];
}
__device__ __forceinline__ Fq ld_s(const uint32_t* base, int slot, int tid) {
    Fq r;
#pragma unroll
    for (int w = 0; w < 8; ++w) r.v[w] = base[(slot * 8 + w) * BA_BLOCK + tid];
    return r;
}

// in: the level's input points (affine, 8 limbs) - or, at level 0, `bases` gathered through `gather`.
// set s owns in[in_off[s] .. in_off[s + 1]) and produces out[out_off[s] ..): one point per pair, then the odd one.
__global__ void __launch_bounds__(BA_BLOCK) batch_add_level_kernel(const uint64_t* in, const uint32_t* gather, uint64_t* out,
                                                                   const uint64_t* in_off, const uint64_t* out_off,
                                                                   const uint64_t* pair_off, size_t nsets, size_t total_pairs) {
    extern __shared__ uint32_t sm[];
    uint32_t* s_pre = sm;                              // [KP][8][256] local prefixes
    uint32_t* s_a = sm + BA_KP * 8 * BA_BLOCK;         // [8][256] scan buffer A
    uint32_t* s_b = s_a + 8 * BA_BLOCK;                // scan buffer B
    __shared__ uint32_t s_inv[8];
    const int tid = threadIdx.x;
    const size_t p0 = ((size_t)blockIdx.x * BA_BLOCK + tid) * BA_KP;
    uint32_t src[BA_KP], dst[BA_KP];
    bool ok[BA_KP];
    auto point_x = [&](uint32_t i) { return ld_elem_rw<Fq>(in, 2 * (size_t)(gather ? gather[i] : i)); };
    auto point_y = [&](uint32_t i) { return ld_elem_rw<Fq>(in, 2 * (size_t)(gather ? gather[i] : i) + 1); };
    Fq acc = Fq::one();
    // locate the first pair's set by binary search, then walk forward
    size_t s = 0;
    if (p0 < total_pairs) {
        size_t lo = 0, hi = nsets;  // pair_off[lo] <= p0 < pair_off[hi]
        while (hi - lo > 1) {
            const size_t mid = (lo + hi) / 2;
            if (pair_off[mid] <= p0) lo = mid;
            else hi = mid;
        }
        s = lo;
    }
#pragma unroll
    for (int k = 0; k < BA_KP; ++k) {
        const size_t p = p0 + k;
        ok[k] = false;
        src[k] = dst[k] = 0;
        st_s(s_pre, k, tid, acc);
        if (p < total_pairs) {
            while (pair_off[s + 1] <= p) ++s;
            const size_t j = p - pair_off[s];
            src[k] = (uint32_t)(in_off[s] + 2 * j);
            dst[k] = (uint32_t)(out_off[s] + j);
            const Fq d = fp_sub(point_x(src[k] + 1), point_x(src[k]));
            ok[k] = !d.is_zero();
            if (ok[k]) acc = fp_mul(acc, d);
        }
    }
    // ---- prefix (exclusive) and suffix (exclusive) products of the per-thread totals ------------------------
    st_s(s_a, 0, tid, acc);
    __syncthreads();
    Fq pre = acc, suf = acc;  // inclusive so far
    for (int off = 1; off < BA_BLOCK; off <<= 1) {
        Fq l = Fq::one(), r = Fq::one();
        const bool hl = tid >= off, hr = tid + off < BA_BLOCK;
        if (hl) l = ld_s(s_a, 0, tid - off);
        if (hr) r = ld_s(s_b, 0, tid + off);
        if (off == 1 && hr) r = ld_s(s_a, 0, tid + off);
        __syncthreads();
        if (hl) pre = fp_mul(pre, l);
        if (hr) suf = fp_mul(suf, r);
        st_s(s_a, 0, tid, pre);
        st_s(s_b, 0, tid, suf);
        __syncthreads();
    }
    // pre = prod_{t <= tid} T_t, suf = prod_{t >= tid} T_t
    if (tid == BA_BLOCK - 1) {
        const Fq inv = fq_inverse(pre);  // the block total is never zero (zero denominators were skipped)
#pragma unroll
        for (int w = 0; w < 8; ++w) s_inv[w] = inv.v[w];
    }
    __syncthreads();
    Fq rinv;
#pragma unroll
    for (int w = 0; w < 8; ++w) rinv.v[w] = s_inv[w];
    // 1 / T_tid = inv_all * prod_{t < tid} T_t * prod_{t > tid} T_t
    if (tid > 0) rinv = fp_mul(rinv, ld_s(s_a, 0, tid - 1));
    if (tid + 1 < BA_BLOCK) rinv = fp_mul(rinv, ld_s(s_b, 0, tid + 1));
    // ---- phase 2: peel the inverses off backwards and add --------------------------------------------------
#pragma unroll
    for (int k = BA_KP - 1; k >= 0; --k) {
        if (p0 + k >= total_pairs) continue;
        const Fq x1 = point_x(src[k]), x2 = point_x(src[k] + 1);
        Fq inv = Fq::zero();
        if (ok[k]) {
            inv = fp_mul(rinv, ld_s(s_pre, k, tid));
            rinv = fp_mul(rinv, fp_sub(x2, x1));
        }
        const Fq y1 = point_y(src[k]), y2 = point_y(src[k] + 1);
        const Fq lambda = fp_mul(fp_sub(y2, y1), inv);
        const Fq x3 = fp_sub(fp_sub(fp_sqr(lambda), x1), x2);
        const Fq y3 = fp_sub(fp_mul(lambda, fp_sub(x1, x3)), y1);
        st_elem(out, 2 * (size_t)dst[k], x3);
        st_elem(out, 2 * (size_t)dst[k] + 1, y3);
    }
}

// the odd element of a working set moves up unchanged (batch_addition.rs:136-140); also level 0's singletons
__global__ void batch_add_carry_kernel(const uint64_t* in, const uint32_t* gather, uint64_t* out, const uint64_t* in_off,
                                       const uint64_t* out_off, size_t nsets) {
    const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nsets) return;
    const uint64_t cnt = in_off[s + 1] - in_off[s];
    if ((cnt & 1) == 0) return;
    const uint64_t i = in_off[s] + cnt - 1;
    const size_t srcp = gather ? gather[i] : i;
    const uint64_t o = out_off[s] + cnt / 2;
    st_elem(out, 2 * o, ld_elem_rw<Fq>(in, 2 * srcp));
    st_elem(out, 2 * o + 1, ld_elem_rw<Fq>(in, 2 * srcp + 1));
}

}  // namespace

extern "C" int jb_g1_batch_add(jb_ctx* c, jb_srs bases, const uint64_t* set_offsets, const uint32_t* indices, size_t nsets,
                               uint64_t* out_xy) {
    if (!c || (nsets && (!set_offsets || !out_xy))) return JB_ERR_INVALID;
    if (nsets == 0) return JB_OK;
    Guard g(c);
    Srs* found = nullptr;
    if (const int st = c->find_srs(bases, &found)) return st;
    const Srs& srs = *found;
    const size_t total = set_offsets[nsets];
    if (total >= ((size_t)1 << 31)) return c->fail(JB_ERR_UNSUPPORTED, "batch_add: fewer than 2^31 indices per call");
    if (total && !indices) return JB_ERR_INVALID;
    for (size_t s = 0; s < nsets; ++s)
        if (set_offsets[s + 1] < set_offsets[s]) return c->fail(JB_ERR_INVALID, "batch_add: set offsets must be non-decreasing");
    for (size_t i = 0; i < total; ++i)
        if (indices[i] >= srs.n) return c->fail(JB_ERR_INVALID, "batch_add: index out of bounds");
    // working-set sizes per level (host: O(nsets) per level)
    std::vector<uint64_t> cnt(nsets);
    size_t max_cnt = 0;
    for (size_t s = 0; s < nsets; ++s) {
        cnt[s] = set_offsets[s + 1] - set_offsets[s];
        max_cnt = cnt[s] > max_cnt ? cnt[s] : max_cnt;
    }
    Scratch scratch(c);
    uint32_t* d_idx = nullptr;
    uint64_t *d_w[2] = {nullptr, nullptr}, *d_off = nullptr;
    int st = JB_OK;
    const size_t w_elems = total / 2 + nsets + 1;  // level-1 size bound: sum ceil(cnt / 2)
    if (total) st = scratch.alloc(total * 4, &d_idx);
    if (st == JB_OK) st = scratch.alloc(w_elems * 64, &d_w[0]);
    if (st == JB_OK) st = scratch.alloc(w_elems * 64, &d_w[1]);
    if (st == JB_OK) st = scratch.alloc(3 * (nsets + 1) * 8, &d_off);
    if (st == JB_OK && total)
        st = c->check(cudaMemcpyAsync(d_idx, indices, total * 4, cudaMemcpyHostToDevice, c->stream), "batch_add indices H2D");
    std::vector<uint64_t> offs(3 * (nsets + 1));
    const uint64_t* cur = srs.xy;  // level 0 reads the bases through the indices
    const uint32_t* gather = d_idx;
    int flip = 0;
    std::vector<uint64_t> in_off(set_offsets, set_offsets + nsets + 1);
    constexpr size_t smem = (size_t)(BA_KP * 8 + 16) * BA_BLOCK * 4;
    static bool attr = [] {
        cudaFuncSetAttribute(batch_add_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        return true;
    }();
    (void)attr;
    while (st == JB_OK && max_cnt > 1) {
        uint64_t* in_o = offs.data();
        uint64_t* out_o = in_o + (nsets + 1);
        uint64_t* pair_o = out_o + (nsets + 1);
        uint64_t acc_out = 0, acc_pair = 0;
        for (size_t s = 0; s < nsets; ++s) {
            in_o[s] = in_off[s];
            out_o[s] = acc_out;
            pair_o[s] = acc_pair;
            acc_out += (cnt[s] + 1) / 2;
            acc_pair += cnt[s] / 2;
        }
        in_o[nsets] = in_off[nsets];
        out_o[nsets] = acc_out;
        pair_o[nsets] = acc_pair;
        st = c->check(cudaMemcpyAsync(d_off, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, c->stream), "batch_add offsets H2D");
        if (st != JB_OK) break;
        st = c->check(cudaStreamSynchronize(c->stream), "batch_add offsets sync");  // (offs is reused by the next level)
        if (st != JB_OK) break;
        uint64_t* outp = d_w[flip];
        const size_t per_block = (size_t)BA_BLOCK * BA_KP;
        if (acc_pair) {
            batch_add_level_kernel<<<(unsigned)((acc_pair + per_block - 1) / per_block), BA_BLOCK, smem, c->stream>>>(
                cur, gather, outp, d_off, d_off + (nsets + 1), d_off + 2 * (nsets + 1), nsets, acc_pair);
            c->launches++;
        }
        batch_add_carry_kernel<<<(unsigned)((nsets + 255) / 256), 256, 0, c->stream>>>(cur, gather, outp, d_off, d_off + (nsets + 1), nsets);
        c->launches++;
        st = c->check(cudaGetLastError(), "batch_add level launch");
        // next level
        max_cnt = 0;
        for (size_t s = 0; s < nsets; ++s) {
            in_off[s] = out_o[s];
            cnt[s] = (cnt[s] + 1) / 2;
            max_cnt = cnt[s] > max_cnt ? cnt[s] : max_cnt;
        }
        in_off[nsets] = acc_out;
        cur = outp;
        gather = nullptr;
        flip ^= 1;
    }
    // results: every set holds at most one point now (empty sets: identity = zeros)
    if (st == JB_OK) {
        std::vector<uint64_t> host;
        const bool from_bases = gather != nullptr;  // no level ran: singletons / empties straight from the bases
        std::vector<uint32_t> hidx;
        if (!from_bases && in_off[nsets]) {
            host.resize(in_off[nsets] * 8);
            st = c->check(cudaMemcpyAsync(host.data(), cur, host.size() * 8, cudaMemcpyDeviceToHost, c->stream), "batch_add D2H");
            if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "batch_add sync");
        }
        for (size_t s = 0; s < nsets && st == JB_OK; ++s) {
            uint64_t* o = out_xy + 8 * s;
            if (cnt[s] == 0) {
                for (int w = 0; w < 8; ++w) o[w] = 0;
            } else if (from_bases) {
                st = c->check(cudaMemcpyAsync(o, srs.xy + 8 * (size_t)indices[in_off[s]], 64, cudaMemcpyDeviceToHost, c->stream),
                              "batch_add D2H");
            } else {
                for (int w = 0; w < 8; ++w) o[w] = host[in_off[s] * 8 + w];
            }
        }
        if (st == JB_OK && from_bases) st = c->check(cudaStreamSynchronize(c->stream), "batch_add sync");
    }
    return st;
}
