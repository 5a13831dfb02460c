// Compact (small-scalar) tables on the device.
//   * jb_table_upload_small : Polynomial<T> -> Polynomial<Fr>, the promotion F::from(T) of
//     crates/jolt-poly/src/dense.rs:129-142 / crates/jolt-field/src/bn254/mod.rs:265-298 (from_u64,
//     from_i64, from_u128, from_i128; mont.rs:309-325) done by a kernel, so only 1-16 bytes per
//     entry cross PCIe instead of 32.
//   * jb_table_bind_small   : Polynomial<T>::bind_to_field (dense.rs:129-142) fused: the compact table
//     is folded under the first challenge straight into a field table of half the length;
//     out[i] = F(lo) + s * (F(hi) - F(lo)), with the difference taken on the integers.
// Integer arithmetic only; results are canonical Montgomery values, bit-identical to promoting on the
// host and binding.
#include <cuda_runtime.h>

#include "columns.cuh"
#include "host_fr.hpp"
#include "poly_kernels.cuh"

using namespace jb;

namespace {

using Guard = CtxGuard;

__global__ void __launch_bounds__(256) promote_small_kernel(const void* values, size_t n, int kind, uint64_t* out) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t mag[4];
        const bool neg = ld_small(values, i, kind, mag);
        st_elem(out, i, promote_small(mag, neg));
    }
}

// sR = s * R (Montgomery form of the Montgomery limbs of s): montmul(sR, d) = s_mont * d for a plain integer d.
template <int ORDER>
__global__ void __launch_bounds__(256) bind_small_kernel(const void* values, size_t half, int kind, BindScalar sR,
                                                         uint64_t* out) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    Fr sv;
#pragma unroll
    for (int j = 0; j < 8; ++j) sv.v[j] = sR.w[j];
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += stride) {
        const size_t il = ORDER == ORDER_HIGH_TO_LOW ? i : 2 * i;
        const size_t ih = ORDER == ORDER_HIGH_TO_LOW ? i + half : 2 * i + 1;
        uint32_t ml[4], mh[4];
        const bool nl = ld_small(values, il, kind, ml);
        const bool nh = ld_small(values, ih, kind, mh);
        // d = hi - lo as sign + magnitude (|d| < 2^129)
        Fr A = Fr::zero(), B = Fr::zero(), D;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            A.v[j] = mh[j];
            B.v[j] = ml[j];
        }
        bool nd;
        if (nl != nh) {  // opposite signs: |d| = |hi| + |lo|, sign of hi
            add8<FrParams>(D.v, A.v, B.v);
            nd = nh;
        } else {
            const uint32_t borrow = sub8(D.v, A.v, B.v);
            nd = nh;
            if (borrow) {  // |lo| > |hi|
                sub8(D.v, B.v, A.v);
                nd = !nh;
            }
        }
        Fr t = fp_mul(D, sv);  // s * |d| (Montgomery form)
        if (nd) t = fp_neg(t);
        st_elem(out, i, fp_add(promote_small(ml, nl), t));
    }
}

}  // namespace

extern "C" {

int jb_table_upload_small(jb_ctx* c, const void* values, size_t len, int kind, jb_table* out) {
    if (!c || !values || !out || len == 0) return JB_ERR_INVALID;
    if (!compact_kind(kind)) return c->fail(JB_ERR_INVALID, "upload_small: unknown scalar kind");
    Guard g(c);
    Scratch scratch(c);
    Table t;
    t.cap = t.len = len;
    int st = c->dev_alloc((void**)&t.buf, len * 32);
    const void* d_vals = nullptr;
    if (st == JB_OK) st = get_column(scratch, values, len * (size_t)small_kind_bytes(kind), 0, &d_vals);
    // (the caller's buffer is only borrowed for the call: a pinned source makes the copy truly asynchronous)
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "upload_small sync");
    if (st == JB_OK) {
        promote_small_kernel<<<launch_grid(c, len, 256, 4), 256, 0, c->stream>>>(d_vals, len, kind, t.buf);
        c->launches++;
        st = c->check(cudaGetLastError(), "promote_small_kernel launch");
    }
    return c->hand_over(st, t, out);
}

int jb_table_bind_small(jb_ctx* c, const void* values, size_t len, int kind, const uint64_t r[4], int order, jb_table* out) {
    if (!c || !values || !out || !r) return JB_ERR_INVALID;
    if (!compact_kind(kind)) return c->fail(JB_ERR_INVALID, "bind_small: unknown scalar kind");
    if (len < 2 || (len & (len - 1))) return c->fail(JB_ERR_INVALID, "bind_small: table length must be a power of two >= 2");
    if (HostFr::geq_p(r)) return c->fail(JB_ERR_INVALID, "bind_small: challenge limbs not canonical (>= r)");
    if (order != JB_HIGH_TO_LOW && order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "bind_small: unknown binding order");
    const size_t half = len / 2;
    Guard g(c);
    Scratch scratch(c);
    Table t;
    t.cap = t.len = half;
    int st = c->dev_alloc((void**)&t.buf, half * 32);
    const HostFr r2{{HostFr::R2[0], HostFr::R2[1], HostFr::R2[2], HostFr::R2[3]}};
    const HostFr sr = HostFr::from_limbs(r) * r2;
    BindScalar s;
    for (int i = 0; i < 4; ++i) {
        s.w[2 * i] = (uint32_t)sr.l[i];
        s.w[2 * i + 1] = (uint32_t)(sr.l[i] >> 32);
    }
    const void* d_vals = nullptr;
    if (st == JB_OK) st = get_column(scratch, values, len * (size_t)small_kind_bytes(kind), 0, &d_vals);
    // (the caller's buffer is only borrowed for the call: a pinned source makes the copy truly asynchronous)
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "bind_small sync");
    if (st == JB_OK) {
        if (order == JB_HIGH_TO_LOW)
            bind_small_kernel<ORDER_HIGH_TO_LOW><<<launch_grid(c, half, 256, 4), 256, 0, c->stream>>>(d_vals, half, kind, s, t.buf);
        else
            bind_small_kernel<ORDER_LOW_TO_HIGH><<<launch_grid(c, half, 256, 4), 256, 0, c->stream>>>(d_vals, half, kind, s, t.buf);
        c->launches++;
        st = c->check(cudaGetLastError(), "bind_small_kernel launch");
    }
    return c->hand_over(st, t, out);
}

}  // extern "C"
