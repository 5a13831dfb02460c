// The LT and eq+1 tables (jb_lt_evals, jb_eq_plus_one_evals): the structured factors of the value-evaluation and
// shift relations, built on the device from the point as jb_eq_evals builds the eq table. Both are linear maps of
// E[t] = scale eq(r, t) (r[0] <-> the most significant index bit):
//   LT[j] = sum_{t > j} E[t]                 (the MLE of [j < t] in t at t = r)
//   E1[j] = E[j - 1] for j >= 1, E1[0] = 0   (EqPlusOne(r, j): the successor of t gets eq(r, t))
//
// E1 is the eq table one entry further on: eq_build writes E into entries 1 .. 2^n of a table of 2^n + 1 (the last
// one lies past the table's length) after entry 0 is zeroed. Every output is written once by eq_stream_kernel.
//
// LT splits j = h 2^11 + k 2^8 + t (h: the leading n - 11 variables, k: the next 3, t: the last 8). With the
// unscaled low tables summing to 1,
//   LT[j] = LT_H[h] + E_H[h] LT_3[k] + E_H[h] eq3[k] LT_8[t],
// where E_H / LT_H are the (scaled) eq and LT tables of the leading variables - LT_H by this routine, recursively -
// and LT_3 / LT_8 / eq3 are unscaled tables of the block's variables. lt_stream_kernel forms v = E_H[h] LT_8[t] (one
// full product) and expands v eq3[k] in registers with eq_stream_kernel's doubling step (products by the point, so
// a 125-bit point takes the 4-row product), then adds the block's c[k] = LT_H[h] + E_H[h] LT_3[k]: per output about
// one product and two additions, no scan, 32 B of HBM write. The small tables (n <= 11) come from lt_expand_kernel,
// which doubles E and LT together: E'[2i+1] = E[i] r, E'[2i] = E[i] - E'[2i+1], LT'[2i+1] = LT[i],
// LT'[2i] = LT[i] + E'[2i+1].
#include <cuda_runtime.h>

#include "member.hpp"

using Guard = CtxGuard;

namespace {

using namespace jb;
using namespace jbi;

// LT table of nv <= EQ_BLOCK_VARS variables in one block: the first nv - 3 variables level by level in shared memory
// (E and LT side by side), the last 3 in registers; each thread writes 8 consecutive outputs.
__global__ void __launch_bounds__(256) lt_expand_kernel(const __grid_constant__ EqVars ev, int nv, uint64_t* out) {
    __shared__ uint32_t te[8 * 256], tl[8 * 256];  // word-major, as eq_expand_kernel
    const int tid = threadIdx.x;
    const int reg_vars = nv < 3 ? nv : 3;
    const int smem_vars = nv - reg_vars;
    if (tid == 0) {
        Fr base = Fr::one();
        if (ev.has_scale) {
#pragma unroll
            for (int w = 0; w < 8; ++w) base.v[w] = ev.scale[w];
        }
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            te[w * 256] = base.v[w];
            tl[w * 256] = 0;
        }
    }
    __syncthreads();
    for (int j = 0; j < smem_vars; ++j) {
        const int cur = 1 << j;
        Fr v, l, hi;
        if (tid < cur) {
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                v.v[w] = te[w * 256 + tid];
                l.v[w] = tl[w * 256 + tid];
            }
            hi = fp_mul(v, eq_var(ev, j));
        }
        __syncthreads();
        if (tid < cur) {
            const Fr lo = fp_sub(v, hi), l0 = fp_add(l, hi);
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                te[w * 256 + 2 * tid] = lo.v[w];
                te[w * 256 + 2 * tid + 1] = hi.v[w];
                tl[w * 256 + 2 * tid] = l0.v[w];
                tl[w * 256 + 2 * tid + 1] = l.v[w];
            }
        }
        __syncthreads();
    }
    if (tid >= (1 << smem_vars)) return;
    Fr e[8], l[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        e[0].v[w] = te[w * 256 + tid];
        l[0].v[w] = tl[w * 256 + tid];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if (j < reg_vars) {  // block-uniform
            const Fr rj = eq_var(ev, smem_vars + j);
#pragma unroll
            for (int i = (1 << j) - 1; i >= 0; --i) {
                const Fr hi = fp_mul(e[i], rj);
                e[2 * i] = fp_sub(e[i], hi);
                e[2 * i + 1] = hi;
                l[2 * i + 1] = l[i];
                l[2 * i] = fp_add(l[i], hi);
            }
        }
    }
    const int cnt = 1 << reg_vars;
    const size_t base_idx = (size_t)tid << reg_vars;
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (i < cnt) st_elem(out, base_idx + i, l[i]);
}

// out[(h << 11) | (k << 8) | t] = LT_H[h] + E_H[h] LT_3[k] + E_H[h] eq3[k] LT_8[t]; lt_lo = LT_8 (256) then LT_3 (8),
// ev = the 3 register-stage variables. HI4: all three are 125-bit challenges. CS: evict-first stores.
template <bool HI4, bool CS>
__global__ void __launch_bounds__(256) lt_stream_kernel(const uint64_t* e_hi, const uint64_t* lt_hi,
                                                        const __grid_constant__ EqVars ev, const uint64_t* lt_lo,
                                                        uint64_t* out) {
    __shared__ uint32_t ck[8 * 8];  // word-major c[k]; every thread reads the same word (broadcast)
    const int tid = threadIdx.x;
    const Fr eh = ld_elem_rw<Fr>(e_hi, blockIdx.x);
    if (tid < 8) {
        const Fr c = fp_add(ld_elem_rw<Fr>(lt_hi, blockIdx.x), fp_mul(eh, ld_elem_rw<Fr>(lt_lo, 256 + tid)));
#pragma unroll
        for (int w = 0; w < 8; ++w) ck[w * 8 + tid] = c.v[w];
    }
    Fr e[8];
    e[0] = fp_mul(eh, ld_elem_rw<Fr>(lt_lo, tid));
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const Fr rj = eq_var(ev, j);
#pragma unroll
        for (int i = (1 << j) - 1; i >= 0; --i) {
            Fr hi = HI4 ? fp_mul_hi4(e[i], rj.v + 4) : fp_mul(e[i], rj);
            e[2 * i] = fp_sub(e[i], hi);
            e[2 * i + 1] = hi;
        }
    }
    __syncthreads();
    const size_t base = ((size_t)blockIdx.x << EQ_BLOCK_VARS) + (size_t)tid;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        Fr c;
#pragma unroll
        for (int w = 0; w < 8; ++w) c.v[w] = ck[w * 8 + k];
        const Fr o = fp_add(c, e[k]);
        const size_t idx = base + ((size_t)k << 8);
        if (CS) st_elem_cs(out, idx, o);
        else st_elem(out, idx, o);
    }
}

int lt_build(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, uint64_t* d_out) {
    if (nvars <= (size_t)EQ_BLOCK_VARS) {
        lt_expand_kernel<<<1, 256, 0, c->stream>>>(eq_vars(r, nvars, scale), (int)nvars, d_out);
        c->launches++;
        return c->check(cudaGetLastError(), "lt_expand_kernel launch");
    }
    const size_t hi_vars = nvars - EQ_BLOCK_VARS;
    Scratch scratch(c);
    uint64_t *d_e = nullptr, *d_lt = nullptr, *d_lo = nullptr;
    int st = scratch.alloc(((size_t)1 << hi_vars) * 32, &d_e);
    if (st == JB_OK) st = scratch.alloc(((size_t)1 << hi_vars) * 32, &d_lt);
    if (st == JB_OK) st = scratch.alloc((256 + 8) * 32, &d_lo);
    if (st == JB_OK) st = eq_build(c, r, hi_vars, scale, d_e);
    if (st == JB_OK) st = lt_build(c, r, hi_vars, scale, d_lt);
    const uint64_t* r3 = r + 4 * hi_vars;
    if (st == JB_OK) st = lt_build(c, r3 + 4 * 3, 8, nullptr, d_lo);
    if (st == JB_OK) st = lt_build(c, r3, 3, nullptr, d_lo + 4 * 256);
    if (st == JB_OK) {
        bool hi4 = true;
        for (int j = 0; j < 3; ++j) hi4 = hi4 && r3[4 * j] == 0 && r3[4 * j + 1] == 0;
        const unsigned g = (unsigned)((size_t)1 << hi_vars);
        const bool cs = nvars >= 22;  // as eq_build: tables beyond what L2 can usefully keep
        const EqVars v3 = eq_vars(r3, 3, nullptr);
#define JB_LT_LAUNCH(H, C) lt_stream_kernel<H, C><<<g, 256, 0, c->stream>>>(d_e, d_lt, v3, d_lo, d_out)
        if (hi4 && cs) JB_LT_LAUNCH(true, true);
        else if (hi4) JB_LT_LAUNCH(true, false);
        else if (cs) JB_LT_LAUNCH(false, true);
        else JB_LT_LAUNCH(false, false);
#undef JB_LT_LAUNCH
        c->launches++;
        st = c->check(cudaGetLastError(), "lt_stream_kernel launch");
    }
    return st;
}

// jb_eq_evals' checks, then a new table of 2^nvars entries (storage for `extra` more) filled by `fill`; after an
// error no table exists.
template <typename Fill>
int structured_table(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, jb_table* out, size_t extra,
                     const char* what, Fill fill) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (!out || (nvars && !r) || nvars > 40) return c->fail(JB_ERR_INVALID, what);
    for (size_t i = 0; i < nvars; ++i)
        if (!canonical_fr(r + 4 * i)) return c->fail(JB_ERR_INVALID, "structured table: point limbs not canonical");
    if (scale && !canonical_fr(scale)) return c->fail(JB_ERR_INVALID, "structured table: scale limbs not canonical");
    Guard g(c);
    Table t;
    t.len = (size_t)1 << nvars;
    t.cap = t.len + extra;
    int st = c->dev_alloc((void**)&t.buf, t.cap * 32);
    if (st == JB_OK) st = fill(t.buf);
    return c->hand_over(st, t, out);
}

}  // namespace

extern "C" {

int jb_lt_evals(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, jb_table* out) {
    return structured_table(c, r, nvars, scale, out, 0, "lt_evals: null pointer or nvars > 40",
                            [&](uint64_t* buf) { return lt_build(c, r, nvars, scale, buf); });
}

int jb_eq_plus_one_evals(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, jb_table* out) {
    return structured_table(c, r, nvars, scale, out, 1, "eq_plus_one_evals: null pointer or nvars > 40",
                            [&](uint64_t* buf) {
                                int st = c->check(cudaMemsetAsync(buf, 0, 32, c->stream), "eq_plus_one: zero entry 0");
                                return st == JB_OK ? eq_build(c, r, nvars, scale, buf + 4) : st;
                            });
}

}  // extern "C"
