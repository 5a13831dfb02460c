// HyperKZG prover side on the device - SURVEY.md section 8(f) rank 1.
//   commit : kzg_commit = one MSM over g1_powers[..len]          crates/jolt-hyperkzg/src/kzg.rs:15-27
//   open   : HyperKZGScheme::open                                 crates/jolt-hyperkzg/src/scheme.rs:122-158
//            fold_polynomials (LowToHigh binds, point[1..] back to front)            scheme.rs:88-114
//            kzg_open_batch: v[t][j] = f_j(u_t) (Horner), B = sum_j q^j f_j,
//            h_t = B / (X - u_t) (compute_witness_polynomial), w_t = commit(h_t)      kzg.rs:34-126
// The folded polynomials stay resident between the fold, the intermediate commitments, the
// evaluations and the batching (the reference re-walks host vectors for each step). The transcript
// stays with the caller: two callbacks deliver r (after the intermediate commitments) and q (after the
// evaluations); group elements cross as Jacobian representatives.
//
// Univariate work is organised as a chunked Horner scan. With S(k) = sum_{i>=k} c_i u^(i-k):
//   f(u) = S(0),   (f / (X - u))[k-1] = S(k)          (kzg.rs:34-46 is exactly s = c_k + u s)
// Each thread owns a contiguous chunk of L coefficients and computes its local value
// T = sum_i c_(lo+i) u^i; an affine Hillis-Steele scan (R_t += (u^L)^(2^s) R_(t+2^s)) over the 256
// threads of a block, and the same scan over <= 1024 block totals, turn the T's into every chunk's
// seed S(hi); a second pass re-walks each chunk from its seed and writes the quotient. Three
// evaluation points (r, -r, r^2) ride along in every pass.
#include <cuda_runtime.h>

#include <cstring>
#include <vector>

#include "ctx.hpp"
#include "host_fr.hpp"
#include "poly_kernels.cuh"

using namespace jb;

extern "C" int jb_msm_g1_device(jb_ctx* c, jb_srs h, size_t offset, const uint64_t* d_scalars, size_t n, uint64_t out_xyz[12]);

namespace {

constexpr int HZ_POINTS = 3;
constexpr int HZ_THREADS = 256;

// powers of one evaluation point, in kernel-parameter space
struct HornerPoint {
    uint32_t u[8];          // the point
    uint32_t a_thread[8][8];   // (u^L)^(2^s), s < 8  : in-block scan multipliers
    uint32_t a_block[10][8];   // (u^(256 L))^(2^s), s < 10 : inter-block scan multipliers
    uint32_t u_l[8];        // u^L
    uint32_t u_bl[8];       // u^(256 L)
};
struct HornerParams {
    HornerPoint p[HZ_POINTS];
};

__device__ __forceinline__ Fr fr_from(const uint32_t* w) {
    Fr x;
#pragma unroll
    for (int i = 0; i < 8; ++i) x.v[i] = w[i];
    return x;
}

// In-block affine suffix scan: on entry x[p] = T_t (thread t, point p); on exit x[p] = R_t =
// sum_{t' >= t} T_t' A^(t'-t), A = u^L (thread level) or u^(256 L) (block level). Points are
// scanned one after the other so the exchange buffer stays at 8 * 1024 words (32 KiB).
__device__ __forceinline__ void block_suffix_scan(Fr (&x)[HZ_POINTS], const HornerParams& hp, uint32_t* smem, bool block_level) {
    const int tid = threadIdx.x;
    const int steps = block_level ? 10 : 8;
    const int n = blockDim.x;
#pragma unroll 1
    for (int p = 0; p < HZ_POINTS; ++p) {
        Fr v = x[p];
        for (int s = 0; s < steps && (1 << s) < n; ++s) {
#pragma unroll
            for (int w = 0; w < 8; ++w) smem[w * 1024 + tid] = v.v[w];
            __syncthreads();
            const int src = tid + (1 << s);
            if (src < n) {
                Fr o;
#pragma unroll
                for (int w = 0; w < 8; ++w) o.v[w] = smem[w * 1024 + src];
                Fr a = fr_from(block_level ? hp.p[p].a_block[s] : hp.p[p].a_thread[s]);
                v = fp_add(v, fp_mul(a, o));
            }
            __syncthreads();
        }
        x[p] = v;
    }
}

// value of the next thread's x (or `last` for the block's last thread), one point at a time
__device__ __forceinline__ Fr shift_down(const Fr& x, const Fr& last, uint32_t* smem) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int w = 0; w < 8; ++w) smem[w * 1024 + tid] = x.v[w];
    __syncthreads();
    Fr o = last;
    if (tid + 1 < (int)blockDim.x) {
#pragma unroll
        for (int w = 0; w < 8; ++w) o.v[w] = smem[w * 1024 + tid + 1];
    }
    __syncthreads();
    return o;
}

// Pass A: per-thread chunk values T (optionally stored) and per-block totals R_0.
// coeffs: len elements; chunk L (power of two); block b covers [b*256*L, (b+1)*256*L).
template <bool STORE_THREAD>
__global__ void __launch_bounds__(HZ_THREADS) horner_totals_kernel(const uint64_t* coeffs, size_t len, int L,
                                                                   const __grid_constant__ HornerParams hp,
                                                                   uint64_t* thread_totals, uint64_t* block_totals) {
    __shared__ uint32_t smem[8 * 1024];
    const size_t gt = (size_t)blockIdx.x * HZ_THREADS + threadIdx.x;
    const size_t lo = gt * L;
    Fr acc[HZ_POINTS];
#pragma unroll
    for (int p = 0; p < HZ_POINTS; ++p) acc[p] = Fr::zero();
    if (lo < len) {
        const size_t hi = lo + L < len ? lo + L : len;
        Fr u[HZ_POINTS];
#pragma unroll
        for (int p = 0; p < HZ_POINTS; ++p) u[p] = fr_from(hp.p[p].u);
        for (size_t k = hi; k-- > lo;) {  // Horner from the top of the chunk
            Fr c = ld_elem<Fr>(coeffs, k);
#pragma unroll
            for (int p = 0; p < HZ_POINTS; ++p) acc[p] = fp_add(fp_mul(acc[p], u[p]), c);
        }
    }
    if (STORE_THREAD) {
#pragma unroll
        for (int p = 0; p < HZ_POINTS; ++p) st_elem(thread_totals, gt * HZ_POINTS + p, acc[p]);
    }
    block_suffix_scan(acc, hp, smem, false);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int p = 0; p < HZ_POINTS; ++p) st_elem(block_totals, (size_t)blockIdx.x * HZ_POINTS + p, acc[p]);
    }
}

// Inter-block scan (one block of 1024 threads, nblocks <= 1024): block_seeds[b] = S(hi of block b) and
// value[p] = S(0) = f(u_p).
__global__ void __launch_bounds__(1024) horner_block_scan_kernel(const uint64_t* block_totals, int nblocks,
                                                                 const __grid_constant__ HornerParams hp,
                                                                 uint64_t* block_seeds, uint64_t* value) {
    __shared__ uint32_t smem[8 * 1024];
    const int b = threadIdx.x;
    Fr x[HZ_POINTS];
#pragma unroll
    for (int p = 0; p < HZ_POINTS; ++p) x[p] = b < nblocks ? ld_elem_rw<Fr>(block_totals, (size_t)b * HZ_POINTS + p) : Fr::zero();
    block_suffix_scan(x, hp, smem, true);  // x = Rb_b = sum_{b' >= b} Tb' (u^(256L))^(b'-b)
    // seed of block b = Rb_(b+1) (zero above the last block)
#pragma unroll 1
    for (int p = 0; p < HZ_POINTS; ++p) {
        Fr s = shift_down(x[p], Fr::zero(), smem);
        if (b < nblocks && block_seeds) st_elem(block_seeds, (size_t)b * HZ_POINTS + p, b + 1 < nblocks ? s : Fr::zero());
    }
    if (b == 0) {
#pragma unroll
        for (int p = 0; p < HZ_POINTS; ++p) st_elem(value, p, x[p]);
    }
}

// Pass C: quotients. h_p[k-1] = S_p(k) for k = 1..len-1, written to out + p*out_stride (elements).
__global__ void __launch_bounds__(HZ_THREADS) horner_divide_kernel(const uint64_t* coeffs, size_t len, int L,
                                                                   const __grid_constant__ HornerParams hp,
                                                                   const uint64_t* thread_totals, const uint64_t* block_seeds,
                                                                   uint64_t* out, size_t out_stride) {
    __shared__ uint32_t smem[8 * 1024];
    const int tid = threadIdx.x;
    const size_t gt = (size_t)blockIdx.x * HZ_THREADS + tid;
    const size_t lo = gt * L;
    Fr x[HZ_POINTS], bseed[HZ_POINTS];
#pragma unroll
    for (int p = 0; p < HZ_POINTS; ++p) {
        x[p] = ld_elem_rw<Fr>(thread_totals, gt * HZ_POINTS + p);
        bseed[p] = ld_elem_rw<Fr>(block_seeds, (size_t)blockIdx.x * HZ_POINTS + p);
        // fold the block's seed into the top chunk: S(lo_255) = T_255 + u^L * S(hi_255)
        if (tid == HZ_THREADS - 1) x[p] = fp_add(x[p], fp_mul(fr_from(hp.p[p].u_l), bseed[p]));
    }
    block_suffix_scan(x, hp, smem, false);  // x = S(lo_t)
    Fr s[HZ_POINTS], u[HZ_POINTS];
#pragma unroll 1
    for (int p = 0; p < HZ_POINTS; ++p) {
        s[p] = shift_down(x[p], bseed[p], smem);  // S(hi_t) = S(lo_(t+1)); the block's seed for the last thread
        u[p] = fr_from(hp.p[p].u);
    }
    if (lo >= len) return;
    const size_t hi = lo + L < len ? lo + L : len;
    for (size_t k = hi; k-- > lo;) {
        Fr c = ld_elem<Fr>(coeffs, k);
#pragma unroll
        for (int p = 0; p < HZ_POINTS; ++p) {
            s[p] = fp_add(fp_mul(s[p], u[p]), c);  // S(k)
            if (k >= 1) st_elem(out, (size_t)p * out_stride + (k - 1), s[p]);
        }
    }
}

// B[i] = sum_j q^j f_j[i]; f_0 = evals (len0), f_j (j >= 1) packed back to back in `folded`.
struct RlcParams {
    uint32_t qpow[40][8];
    int npolys;
};
__global__ void __launch_bounds__(256) rlc_kernel(const uint64_t* evals, const uint64_t* folded, size_t len0,
                                                  const __grid_constant__ RlcParams rp, uint64_t* out) {
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < len0; i += stride) {
        Fr acc = ld_elem<Fr>(evals, i);  // q^0 = 1
        size_t off = 0, lenj = len0 >> 1;
        for (int j = 1; j < rp.npolys && i < lenj; ++j) {
            acc = fp_add(acc, fp_mul(fr_from(rp.qpow[j]), ld_elem<Fr>(folded, off + i)));
            off += lenj;
            lenj >>= 1;
        }
        st_elem(out, i, acc);
    }
}

void store_words(uint32_t* dst, const HostFr& x) {
    for (int w = 0; w < 4; ++w) {
        dst[2 * w] = (uint32_t)x.l[w];
        dst[2 * w + 1] = (uint32_t)(x.l[w] >> 32);
    }
}

HornerParams horner_params(const HostFr u[HZ_POINTS], int L) {
    HornerParams hp;
    std::memset(&hp, 0, sizeof hp);
    for (int p = 0; p < HZ_POINTS; ++p) {
        store_words(hp.p[p].u, u[p]);
        HostFr ul = u[p];
        for (int s = 1; s < L; s <<= 1) ul = ul * ul;  // u^L (L a power of two)
        store_words(hp.p[p].u_l, ul);
        HostFr a = ul;
        for (int s = 0; s < 8; ++s) {
            store_words(hp.p[p].a_thread[s], a);
            a = a * a;
        }
        store_words(hp.p[p].u_bl, a);  // (u^L)^256
        for (int s = 0; s < 10; ++s) {
            store_words(hp.p[p].a_block[s], a);
            a = a * a;
        }
    }
    return hp;
}

using Guard = CtxGuard;

// chunk length so that a polynomial of `len` coefficients needs <= 1024 blocks of 256 chunks
int chunk_for(size_t len) {
    int L = 32;
    while ((len + (size_t)L * HZ_THREADS - 1) / ((size_t)L * HZ_THREADS) > 1024) L <<= 1;
    return L;
}

// f(u_p) for the three points -> d_value[3] (device)
int eval3(jb_ctx* c, const uint64_t* d_coeffs, size_t len, const HostFr u[HZ_POINTS], uint64_t* d_block_totals,
          uint64_t* d_value) {
    const int L = chunk_for(len);
    const HornerParams hp = horner_params(u, L);
    const size_t nblocks = (len + (size_t)L * HZ_THREADS - 1) / ((size_t)L * HZ_THREADS);
    horner_totals_kernel<false><<<(unsigned)nblocks, HZ_THREADS, 0, c->stream>>>(d_coeffs, len, L, hp, nullptr, d_block_totals);
    horner_block_scan_kernel<<<1, 1024, 0, c->stream>>>(d_block_totals, (int)nblocks, hp, nullptr, d_value);
    c->launches += 2;
    return c->check(cudaGetLastError(), "horner eval launch");
}

}  // namespace

extern "C" {

int jb_hyperkzg_open(jb_ctx* c, jb_srs srs, jb_table evals, const uint64_t* point, size_t ell,
                     jb_hkzg_challenge_r_fn challenge_r, jb_hkzg_challenge_q_fn challenge_q, void* user,
                     uint64_t* out_com, uint64_t* out_w, uint64_t* out_v) {
    if (!c) return JB_ERR_INVALID;
    if (ell == 0) return c->fail(JB_ERR_INVALID, "HyperKZGError::EmptyPoint");
    if (!point || !challenge_r || !challenge_q || !out_w || !out_v || (ell > 1 && !out_com))
        return c->fail(JB_ERR_INVALID, "hyperkzg: null argument");
    if (ell > 33) return c->fail(JB_ERR_UNSUPPORTED, "hyperkzg: ell must be <= 33");
    const size_t n = (size_t)1 << ell;
    const uint64_t* d_evals = nullptr;
    {
        Guard g(c);
        Table* t = c->find(evals);
        if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
        if (t->len != n) return c->fail(JB_ERR_INVALID, "hyperkzg: evaluation count must be 2^ell");
        auto it = c->srs.find(srs);
        if (it == c->srs.end()) return c->fail(JB_ERR_INVALID, "unknown srs handle");
        if (it->second.n < n) return c->fail(JB_ERR_LENGTH, "HyperKZGError::SrsTooSmall");
        for (size_t i = 0; i < ell; ++i)
            if (HostFr::geq_p(point + 4 * i)) return c->fail(JB_ERR_INVALID, "hyperkzg: point limbs not canonical");
        d_evals = t->buf;
    }
    // ---- workspace -------------------------------------------------------------------------------
    uint64_t *d_folded = nullptr, *d_b = nullptr, *d_h = nullptr, *d_tt = nullptr, *d_bt = nullptr, *d_bs = nullptr,
             *d_vals = nullptr;
    const int Lb = chunk_for(n);
    const size_t threads_b = (n + Lb - 1) / Lb;
    const size_t nblocks_b = (threads_b + HZ_THREADS - 1) / HZ_THREADS;
    int st;
    {
        Guard g(c);
        st = c->dev_alloc((void**)&d_folded, n * 32);  // sum_{j>=1} 2^(ell-j) < n
        if (st == JB_OK) st = c->dev_alloc((void**)&d_b, n * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_h, (size_t)HZ_POINTS * n * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_tt, nblocks_b * HZ_THREADS * HZ_POINTS * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_bt, 1024 * HZ_POINTS * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_bs, 1024 * HZ_POINTS * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_vals, (ell + 1) * HZ_POINTS * 32);
        // ---- phase 1: fold (scheme.rs:88-114): P_i = bind_low_to_high(P_(i-1), point[ell - i]) ------------
        const uint64_t* prev = d_evals;
        size_t off = 0, len = n;
        for (size_t i = 1; i < ell && st == JB_OK; ++i) {
            const uint64_t* x = point + 4 * (ell - i);
            BindScalar s;
            for (int w = 0; w < 4; ++w) {
                s.w[2 * w] = (uint32_t)x[w];
                s.w[2 * w + 1] = (uint32_t)(x[w] >> 32);
            }
            const bool hi4 = x[0] == 0 && x[1] == 0;
            const size_t half = len / 2;
            const unsigned grid = (unsigned)std::min<size_t>((half + 255) / 256, (size_t)c->sm_count * 8);
            uint64_t* dst = d_folded + 4 * off;
            if (hi4) bind_kernel<ORDER_LOW_TO_HIGH, true><<<grid, 256, 0, c->stream>>>(prev, dst, half, s);
            else bind_kernel<ORDER_LOW_TO_HIGH, false><<<grid, 256, 0, c->stream>>>(prev, dst, half, s);
            c->launches++;
            st = c->check(cudaGetLastError(), "hyperkzg fold launch");
            prev = dst;
            off += half;
            len = half;
        }
    }
    // ---- phase 1b: commit the intermediate polynomials (scheme.rs:141-145) ------------------------------
    {
        // The polynomials of <= 2^15 entries (the last min(ell - 1, 15) of them) are packed back to back with halving
        // lengths: one row-batched pass of the MSM pipeline commits them all (msm_halving_rows_device); 15 separate
        // MSMs of that size are latency-bound, one launch sequence each. The longer ones go one by one.
        const int h = ell >= 3 ? (int)(ell < 16 ? ell : 16) : 0;  // tail = the polynomials of lengths 2^(h-1) .. 2
        size_t off = 0, len = n / 2;
        size_t i = 1;
        for (; i < ell && st == JB_OK && (h == 0 || len > ((size_t)1 << (h - 1))); ++i) {
            st = jb_msm_g1_device(c, srs, 0, d_folded + 4 * off, len, out_com + 12 * (i - 1));
            off += len;
            len /= 2;
        }
        if (st == JB_OK && i < ell) {
            int rs = jb::msm_halving_rows_device(c, srs, d_folded + 4 * off, h, out_com + 12 * (i - 1));
            if (rs == JB_ERR_UNSUPPORTED) {  // no small table on this SRS handle: one by one
                for (; i < ell && st == JB_OK; ++i) {
                    st = jb_msm_g1_device(c, srs, 0, d_folded + 4 * off, len, out_com + 12 * (i - 1));
                    off += len;
                    len /= 2;
                }
            } else {
                st = rs;
            }
        }
    }
    uint64_t r_limbs[4], q_limbs[4];
    if (st == JB_OK && challenge_r(user, out_com, ell - 1, r_limbs) != 0) st = c->fail(JB_ERR_INVALID, "challenge_r callback failed");
    if (st == JB_OK && HostFr::geq_p(r_limbs)) st = c->fail(JB_ERR_INVALID, "challenge r not canonical");
    HostFr u[HZ_POINTS];
    if (st == JB_OK) {
        // ---- phase 3a: v[t][j] = f_j(u_t), u = [r, -r, r^2] (scheme.rs:151, kzg.rs:84-85) --------------------
        u[0] = HostFr::from_limbs(r_limbs);
        u[1] = -u[0];
        u[2] = u[0] * u[0];
        Guard g(c);
        size_t off = 0, len = n;
        for (size_t j = 0; j < ell && st == JB_OK; ++j) {
            const uint64_t* f = j == 0 ? d_evals : d_folded + 4 * off;
            st = eval3(c, f, len, u, d_bt, d_vals + 4 * HZ_POINTS * j);
            if (j >= 1) off += len;
            len /= 2;
        }
        std::vector<uint64_t> hv(ell * HZ_POINTS * 4);
        if (st == JB_OK) st = c->check(cudaMemcpyAsync(hv.data(), d_vals, hv.size() * 8, cudaMemcpyDeviceToHost, c->stream), "hyperkzg v D2H");
        if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "hyperkzg v sync");
        if (st == JB_OK)
            for (size_t j = 0; j < ell; ++j)
                for (int p = 0; p < HZ_POINTS; ++p) std::memcpy(out_v + ((size_t)p * ell + j) * 4, hv.data() + (j * HZ_POINTS + p) * 4, 32);
    }
    if (st == JB_OK && challenge_q(user, out_v, ell, q_limbs) != 0) st = c->fail(JB_ERR_INVALID, "challenge_q callback failed");
    if (st == JB_OK && HostFr::geq_p(q_limbs)) st = c->fail(JB_ERR_INVALID, "challenge q not canonical");
    if (st == JB_OK) {
        // ---- phase 3b: B = sum_j q^j f_j (kzg.rs:99-105), then the three quotients (kzg.rs:108-116) ----------
        Guard g(c);
        RlcParams rp;
        std::memset(&rp, 0, sizeof rp);
        rp.npolys = (int)ell;
        HostFr qp = HostFr::one(), q = HostFr::from_limbs(q_limbs);
        for (size_t j = 0; j < ell; ++j) {
            store_words(rp.qpow[j], qp);
            qp = qp * q;
        }
        rlc_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)c->sm_count * 8), 256, 0, c->stream>>>(d_evals, d_folded, n, rp, d_b);
        const HornerParams hp = horner_params(u, Lb);
        horner_totals_kernel<true><<<(unsigned)nblocks_b, HZ_THREADS, 0, c->stream>>>(d_b, n, Lb, hp, d_tt, d_bt);
        horner_block_scan_kernel<<<1, 1024, 0, c->stream>>>(d_bt, (int)nblocks_b, hp, d_bs, d_vals);
        horner_divide_kernel<<<(unsigned)nblocks_b, HZ_THREADS, 0, c->stream>>>(d_b, n, Lb, hp, d_tt, d_bs, d_h, n);
        c->launches += 4;
        st = c->check(cudaGetLastError(), "hyperkzg quotient launches");
    }
    for (int p = 0; p < HZ_POINTS && st == JB_OK; ++p) {
        if (n > 1) st = jb_msm_g1_device(c, srs, 0, d_h + (size_t)p * n * 4, n - 1, out_w + 12 * p);
    }
    {
        Guard g(c);
        c->dev_free(d_folded);
        c->dev_free(d_b);
        c->dev_free(d_h);
        c->dev_free(d_tt);
        c->dev_free(d_bt);
        c->dev_free(d_bs);
        c->dev_free(d_vals);
    }
    return st;
}

}  // extern "C"
