// Multilinear evaluation at a point on the device: Polynomial::evaluate (crates/jolt-poly/src/dense.rs:339-360)
//   * jb_table_evaluate_batch : resident field tables, left untouched
//   * jb_small_evaluate_batch : compact integer columns (the value of the promoted polynomial F::from(v))
//   * jb_one_hot_evaluate     : one-hot (RA) polynomials straight from their address columns
//   * jb_one_hot_pushforward  : G[k] = sum_{j: addr_j = k} eq(r_cycle, j), as resident tables
//
// One skeleton serves the first three. The point is split into n_hi + n_lo coordinates (n_lo <= 11) and the index
// x = h L + l (L = 2^n_lo), so eq(point, x) = e_hi[h] e_lo[l] with two small tables built by eq_build; the 2^n eq
// table is never formed. A thread owns a column l and walks rows h, accumulating sum_h e_hi[h] v(h L + l) UNREDUCED in
// a 17-word register accumulator (one plain 256 x 256 product per element, 256 x <= 128 for compact values). It
// reduces once, multiplies by e_lo[l] (again unreduced), and the block sums those products into per-output u64 lanes
// of 32-bit limb sums (REDUX over each warp, one atomic per lane per block); jb_wide_lanes_reduce_host folds the
// lanes. Integer lane sums are exact and order-free: results are bit-exact and deterministic whatever the schedule.
//
// Compact values are plain integers, not Montgomery values: sum e~ v (e~ = e R) is already R * sum e v, so the lanes
// fold to the plain integer value of the sum and the host multiplies by R^2 once (a Montgomery product) to get its
// Montgomery form. A negative value accumulates (p - e~) |v|.
//
// The pushforward is a scatter of eq(r_cycle, j) into K bins of 8 u64 lanes (32-bit limb sums, exact). A thread keeps
// a run (its current address and the field sum of its weights) and flushes it when the address changes; flushes are
// warp-aggregated (match.any, then one REDUX per 16-bit half-limb per group) so a skewed column - every cycle at one
// address, address-major runs - neither serialises on one bin nor costs an atomic per entry. Bins live in shared
// memory for K <= PF_SMEM_K (flushed once per block) and in global memory beyond.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "member.hpp"
#include "small_scalar.cuh"

using namespace jb;
using namespace jbi;
using Guard = CtxGuard;

namespace {

constexpr int EV_LO_MAX = 11;          // e_lo has at most 2^11 entries
constexpr int EV_BLOCK = 256;
constexpr uint32_t OH_SMEM_K = 256;    // one-hot evaluation: eq(r_addr, .) staged in shared memory up to 8 KiB
constexpr uint32_t PF_SMEM_K = 512;    // pushforward: block-private bins (K x 64 B) in shared memory up to 32 KiB
constexpr uint32_t NO_KEY = 0xffffffffu;

struct EvalCol {  // one output of a launch: its source and its lane block
    const void* ptr;
    uint64_t out;
};

// ---- value loaders: A += e * v(i) -----------------------------------------------------------------------------------
struct FieldSrc {
    static constexpr int SMEM_U4 = 1;
    __device__ void init(uint4*) const {}
    __device__ __forceinline__ void acc(uint32_t (&A)[17], const Fr& e, const void* p, size_t i, const uint4*) const {
        const Fr v = ld_elem<Fr>(static_cast<const uint64_t*>(p), i);
        mul_wide_acc_reg(A, e.v, v.v);
    }
};

template <int KIND>
struct SmallSrc {
    static constexpr int SMEM_U4 = 1;
    // 32-bit words of the magnitude
    static constexpr int BW = KIND <= SK_U32 ? 1 : (KIND == SK_U64 || KIND == SK_I64 || KIND == SK_S64) ? 2 : 4;
    __device__ void init(uint4*) const {}
    __device__ __forceinline__ void acc(uint32_t (&A)[17], const Fr& e, const void* p, size_t i, const uint4*) const {
        uint32_t mag[4];
        const bool neg = ld_small(p, i, KIND, mag);
        if (neg) {  // (p - e~) |v|: the Montgomery form of -e times |v|, still an exact non-negative integer product
            uint32_t ne[8];
            const uint32_t pm[8] = {FrParams::P(0), FrParams::P(1), FrParams::P(2), FrParams::P(3),
                                    FrParams::P(4), FrParams::P(5), FrParams::P(6), FrParams::P(7)};
            sub8(ne, pm, e.v);
            mul_wide_acc_bw<BW>(A, ne, mag);
        } else {
            mul_wide_acc_bw<BW>(A, e.v, mag);
        }
    }
};

// v_j = eq(r_addr, addr_j), 0 for the none value; an address >= K that is not none raises *bad and counts as 0.
template <int KIND, bool SMEM>
struct OneHotSrc {
    static constexpr int SMEM_U4 = SMEM ? 2 * OH_SMEM_K : 1;
    const uint64_t* eq_addr;
    uint32_t K;
    unsigned int* bad;
    __device__ void init(uint4* s) const {
        if (SMEM)
            for (uint32_t i = threadIdx.x; i < 2 * K; i += blockDim.x) s[i] = reinterpret_cast<const uint4*>(eq_addr)[i];
    }
    __device__ __forceinline__ void acc(uint32_t (&A)[17], const Fr& e, const void* p, size_t i, const uint4* s) const {
        const uint32_t a = KIND == SK_U8 ? (uint32_t)static_cast<const uint8_t*>(p)[i] : (uint32_t)static_cast<const uint16_t*>(p)[i];
        const uint32_t none = KIND == SK_U8 ? 0xffu : 0xffffu;
        if (a == none) return;
        if (a >= K) {
            atomicOr(bad, 1u);
            return;
        }
        const Fr v = SMEM ? elem_from<Fr>(s[2 * a], s[2 * a + 1]) : ld_elem_rw<Fr>(eq_addr, a);
        mul_wide_acc_reg(A, e.v, v.v);
    }
};

// grid: x = column blocks of L, y = row chunks of rpb rows, z strides over the outputs.
template <class Src>
__global__ void __launch_bounds__(EV_BLOCK, 2)
    mle_eval_kernel(Src src, const EvalCol* cols, size_t count, const uint64_t* e_hi, const uint64_t* e_lo, int n_lo,
                    size_t rows, size_t rpb, unsigned long long* lanes) {
    __shared__ uint4 s_tab[Src::SMEM_U4];
    __shared__ unsigned long long s_red[17];
    const int tid = threadIdx.x, lane = tid & 31;
    const size_t L = (size_t)1 << n_lo;
    const size_t l = (size_t)blockIdx.x * EV_BLOCK + tid;
    const size_t h0 = (size_t)blockIdx.y * rpb, h1 = min(rows, h0 + rpb);
    src.init(s_tab);
    const Fr el = l < L ? ld_elem<Fr>(e_lo, l) : Fr::zero();
    for (size_t z = blockIdx.z; z < count; z += gridDim.z) {
        if (tid < 17) s_red[tid] = 0;
        __syncthreads();  // (also orders src.init before the first gather)
        const void* p = cols[z].ptr;
        uint32_t A[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) A[k] = 0;
        if (l < L) {
#pragma unroll 2
            for (size_t h = h0; h < h1; ++h) src.acc(A, ld_elem<Fr>(e_hi, h), p, h * L + l, s_tab);
        }
        const Fr s = reduce_wide17<FrParams>(A, 1);
        uint32_t B[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) B[k] = 0;
        mul_wide_acc_reg(B, s.v, el.v);
        // sum each word over the warp (16-bit halves: no overflow in REDUX), then over the block, one atomic per lane
        unsigned long long mine = 0;
#pragma unroll
        for (int w = 0; w < 17; ++w) {
            const uint32_t lo = __reduce_add_sync(0xffffffffu, B[w] & 0xffffu);
            const uint32_t hi = __reduce_add_sync(0xffffffffu, B[w] >> 16);
            if (lane == w) mine = (unsigned long long)lo + ((unsigned long long)hi << 16);
        }
        if (lane < 17 && mine) atomicAdd(&s_red[lane], mine);
        __syncthreads();
        if (tid < 17 && s_red[tid]) atomicAdd(lanes + cols[z].out * 17 + tid, s_red[tid]);
        __syncthreads();
    }
}

// Warp-aggregated bin update: every thread with emit adds its field value `v` (8 canonical limbs) to bin `key`.
__device__ __forceinline__ void pf_flush(bool emit, uint32_t key, const Fr& v, unsigned long long* bins, int lane) {
    const unsigned m = __ballot_sync(0xffffffffu, emit);
    if (!emit) return;
    const unsigned peers = __match_any_sync(m, key);
    const int leader = __ffs(peers) - 1;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const uint32_t lo = __reduce_add_sync(peers, v.v[w] & 0xffffu);
        const uint32_t hi = __reduce_add_sync(peers, v.v[w] >> 16);
        if (lane == leader) atomicAdd(bins + (size_t)key * 8 + w, (unsigned long long)lo + ((unsigned long long)hi << 16));
    }
}

// lanes: count x K x 8 (zeroed); the grid is that of mle_eval_kernel over the T cycles.
template <int KIND, bool SMEM>
__global__ void __launch_bounds__(EV_BLOCK)
    pushforward_kernel(const EvalCol* cols, size_t count, const uint64_t* e_hi, const uint64_t* e_lo, int n_lo,
                       size_t rows, size_t rpb, uint32_t K, unsigned long long* lanes, unsigned int* bad) {
    __shared__ unsigned long long s_bins[SMEM ? PF_SMEM_K * 8 : 1];
    const int tid = threadIdx.x, lane = tid & 31;
    const size_t L = (size_t)1 << n_lo;
    const size_t l = (size_t)blockIdx.x * EV_BLOCK + tid;
    const size_t h0 = (size_t)blockIdx.y * rpb, h1 = min(rows, h0 + rpb);
    const uint32_t none = KIND == SK_U8 ? 0xffu : 0xffffu;
    const Fr el = l < L ? ld_elem<Fr>(e_lo, l) : Fr::zero();
    for (size_t z = blockIdx.z; z < count; z += gridDim.z) {
        unsigned long long* g_bins = lanes + cols[z].out * K * 8;
        unsigned long long* bins = SMEM ? s_bins : g_bins;
        if (SMEM) {
            for (uint32_t i = tid; i < K * 8; i += EV_BLOCK) s_bins[i] = 0;
            __syncthreads();
        }
        const void* p = cols[z].ptr;
        uint32_t cur = NO_KEY;  // the thread's run: address and the field sum of its weights
        Fr acc = Fr::zero();
        for (size_t h = h0; h < h1; ++h) {  // block-uniform trip count: the warp stays converged for pf_flush
            uint32_t a = NO_KEY;
            Fr w;
            if (l < L) {
                const size_t j = h * L + l;
                a = KIND == SK_U8 ? (uint32_t)static_cast<const uint8_t*>(p)[j] : (uint32_t)static_cast<const uint16_t*>(p)[j];
                if (a == none) {
                    a = NO_KEY;
                } else if (a >= K) {
                    atomicOr(bad, 1u);
                    a = NO_KEY;
                } else {
                    w = fp_mul(ld_elem<Fr>(e_hi, h), el);
                }
            }
            pf_flush(a != NO_KEY && cur != NO_KEY && a != cur, cur, acc, bins, lane);
            if (a != NO_KEY) {
                acc = a == cur ? fp_add(acc, w) : w;
                cur = a;
            }
        }
        pf_flush(cur != NO_KEY, cur, acc, bins, lane);
        if (SMEM) {
            __syncthreads();
            for (uint32_t i = tid; i < K * 8; i += EV_BLOCK)
                if (s_bins[i]) atomicAdd(g_bins + i, s_bins[i]);
            __syncthreads();
        }
    }
}

// n bins of 8 u64 limb-sum lanes -> canonical Montgomery elements (the lanes hold sums of Montgomery values, so the
// integer they encode is reduced mod p, not Montgomery-reduced): V = lo + top 2^256, V mod p = (lo mod p) + top R.
__global__ void __launch_bounds__(EV_BLOCK) bins_to_fr_kernel(const unsigned long long* lanes, size_t n, uint64_t* out) {
    for (size_t i = (size_t)blockIdx.x * EV_BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * EV_BLOCK) {
        Fr lo, top = Fr::zero();
        unsigned long long carry = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const unsigned long long v = lanes[i * 8 + w];
            const unsigned long long s = (v & 0xffffffffull) + (carry & 0xffffffffull);
            lo.v[w] = (uint32_t)s;
            carry = (v >> 32) + (carry >> 32) + (s >> 32);
        }
        top.v[0] = (uint32_t)carry;
        top.v[1] = (uint32_t)(carry >> 32);
#pragma unroll
        for (int k = 0; k < 5; ++k) cond_sub_p<FrParams>(lo.v);  // lo < 2^256 < 6p
        st_elem(out, i, fp_add(lo, fp_mul(top, Fr::r2())));  // top < 2^64 < p: montmul(top, R^2) = top R mod p
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------
bool pow2(size_t x) { return x != 0 && (x & (x - 1)) == 0; }
int log2_of(size_t x) {
    int l = 0;
    while (x >> (l + 1)) ++l;
    return l;
}

int check_point(jb_ctx* c, const uint64_t* point, size_t nvars, const char* what) {
    if (nvars && !point) return c->fail(JB_ERR_INVALID, what);
    for (size_t i = 0; i < nvars; ++i)
        if (!canonical_fr(point + 4 * i)) return c->fail(JB_ERR_INVALID, "evaluate: point limbs not canonical (>= r)");
    return JB_OK;
}

// What every evaluation shares: the split of the point, its two eq tables, the launch shape and the lane tail.
struct EvalPlan {
    jb_ctx* c;
    int n_lo = 0;
    size_t L = 1, rows = 1, rpb = 1, count = 0;
    dim3 grid;
    uint64_t* d_e = nullptr;                 // e_hi (rows entries), then e_lo (L entries)
    EvalCol* d_cols = nullptr;
    unsigned long long* d_lanes = nullptr;   // the outputs' lanes, then one word for the bad-address flag
    size_t nlanes = 0;
    std::vector<EvalCol> cols;
    explicit EvalPlan(jb_ctx* ctx) : c(ctx) {}
    ~EvalPlan() {
        c->dev_free(d_e);
        c->dev_free(d_cols);
        c->dev_free(d_lanes);
    }
    const uint64_t* e_hi() const { return d_e; }
    const uint64_t* e_lo() const { return d_e + 4 * rows; }
    unsigned int* bad() const { return reinterpret_cast<unsigned int*>(d_lanes + nlanes); }

    // point: nvars coordinates (validated); lanes_per_output u64 lanes per column (17 or K x 8), zeroed.
    int begin(const uint64_t* point, size_t nvars, size_t lanes_per_output) {
        n_lo = (int)std::min<size_t>(nvars, EV_LO_MAX);
        L = (size_t)1 << n_lo;
        rows = (size_t)1 << (nvars - n_lo);
        count = cols.size();
        nlanes = count * lanes_per_output;
        int st = c->dev_alloc((void**)&d_e, (rows + L) * 32);
        if (st == JB_OK) st = c->dev_alloc((void**)&d_cols, count * sizeof(EvalCol));
        if (st == JB_OK) st = c->dev_alloc((void**)&d_lanes, (nlanes + 1) * 8);
        if (st != JB_OK) return st;
        st = c->check(cudaMemsetAsync(d_lanes, 0, (nlanes + 1) * 8, c->stream), "evaluate lanes memset");
        if (st == JB_OK)
            st = c->check(cudaMemcpyAsync(d_cols, cols.data(), count * sizeof(EvalCol), cudaMemcpyHostToDevice, c->stream),
                          "evaluate columns H2D");
        if (st == JB_OK) st = eq_build(c, point, nvars - n_lo, nullptr, d_e);
        if (st == JB_OK) st = eq_build(c, point + 4 * (nvars - n_lo), n_lo, nullptr, d_e + 4 * rows);
        // one wave at two blocks per SM over all outputs; a block walks at least its share of the rows
        const size_t gx = (L + EV_BLOCK - 1) / EV_BLOCK, gz = std::min<size_t>(count, 65535);
        const size_t target = (size_t)c->sm_count * 2;
        size_t gy = std::max<size_t>(1, target / (gx * gz));
        gy = std::min(gy, rows);
        rpb = (rows + gy - 1) / gy;
        gy = (rows + rpb - 1) / rpb;
        grid = dim3((unsigned)gx, (unsigned)gy, (unsigned)gz);
        return st;
    }

    // Waits for the launches, checks the flag and folds the lanes: out[i] (4 limbs each, count of them); outputs with
    // plain[i] set hold a plain integer value and are moved to Montgomery form.
    int finish(uint64_t* out, const std::vector<char>* plain) {
        std::vector<uint64_t> h(nlanes + 1);
        int st = c->check(cudaMemcpyAsync(h.data(), d_lanes, (nlanes + 1) * 8, cudaMemcpyDeviceToHost, c->stream),
                          "evaluate lanes D2H");
        if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "evaluate sync");
        if (st != JB_OK) return st;
        if ((uint32_t)h[nlanes]) return c->fail(JB_ERR_INVALID, "one-hot: an address >= K that is not the none value");
        jb_wide_lanes_reduce_host(h.data(), count, out);
        if (plain) {
            const HostFr r2{{HostFr::R2[0], HostFr::R2[1], HostFr::R2[2], HostFr::R2[3]}};
            for (size_t i = 0; i < count; ++i)
                if ((*plain)[i]) (HostFr::from_limbs(out + 4 * i) * r2).store(out + 4 * i);
        }
        return JB_OK;
    }
};

template <class Src>
int launch_eval(EvalPlan& p, const Src& src, size_t first, size_t n) {
    if (n == 0) return JB_OK;
    dim3 g = p.grid;
    g.z = (unsigned)std::min<size_t>(n, g.z);
    mle_eval_kernel<Src><<<g, EV_BLOCK, 0, p.c->stream>>>(src, p.d_cols + first, n, p.e_hi(), p.e_lo(), p.n_lo, p.rows,
                                                          p.rpb, p.d_lanes);
    p.c->launches++;
    return p.c->check(cudaGetLastError(), "mle_eval_kernel launch");
}

int launch_small(EvalPlan& p, int kind, size_t first, size_t n) {
    switch (kind) {
        case SK_U8: return launch_eval(p, SmallSrc<SK_U8>{}, first, n);
        case SK_U16: return launch_eval(p, SmallSrc<SK_U16>{}, first, n);
        case SK_U32: return launch_eval(p, SmallSrc<SK_U32>{}, first, n);
        case SK_U64: return launch_eval(p, SmallSrc<SK_U64>{}, first, n);
        case SK_U128: return launch_eval(p, SmallSrc<SK_U128>{}, first, n);
        case SK_I64: return launch_eval(p, SmallSrc<SK_I64>{}, first, n);
        case SK_I128: return launch_eval(p, SmallSrc<SK_I128>{}, first, n);
        case SK_S64: return launch_eval(p, SmallSrc<SK_S64>{}, first, n);
        default: return launch_eval(p, SmallSrc<SK_S128>{}, first, n);
    }
}

int check_one_hot(jb_ctx* c, const void* const* columns, size_t count, int kind, size_t T, size_t K, int on_device,
                  const char* what) {
    if (kind != SK_U8 && kind != SK_U16) return c->fail(JB_ERR_INVALID, "one-hot: addresses must be JB_SCALAR_U8 or JB_SCALAR_U16");
    if (!pow2(T) || !pow2(K)) return c->fail(JB_ERR_INVALID, "one-hot: K and T must be powers of two");
    if (on_device != 0 && on_device != 1) return c->fail(JB_ERR_INVALID, "one-hot: on_device must be 0 or 1");
    if (T >= ((size_t)1 << 31)) return c->fail(JB_ERR_UNSUPPORTED, "one-hot: T must be < 2^31");
    if (K > ((size_t)1 << 16)) return c->fail(JB_ERR_UNSUPPORTED, "one-hot: K must be <= 2^16");
    if (count && !columns) return c->fail(JB_ERR_INVALID, what);
    for (size_t p = 0; p < count; ++p) {
        if (!columns[p]) return c->fail(JB_ERR_INVALID, what);
        if (on_device && ((uintptr_t)columns[p] % (size_t)small_kind_bytes(kind)))
            return c->fail(JB_ERR_INVALID, "one-hot: misaligned device column");
    }
    return JB_OK;
}

}  // namespace

extern "C" {

int jb_table_evaluate_batch(jb_ctx* c, const jb_table* tables, size_t count, const uint64_t* point, size_t nvars,
                            uint64_t* out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;  // without a device there is no context
    if (count && (!tables || !out)) return c->fail(JB_ERR_INVALID, "table_evaluate: null pointer");
    int st = check_point(c, point, nvars, "table_evaluate: null point");
    if (st != JB_OK) return st;
    if (nvars > 40) return c->fail(JB_ERR_UNSUPPORTED, "table_evaluate: at most 40 variables");
    if (count == 0) return JB_OK;
    Guard g(c);
    EvalPlan p(c);
    for (size_t i = 0; i < count; ++i) {
        Table* t = c->find(tables[i]);
        if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
        if (t->len != ((size_t)1 << nvars)) return c->fail(JB_ERR_INVALID, "table_evaluate: every table must have 2^nvars entries");
        p.cols.push_back(EvalCol{t->buf, i});
    }
    st = p.begin(point, nvars, 17);
    if (st == JB_OK) st = launch_eval(p, FieldSrc{}, 0, count);
    if (st == JB_OK) st = p.finish(out, nullptr);
    return st;
}

int jb_small_evaluate_batch(jb_ctx* c, const void* const* columns, size_t count, const int* kinds, size_t len,
                            int on_device, const uint64_t* point, size_t nvars, uint64_t* out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;
    if (count && (!columns || !kinds || !out)) return c->fail(JB_ERR_INVALID, "small_evaluate: null pointer");
    if (on_device != 0 && on_device != 1) return c->fail(JB_ERR_INVALID, "small_evaluate: on_device must be 0 or 1");
    if (!pow2(len)) return c->fail(JB_ERR_INVALID, "small_evaluate: the length must be a power of two");
    if (nvars != (size_t)log2_of(len)) return c->fail(JB_ERR_INVALID, "small_evaluate: nvars != log2(length)");
    int st = check_point(c, point, nvars, "small_evaluate: null point");
    if (st != JB_OK) return st;
    if (nvars > 40) return c->fail(JB_ERR_UNSUPPORTED, "small_evaluate: at most 40 variables");
    for (size_t i = 0; i < count; ++i) {
        if (kinds[i] < SK_U8 || kinds[i] > SK_LAST) return c->fail(JB_ERR_INVALID, "small_evaluate: unknown scalar kind");
        if (!columns[i]) return c->fail(JB_ERR_INVALID, "small_evaluate: null column");
        const size_t align = std::min(8, small_kind_bytes(kinds[i]));
        if (on_device && ((uintptr_t)columns[i] % align)) return c->fail(JB_ERR_INVALID, "small_evaluate: misaligned device column");
    }
    if (count == 0) return JB_OK;
    Guard g(c);
    EvalPlan p(c);
    Columns cols(c);
    // one launch per kind: the outputs are grouped by kind, each keeping its own lane block
    std::vector<size_t> first(SK_LAST + 2, 0);
    for (int k = SK_U8; k <= SK_LAST; ++k) {
        first[k] = p.cols.size();
        for (size_t i = 0; i < count && st == JB_OK; ++i) {
            if (kinds[i] != k) continue;
            const void* d = nullptr;
            st = cols.get(columns[i], len * (size_t)small_kind_bytes(k), on_device, &d);
            p.cols.push_back(EvalCol{d, i});
        }
    }
    first[SK_LAST + 1] = p.cols.size();
    if (st == JB_OK) st = p.begin(point, nvars, 17);
    for (int k = SK_U8; k <= SK_LAST && st == JB_OK; ++k) st = launch_small(p, k, first[k], first[k + 1] - first[k]);
    const std::vector<char> plain(count, 1);
    if (st == JB_OK) st = p.finish(out, &plain);
    return st;
}

int jb_one_hot_evaluate(jb_ctx* c, const void* const* columns, size_t count, int kind, size_t T, size_t K, int layout,
                        int on_device, const uint64_t* point, uint64_t* out) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;
    int st = check_one_hot(c, columns, count, kind, T, K, on_device, "one_hot_evaluate: null pointer");
    if (st != JB_OK) return st;
    if (layout != JB_ONE_HOT_CYCLE_MAJOR && layout != JB_ONE_HOT_ADDRESS_MAJOR)
        return c->fail(JB_ERR_INVALID, "one_hot_evaluate: unknown layout");
    const size_t log_t = (size_t)log2_of(T), log_k = (size_t)log2_of(K);
    if (count && !out) return c->fail(JB_ERR_INVALID, "one_hot_evaluate: null pointer");
    if ((st = check_point(c, point, log_t + log_k, "one_hot_evaluate: null point")) != JB_OK) return st;
    if (count == 0) return JB_OK;
    const uint64_t* r_cycle = layout == JB_ONE_HOT_CYCLE_MAJOR ? point : point + 4 * log_k;
    const uint64_t* r_addr = layout == JB_ONE_HOT_CYCLE_MAJOR ? point + 4 * log_t : point;
    Guard g(c);
    EvalPlan p(c);
    Columns cols(c);
    for (size_t i = 0; i < count && st == JB_OK; ++i) {
        const void* d = nullptr;
        st = cols.get(columns[i], T * (size_t)small_kind_bytes(kind), on_device, &d);
        p.cols.push_back(EvalCol{d, i});
    }
    uint64_t* d_eq = nullptr;
    if (st == JB_OK) st = c->dev_alloc((void**)&d_eq, K * 32);
    if (st == JB_OK) st = eq_build(c, r_addr, log_k, nullptr, d_eq);
    if (st == JB_OK) st = p.begin(r_cycle, log_t, 17);
    if (st == JB_OK) {
        const bool sm = K <= OH_SMEM_K;
        if (kind == SK_U8) st = sm ? launch_eval(p, OneHotSrc<SK_U8, true>{d_eq, (uint32_t)K, p.bad()}, 0, count)
                                   : launch_eval(p, OneHotSrc<SK_U8, false>{d_eq, (uint32_t)K, p.bad()}, 0, count);
        else st = sm ? launch_eval(p, OneHotSrc<SK_U16, true>{d_eq, (uint32_t)K, p.bad()}, 0, count)
                     : launch_eval(p, OneHotSrc<SK_U16, false>{d_eq, (uint32_t)K, p.bad()}, 0, count);
    }
    if (st == JB_OK) st = p.finish(out, nullptr);
    c->dev_free(d_eq);
    return st;
}

int jb_one_hot_pushforward(jb_ctx* c, const void* const* columns, size_t count, int kind, size_t T, size_t K,
                           int on_device, const uint64_t* r_cycle, jb_table* out_tables) {
    if (!c) return jb_device_count() > 0 ? JB_ERR_INVALID : JB_ERR_NO_DEVICE;
    int st = check_one_hot(c, columns, count, kind, T, K, on_device, "one_hot_pushforward: null pointer");
    if (st != JB_OK) return st;
    const size_t log_t = (size_t)log2_of(T);
    if (count && !out_tables) return c->fail(JB_ERR_INVALID, "one_hot_pushforward: null pointer");
    if ((st = check_point(c, r_cycle, log_t, "one_hot_pushforward: null point")) != JB_OK) return st;
    if (count == 0) return JB_OK;
    Guard g(c);
    EvalPlan p(c);
    Columns cols(c);
    for (size_t i = 0; i < count && st == JB_OK; ++i) {
        const void* d = nullptr;
        st = cols.get(columns[i], T * (size_t)small_kind_bytes(kind), on_device, &d);
        p.cols.push_back(EvalCol{d, i});
    }
    if (st == JB_OK) st = p.begin(r_cycle, log_t, K * 8);
    if (st == JB_OK) {
        const bool sm = K <= PF_SMEM_K;
#define JB_PF_LAUNCH(KD, SM)                                                                                       \
    pushforward_kernel<KD, SM><<<p.grid, EV_BLOCK, 0, c->stream>>>(p.d_cols, count, p.e_hi(), p.e_lo(), p.n_lo, p.rows, \
                                                                    p.rpb, (uint32_t)K, p.d_lanes, p.bad())
        if (kind == SK_U8) { if (sm) JB_PF_LAUNCH(SK_U8, true); else JB_PF_LAUNCH(SK_U8, false); }
        else { if (sm) JB_PF_LAUNCH(SK_U16, true); else JB_PF_LAUNCH(SK_U16, false); }
#undef JB_PF_LAUNCH
        c->launches++;
        st = c->check(cudaGetLastError(), "pushforward_kernel launch");
    }
    unsigned int flag = 0;
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(&flag, p.bad(), 4, cudaMemcpyDeviceToHost, c->stream), "pushforward flag D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "pushforward sync");
    if (st == JB_OK && flag) st = c->fail(JB_ERR_INVALID, "one-hot: an address >= K that is not the none value");
    // the tables are created only once the bins are known to be valid
    std::vector<jb_table> made;
    for (size_t i = 0; i < count && st == JB_OK; ++i) {
        Table t;
        st = c->dev_alloc((void**)&t.buf, K * 32);
        if (st != JB_OK) break;
        t.cap = t.len = K;
        const jb_table h = c->next_id++;
        c->tables[h] = t;
        made.push_back(h);
        const unsigned grid = (unsigned)std::min<size_t>((K + EV_BLOCK - 1) / EV_BLOCK, (size_t)c->sm_count * 8);
        bins_to_fr_kernel<<<grid, EV_BLOCK, 0, c->stream>>>(p.d_lanes + i * K * 8, K, t.buf);
        c->launches++;
        st = c->check(cudaGetLastError(), "bins_to_fr_kernel launch");
    }
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "pushforward tables sync");
    if (st != JB_OK) {
        for (jb_table h : made) {
            c->release(c->tables[h]);
            c->tables.erase(h);
        }
        return st;
    }
    std::memcpy(out_tables, made.data(), count * sizeof(jb_table));
    return JB_OK;
}

}  // extern "C"
