// Product members over sources (jb_member_create_product_sources): one round of
//   sum_x [scale * eq(w, x) *] prod_{i < d} f_i(x)        (1 <= d <= 16 sources)
// per launch, one thread per pair index y (grid-stride). Rounds 0 and 1 read the sources in their own format (the
// loads of sources.cuh; round 1 binds them into the member's len/2 buffers with bind_pair, as source_round_kernel
// does); later rounds read and bind the field tables (HighToLow in place, LowToHigh ping-pong).
//
// Evaluation by a product tree instead of per point. A node of degree k is held as its values at t = 0..k-1 and its
// leading coefficient L (the value "at infinity"), k + 1 field elements; a leaf is (lo, D = hi - lo). Two nodes A, B
// of degrees a, b make C = A B of degree c = a + b: L_C = L_A L_B and C(t) = A(t) B(t) for t < c, where A and B are
// extended past their own points by their backward difference tables (a steps of additions per point; the a-th
// difference is the constant a! L_A, formed by double-and-add). So C costs c + 1 Montgomery products where the
// per-point loop of expr_sweep costs (c - 1) products at each of c + 1 points. Nodes are merged as a binary counter
// over the factors (a balanced tree for d a power of two); the root's values are s_y(0), s_y(1), .., s_y(d - 1) and
// s_y(inf), and the split-eq weight of the pair is multiplied into the first leaf (2 products) instead of into
// every point. Field arithmetic is exact, so the published sums are bit-identical to evaluating prod_i (lo_i + t D_i)
// directly (tests/test_product_ref_cpu.py models the scheme step by step).
//
// The nodes live in a per-thread column of dynamic shared memory laid out [word][thread] as in expr_pass.cuh (node
// positions depend on d, a runtime value, so they cannot be registers without local memory), and so do the round's
// sums (product_epilogue). Merges write C over A and B in place: C(t) lands on the slot of A(t), read at the same
// step, or of a B value consumed earlier. The difference tables sit above the stack.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>

#include "member.hpp"
#include "sources.cuh"

using namespace jb;
using namespace jbi;

namespace {

constexpr int PROD_BLOCK = 64;
constexpr int PROD_MAX = JB_PRODUCT_MAX_FACTORS;
constexpr int PROD_MAX_POINTS = PROD_MAX + 1;      // s(0), s(1), s(2..d-1), s(inf)
constexpr int PROD_MAX_STEPS = 2 * PROD_MAX - 1;   // d leaves, d - 1 merges
constexpr int PROD_MAX_CHILD = PROD_MAX / 2;       // a merged child has degree <= 8 (binary counter, d <= 16)
constexpr int PROD_INF = -1;
constexpr size_t PROD_SMEM_MAX = 224 * 1024;       // dynamic shared memory: below sm_90's 227 KiB opt-in ceiling with the static part
enum : uint8_t { PROD_LEAF = 0, PROD_MERGE = 1 };

// The kernel parameter: tables, sources and the evaluation program of the member (every existing pass keeps its own
// 8-table structs). Node slots are 8 words each in the thread's column.
struct ProductParams {
    static constexpr int ADDRESS_WIDEST = SK_U32;  // product members over sources: u8 / u16 / u32 addresses
    const uint64_t* in[PROD_MAX];   // field tables (null for a source read from its column)
    uint64_t* out[PROD_MAX];        // bind destinations
    const uint64_t* e_out;          // WEIGHTED: the split-eq weight e_out[y >> in_bits] * e_in[y & mask]
    const uint64_t* e_in;
    int in_bits;
    // sources (rounds 0 and 1; the fields src_value reads)
    const void* values[PROD_MAX];
    const uint64_t* eq[PROD_MAX];
    uint32_t K[PROD_MAX];
    uint32_t smem[PROD_MAX];
    uint8_t type[PROD_MAX];
    uint8_t kind[PROD_MAX];
    // program: LEAF puts factor arg[s] at slot base[s]; MERGE multiplies the node at base[s] (degree a[s]) by the
    // one above it (degree b[s]); the last step is the root, at slot 0
    uint8_t op[PROD_MAX_STEPS], arg[PROD_MAX_STEPS], base[PROD_MAX_STEPS], a[PROD_MAX_STEPS], b[PROD_MAX_STEPS];
    uint32_t fact[PROD_MAX_CHILD + 1];  // k!
    int8_t point[PROD_MAX_POINTS];      // published points in kernel-value order (PROD_INF = infinity)
    int d, nsteps, npoints, skip1;
    int acc;                            // first slot of the thread's round sums
    uint32_t red;                       // word offset of the block-sum scratch
};
static_assert(sizeof(ProductParams) < 4096, "the program must stay a small kernel parameter");

__device__ __forceinline__ Fr prod_ld(const uint32_t* col, int slot) {
    Fr x;
#pragma unroll
    for (int w = 0; w < 8; ++w) x.v[w] = col[(slot * 8 + w) * PROD_BLOCK];
    return x;
}
__device__ __forceinline__ void prod_st(uint32_t* col, int slot, const Fr& x) {
#pragma unroll
    for (int w = 0; w < 8; ++w) col[(slot * 8 + w) * PROD_BLOCK] = x.v[w];
}

// k x by double-and-add (k >= 1 small: the additions are the "small-integer multiple" of DESIGN section 4)
__device__ __forceinline__ Fr mul_small(const Fr& x, uint32_t k) {
    Fr r = x;
    for (int bit = 30 - __clz(k); bit >= 0; --bit) {
        r = fp_add(r, r);
        if ((k >> bit) & 1) r = fp_add(r, x);
    }
    return r;
}

// The backward difference table at t = k - 1 of the node at S (degree k) into T: T[k-1-l] = nabla^l p(k - 1), and
// T[k] = k! L, the constant k-th difference.
__device__ __forceinline__ void diff_table(uint32_t* col, int S, int k, int T, uint32_t fact) {
    for (int j = 0; j + 1 < k; ++j) prod_st(col, T + j, fp_sub(prod_ld(col, S + j + 1), prod_ld(col, S + j)));
    prod_st(col, T + k - 1, prod_ld(col, S + k - 1));
    for (int l = 2; l < k; ++l)
        for (int j = 0; j + l < k; ++j) prod_st(col, T + j, fp_sub(prod_ld(col, T + j + 1), prod_ld(col, T + j)));
    prod_st(col, T + k, mul_small(prod_ld(col, S + k), fact));
}

// The table's node at the next point: k additions.
__device__ __forceinline__ Fr diff_step(uint32_t* col, int T, int k) {
    Fr v = fp_add(prod_ld(col, T), prod_ld(col, T + k));
    prod_st(col, T, v);
    for (int j = 1; j < k; ++j) {
        v = fp_add(prod_ld(col, T + j), v);
        prod_st(col, T + j, v);
    }
    return v;
}

// C = A B in place (A at SA, degree a; B right above it, degree b). skip1: C(1) is not needed (the root of a round
// whose s(1) comes from the claim).
__device__ __forceinline__ void merge(uint32_t* col, const ProductParams& pp, int SA, int a, int b, bool skip1) {
    const int SB = SA + a + 1, c = a + b, TA = SB + b + 1, TB = TA + a + 1;
    diff_table(col, SA, a, TA, pp.fact[a]);
    diff_table(col, SB, b, TB, pp.fact[b]);
    const Fr lc = fp_mul(prod_ld(col, SA + a), prod_ld(col, SB + b));
    for (int t = 0; t < c; ++t) {
        const Fr x = t < a ? prod_ld(col, SA + t) : diff_step(col, TA, a);
        const Fr z = t < b ? prod_ld(col, SB + t) : diff_step(col, TB, b);
        if (skip1 && t == 1) continue;
        prod_st(col, SA + t, fp_mul(x, z));
    }
    prod_st(col, SA + c, lc);
}

// Block sum of every thread's x into tot (thread 0 writes; the caller synchronises before red and tot are used again).
__device__ __forceinline__ void block_sum_slot(Fr x, uint32_t* red, uint32_t* tot) {
    Fr one[1] = {x};
    block_sum<1>(one, red);
    if (threadIdx.x == 0)
#pragma unroll
        for (int w = 0; w < 8; ++w) tot[w] = one[0].v[w];
}

// round_epilogue one point at a time: the round's up to 17 sums never sit in registers together (block_sum /
// round_epilogue over all of them would hold 2 x 17 elements and spill). Same ticket counter, partial layout and
// host-mapped publish as round_epilogue with lanes == 0 (product members are not sharded); the slot holds 16 values
// below its sequence flag (word 64), so a 17th goes to words [72, 76).
__device__ __forceinline__ void product_epilogue(const uint32_t* col, const ProductParams& pp, uint32_t* red,
                                                 const RoundOut& out) {
    __shared__ bool is_last;
    uint32_t* tot = red + (PROD_BLOCK / 32) * 8;  // the block's totals, PROD_MAX_POINTS x 8 words
    for (int e = 0; e < pp.npoints; ++e) {
        block_sum_slot(prod_ld(col, pp.acc + e), red, tot + 8 * e);
        __syncthreads();
    }
    if (gridDim.x > 1) {
        if (threadIdx.x == 0) {
            for (int e = 0; e < pp.npoints; ++e) {
                Fr x;
#pragma unroll
                for (int w = 0; w < 8; ++w) x.v[w] = tot[8 * e + w];
                st_elem(out.partial, (size_t)blockIdx.x * PROD_MAX_POINTS + e, x);
            }
            __threadfence();
            const unsigned int ticket = atomicAdd(out.counter, 1u);
            is_last = (ticket == gridDim.x - 1);
        }
        __syncthreads();
        if (!is_last) return;
        __threadfence();
        for (int e = 0; e < pp.npoints; ++e) {
            Fr x = Fr::zero();
            for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x)
                x = fp_add(x, ld_elem_cg<Fr>(out.partial, (size_t)b * PROD_MAX_POINTS + e));
            block_sum_slot(x, red, tot + 8 * e);
            __syncthreads();
        }
        if (threadIdx.x == 0) *out.counter = 0;
    }
    if (threadIdx.x != 0) return;
    for (int e = 0; e < pp.npoints; ++e)
        for (int w = 0; w < 4; ++w)
            out.result[4 * e + (e < 16 ? 0 : 8) + w] = (uint64_t)tot[8 * e + 2 * w] | ((uint64_t)tot[8 * e + 2 * w + 1] << 32);
    if (out.flag) {
        __threadfence_system();
        *out.flag = out.seq;
    }
}

// Factor j's pair: HighToLow y, y + P [, y + 2P, y + 3P]; LowToHigh 2y, 2y + 1 [4y .. 4y + 3]. SRC: the factor may
// still be a column; BIND: bind first and store the bound pair.
template <int ORDER, bool SRC, bool BIND, bool HI4>
__device__ __forceinline__ void load_factor(const ProductParams& pp, int j, size_t y, size_t pairs, const BindScalar& s,
                                            const uint32_t* dsm, Fr& lo, Fr& hi) {
    const size_t i0 = ORDER == ORDER_HIGH_TO_LOW ? y : (BIND ? 4 : 2) * y;
    const size_t i1 = ORDER == ORDER_HIGH_TO_LOW ? (BIND ? y + 2 * pairs : y + pairs) : i0 + 1;
    const size_t i2 = ORDER == ORDER_HIGH_TO_LOW ? y + pairs : i0 + 2;
    const size_t i3 = ORDER == ORDER_HIGH_TO_LOW ? y + 3 * pairs : i0 + 3;
    if (!SRC || pp.type[j] == JB_SOURCE_TABLE) {
        const uint64_t* in = pp.in[j];
        if (BIND) {
            if (ORDER == ORDER_HIGH_TO_LOW) {
                lo = bind_pair<HI4>(ld_elem_rw<Fr>(in, i0), ld_elem_rw<Fr>(in, i1), s);
                hi = bind_pair<HI4>(ld_elem_rw<Fr>(in, i2), ld_elem_rw<Fr>(in, i3), s);
            } else {
                lo = bind_pair<HI4>(ld_elem<Fr>(in, i0), ld_elem<Fr>(in, i1), s);
                hi = bind_pair<HI4>(ld_elem<Fr>(in, i2), ld_elem<Fr>(in, i3), s);
            }
        } else if (ORDER == ORDER_HIGH_TO_LOW) {
            lo = ld_elem_rw<Fr>(in, i0);
            hi = ld_elem_rw<Fr>(in, i1);
        } else {
            lo = ld_elem<Fr>(in, i0);
            hi = ld_elem<Fr>(in, i1);
        }
    } else if (BIND) {
        lo = bind_pair<HI4>(src_value(pp, j, i0, dsm), src_value(pp, j, i1, dsm), s);
        hi = bind_pair<HI4>(src_value(pp, j, i2, dsm), src_value(pp, j, i3, dsm), s);
    } else {
        lo = src_value(pp, j, i0, dsm);
        hi = src_value(pp, j, i1, dsm);
    }
    if (BIND) {
        st_elem(pp.out[j], ORDER == ORDER_HIGH_TO_LOW ? y : 2 * y, lo);
        st_elem(pp.out[j], ORDER == ORDER_HIGH_TO_LOW ? y + pairs : 2 * y + 1, hi);
    }
}

// One round. SRC (rounds 0 and 1): factors may be columns, one-hot eq tables staged in shared memory where
// pp.smem says so. Always PROD_MAX_POINTS sums are published (values >= 16 past the slot's sequence flag); the host
// reads `npoints`.
template <int ORDER, bool SRC, bool BIND, bool HI4, bool WEIGHTED>
__global__ void __launch_bounds__(PROD_BLOCK, 4)
    product_round_kernel(const __grid_constant__ ProductParams pp, size_t pairs, BindScalar s, RoundOut out) {
    extern __shared__ uint32_t dsm[];
    uint32_t* col = dsm + threadIdx.x;
    if (SRC) {
        for (int j = 0; j < pp.d; ++j)
            if (pp.type[j] == JB_SOURCE_ONE_HOT && pp.smem[j] != SRC_NO_SMEM)
                for (uint32_t i = threadIdx.x; i < 2 * pp.K[j]; i += blockDim.x)
                    reinterpret_cast<uint4*>(dsm + pp.smem[j])[i] = reinterpret_cast<const uint4*>(pp.eq[j])[i];
        __syncthreads();
    }
    // the round's sums: slots of the column while pairs are swept (registers would hold 17 elements across the
    // merges), registers for the block sum
    for (int e = 0; e < pp.npoints; ++e) prod_st(col, pp.acc + e, Fr::zero());
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < pairs; y += stride) {
        const size_t yn = y + stride;
        if (yn < pairs) {
            for (int j = 0; j < pp.d; ++j) {
                if (SRC && pp.type[j] != JB_SOURCE_TABLE) continue;  // (a column entry is 1-24 bytes: the lines are shared)
                if (ORDER == ORDER_HIGH_TO_LOW) {
                    prefetch_l2(pp.in[j], yn);
                    prefetch_l2(pp.in[j], yn + pairs);
                    if (BIND) {
                        prefetch_l2(pp.in[j], yn + 2 * pairs);
                        prefetch_l2(pp.in[j], yn + 3 * pairs);
                    }
                } else {
                    prefetch_l2(pp.in[j], (BIND ? 4 : 2) * yn);
                }
            }
        }
        Fr wgt;
        if (WEIGHTED) {
            const size_t yo = y >> pp.in_bits;
            wgt = fp_mul(ld_elem<Fr>(pp.e_out, yo), ld_elem<Fr>(pp.e_in, y - (yo << pp.in_bits)));
        }
        for (int st = 0; st < pp.nsteps; ++st) {
            if (pp.op[st] == PROD_LEAF) {
                const int j = pp.arg[st];
                Fr lo, hi;
                load_factor<ORDER, SRC, BIND, HI4>(pp, j, y, pairs, s, dsm, lo, hi);
                Fr dl = fp_sub(hi, lo);
                if (WEIGHTED && st == 0) {  // the pair's weight goes into the first leaf only
                    lo = fp_mul(lo, wgt);
                    dl = fp_mul(dl, wgt);
                }
                prod_st(col, pp.base[st], lo);
                prod_st(col, pp.base[st] + 1, dl);
            } else {
                merge(col, pp, pp.base[st], pp.a[st], pp.b[st], pp.skip1 && st + 1 == pp.nsteps);
            }
        }
        if (pp.d == 1) prod_st(col, 1, fp_add(prod_ld(col, 0), prod_ld(col, 1)));  // s_y(1) = lo + D (no inf point)
        for (int e = 0; e < pp.npoints; ++e) {
            const int t = pp.point[e];
            prod_st(col, pp.acc + e, fp_add(prod_ld(col, pp.acc + e), prod_ld(col, t == PROD_INF ? pp.d : t)));
        }
    }
    product_epilogue(col, pp, dsm + pp.red, out);
}

// The program of d factors (binary-counter merges); returns the slots a thread's column needs.
int build_program(int d, ProductParams& pp) {
    struct Node {
        int base, deg, leaves;
    };
    Node stk[PROD_MAX];
    int n = 0, steps = 0, slots = 0;
    auto merge_top = [&] {
        const Node A = stk[n - 2], B = stk[n - 1];
        pp.op[steps] = PROD_MERGE;
        pp.base[steps] = (uint8_t)A.base;
        pp.a[steps] = (uint8_t)A.deg;
        pp.b[steps] = (uint8_t)B.deg;
        ++steps;
        slots = std::max(slots, A.base + 2 * (A.deg + B.deg) + 4);  // C, L_B, both tables
        n -= 2;
        stk[n++] = Node{A.base, A.deg + B.deg, A.leaves + B.leaves};
    };
    for (int j = 0; j < d; ++j) {
        const int base = n ? stk[n - 1].base + stk[n - 1].deg + 1 : 0;
        pp.op[steps] = PROD_LEAF;
        pp.arg[steps] = (uint8_t)j;
        pp.base[steps] = (uint8_t)base;
        ++steps;
        slots = std::max(slots, base + 2);
        stk[n++] = Node{base, 1, 1};
        while (n >= 2 && stk[n - 1].leaves == stk[n - 2].leaves) merge_top();
    }
    while (n >= 2) merge_top();
    pp.nsteps = steps;
    uint32_t f = 1;
    pp.fact[0] = 1;
    for (int k = 1; k <= PROD_MAX_CHILD; ++k) pp.fact[k] = f *= (uint32_t)k;
    return slots;
}

size_t column_bytes(int slots) { return (size_t)slots * 8 * PROD_BLOCK * 4; }
constexpr size_t RED_BYTES = ((size_t)(PROD_BLOCK / 32) * 8 + PROD_MAX_POINTS * 8) * 4;  // block_sum scratch, totals

template <int ORDER, bool SRC, bool BIND, bool HI4, bool WEIGHTED>
auto kernel_of() {
    auto kernel = product_round_kernel<ORDER, SRC, BIND, HI4, WEIGHTED>;
    static const bool attr = [&] {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PROD_SMEM_MAX);
        return true;
    }();
    (void)attr;
    return kernel;
}

template <class Kernel>
int blocks_per_sm(Kernel kernel, size_t smem) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, PROD_BLOCK, smem) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    return per_sm;
}

template <int ORDER, bool SRC, bool BIND, bool HI4, bool WEIGHTED>
int launch_product(jb_ctx* c, const jb_member* mem, ProductParams& pp, size_t words, size_t pairs, const BindScalar& s,
                   const RoundOut& out) {
    auto kernel = kernel_of<ORDER, SRC, BIND, HI4, WEIGHTED>();
    int per_sm;
    if (SRC) {
        // a one-hot source's eq table (K <= SRC_SMEM_K) is staged in shared memory while that keeps the blocks per SM
        // of the unstaged launch; beyond that cut the tables are read through L2 (they stay cached: <= 8 KiB each)
        per_sm = blocks_per_sm(kernel, words * 4 + RED_BYTES);
        for (int j = 0; j < pp.d; ++j) {
            const SourceCol& sc = mem->src[j];
            if (sc.type != JB_SOURCE_ONE_HOT || sc.K > SRC_SMEM_K) continue;
            const size_t more = words + (size_t)sc.K * 8;
            if (more * 4 + RED_BYTES > PROD_SMEM_MAX || blocks_per_sm(kernel, more * 4 + RED_BYTES) < per_sm) break;
            pp.smem[j] = (uint32_t)words;
            words = more;
        }
    } else {
        static std::atomic<int> per_sm_by_d[PROD_MAX + 1][2];  // occupancy depends on the column size: d, skip1
        per_sm = per_sm_by_d[pp.d][pp.skip1].load(std::memory_order_relaxed);
        if (per_sm == 0) {
            per_sm = blocks_per_sm(kernel, words * 4 + RED_BYTES);
            per_sm_by_d[pp.d][pp.skip1].store(per_sm, std::memory_order_relaxed);
        }
    }
    pp.red = (uint32_t)words;
    return launch_round(c, kernel, PROD_BLOCK, words * 4 + RED_BYTES, per_sm, pairs, PROD_MAX_POINTS, BIND ? 0 : 2, pp.d,
                        "product_round_kernel launch", out, pp, pairs, s);
}

template <int ORDER, bool WEIGHTED>
int dispatch_product2(jb_ctx* c, const jb_member* mem, ProductParams& pp, size_t words, size_t pairs, bool src, bool bind,
                      bool hi4, const BindScalar& s, const RoundOut& out) {
    if (src && !bind) return launch_product<ORDER, true, false, false, WEIGHTED>(c, mem, pp, words, pairs, s, out);
    if (src)
        return hi4 ? launch_product<ORDER, true, true, true, WEIGHTED>(c, mem, pp, words, pairs, s, out)
                   : launch_product<ORDER, true, true, false, WEIGHTED>(c, mem, pp, words, pairs, s, out);
    if (!bind) return c->fail(JB_ERR_INVALID, "product member: a round over field tables binds");  // (round 0 reads the sources)
    return hi4 ? launch_product<ORDER, false, true, true, WEIGHTED>(c, mem, pp, words, pairs, s, out)
               : launch_product<ORDER, false, true, false, WEIGHTED>(c, mem, pp, words, pairs, s, out);
}

// The source fields of the params (SRC_NO_SMEM everywhere: staging is the launch's decision).
void fill_sources(const jb_member* mem, ProductParams& pp) {
    for (int j = 0; j < mem->m; ++j) {
        pp.smem[j] = SRC_NO_SMEM;
        if (mem->src.empty()) continue;
        const SourceCol& sc = mem->src[j];
        pp.type[j] = (uint8_t)sc.type;
        pp.kind[j] = (uint8_t)sc.kind;
        pp.values[j] = sc.values;
        pp.eq[j] = sc.eq;
        pp.K[j] = sc.K;
    }
}

}  // namespace

int product_round(jb_ctx* c, const jb_member* mem, const uint64_t* const* in, uint64_t* const* out, const EqWeights* eqw,
                  bool skip1, size_t pairs, bool bind, bool hi4, const BindScalar& s, RoundOut ro) {
    ProductParams pp;
    std::memset(&pp, 0, sizeof pp);
    const int d = mem->m;
    pp.d = d;
    for (int j = 0; j < d; ++j) {
        pp.in[j] = in[j];
        pp.out[j] = out[j];
    }
    if (eqw) {
        pp.e_out = eqw->e_out;
        pp.e_in = eqw->e_in;
        pp.in_bits = eqw->in_bits;
    }
    fill_sources(mem, pp);
    // the round's points in kernel-value order: 0, [1 unless skip1], 2, .., d-1, inf (d >= 2); 0, [1] (d == 1)
    int n = 0;
    pp.point[n++] = 0;
    if (!skip1) pp.point[n++] = 1;
    for (int t = 2; t < d; ++t) pp.point[n++] = (int8_t)t;
    if (d >= 2) pp.point[n++] = PROD_INF;
    pp.npoints = n;
    pp.skip1 = skip1 ? 1 : 0;
    pp.acc = build_program(d, pp);
    const size_t words = column_bytes(pp.acc + n) / 4;
    const bool src = !mem->src.empty();
    if (mem->order == JB_LOW_TO_HIGH)
        return eqw ? dispatch_product2<ORDER_LOW_TO_HIGH, true>(c, mem, pp, words, pairs, src, bind, hi4, s, ro)
                   : dispatch_product2<ORDER_LOW_TO_HIGH, false>(c, mem, pp, words, pairs, src, bind, hi4, s, ro);
    return eqw ? dispatch_product2<ORDER_HIGH_TO_LOW, true>(c, mem, pp, words, pairs, src, bind, hi4, s, ro)
               : dispatch_product2<ORDER_HIGH_TO_LOW, false>(c, mem, pp, words, pairs, src, bind, hi4, s, ro);
}

int product_finish(jb_member* mem, const uint64_t r[4]) {
    ProductParams pp;
    std::memset(&pp, 0, sizeof pp);
    pp.d = mem->m;
    fill_sources(mem, pp);
    return finish_sources(mem, r, pp, pp);  // (pp's out pointers are the bind's destinations)
}
