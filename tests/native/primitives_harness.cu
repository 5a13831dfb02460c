// Device harness for the arithmetic primitives every kernel is built from: the BN254 Montgomery field
// (field.cuh), the 544-bit deferred-reduction accumulators and reduce_wide17 (field.cuh), the lane bins
// (lane_bins.cuh) and the XYZZ group law with fq_inverse (ec.cuh). The headers are included as the library
// compiles them; tests/test_gpu_primitives.py builds this file with the library's nvcc flags and compares every
// output word with Python big integers.
//
// Each entry point copies host arrays in, launches one grid-stride kernel, copies the result back and
// synchronises; it returns the cudaError_t rather than aborting. Field elements are 4 x u64 (= 8 x u32) raw
// limbs, as in the library's tables; `fld` selects Fr (0) or Fq (1).
#include <cstddef>
#include <cstdint>
#include <type_traits>

#include "field.cuh"
#include "ec.cuh"
#include "lane_bins.cuh"

using namespace jb;

namespace {

constexpr int BLOCK = 256;

unsigned grid_for(size_t n) {
    const size_t g = (n + BLOCK - 1) / BLOCK;
    return (unsigned)(g < 1 ? 1 : g > 512 ? 512 : g);  // capped, so large inputs take several grid strides
}

enum FieldOp : int {
    OP_ADD, OP_SUB, OP_MUL, OP_SQR, OP_NEG, OP_DBL, OP_FROM_MONT, OP_TO_MONT, OP_EQ,
    OP_SUB_LAZY, OP_MUL_LAZY, OP_MUL_HI4_LAZY, OP_MUL_HI4, OP_INVERSE, OP_COUNT
};

// out[i] = op(a[i], b[i]). OP_EQ writes (a == b, a.is_zero()) into words 0 and 1; the hi4 products take words
// 4..7 of b as the multiplier, as the bind kernels do; OP_INVERSE is Fq only.
template <class PR>
__global__ void __launch_bounds__(BLOCK) field_op_kernel(int op, const uint64_t* a, const uint64_t* b, uint64_t* out,
                                                         size_t n) {
    using F = Fp<PR>;
    for (size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * BLOCK) {
        const F x = ld_elem_rw<F>(a, i), y = ld_elem_rw<F>(b, i);
        F r = F::zero();
        switch (op) {
            case OP_ADD: r = fp_add(x, y); break;
            case OP_SUB: r = fp_sub(x, y); break;
            case OP_MUL: r = fp_mul(x, y); break;
            case OP_SQR: r = fp_sqr(x); break;
            case OP_NEG: r = fp_neg(x); break;
            case OP_DBL: r = fp_dbl(x); break;
            case OP_FROM_MONT: r = fp_from_mont(x); break;
            case OP_TO_MONT: r = fp_to_mont(x); break;
            case OP_EQ:
                r.v[0] = x == y;
                r.v[1] = x.is_zero();
                break;
            case OP_SUB_LAZY: r = fp_sub_lazy(x, y); break;
            case OP_MUL_LAZY: r = fp_mul_lazy(x, y); break;
            case OP_MUL_HI4_LAZY: r = fp_mul_hi4_lazy(x, y.v + 4); break;
            case OP_MUL_HI4: r = fp_mul_hi4(x, y.v + 4); break;
            case OP_INVERSE:
                if constexpr (std::is_same<PR, FqParams>::value) r = fq_inverse(x);
                break;
        }
        st_elem(out, i, r);
    }
}

// Wide-accumulator forms, selected by `mode`.
enum WideMode : int { W_REG, W_SMEM, W_BW1, W_BW2, W_BW4, W_BW8, W_COUNT };

// Thread i: A = seed[i] (17 words), then reps times over its `count` products A += a[i, j] * b[i, j]; out[i] = A.
// The shared-memory form keeps A at sacc[k * blockDim.x + threadIdx.x], a stride of blockDim.x words.
__global__ void __launch_bounds__(BLOCK) wide_acc_kernel(int mode, const uint32_t* seed, const uint32_t* a,
                                                         const uint32_t* b, int count, int reps, uint32_t* out,
                                                         size_t n) {
    extern __shared__ uint32_t sacc[];
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t A[17];
        uint32_t* col = sacc + threadIdx.x;
#pragma unroll
        for (int k = 0; k < 17; ++k) {
            A[k] = seed[i * 17 + k];
            if (mode == W_SMEM) col[k * blockDim.x] = A[k];
        }
        for (int r = 0; r < reps; ++r) {
            for (int j = 0; j < count; ++j) {
                const uint32_t* x = a + (i * count + j) * 8;
                const uint32_t* y = b + (i * count + j) * 8;
                switch (mode) {
                    case W_REG: mul_wide_acc_reg(A, x, y); break;
                    case W_SMEM: mul_wide_acc_smem(col, (int)blockDim.x, x, y); break;
                    case W_BW1: mul_wide_acc_bw<1>(A, x, y); break;
                    case W_BW2: mul_wide_acc_bw<2>(A, x, y); break;
                    case W_BW4: mul_wide_acc_bw<4>(A, x, y); break;
                    case W_BW8: mul_wide_acc_bw<8>(A, x, y); break;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 17; ++k) out[i * 17 + k] = mode == W_SMEM ? col[k * blockDim.x] : A[k];
    }
}

// out[i] = reduce_wide17(acc + i, stride n): value i's 17 words are acc[k * n + i].
template <class PR>
__global__ void __launch_bounds__(BLOCK) reduce_kernel(const uint32_t* acc, uint64_t* out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * BLOCK)
        st_elem(out, i, reduce_wide17<PR>(acc + i, (int)n));
}

// Thread i calls pf_flush(emit[i], key[i], val[i]). n is a multiple of 32 and so is the grid stride, so every
// warp runs the loop with all 32 lanes, as pf_flush's warp collectives require.
__global__ void __launch_bounds__(BLOCK) flush_kernel(const uint32_t* emit, const uint32_t* key, const uint64_t* val,
                                                      size_t n, unsigned long long* bins) {
    for (size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * BLOCK)
        pf_flush(emit[i] != 0, key[i], ld_elem_rw<Fr>(val, i), bins, (int)(threadIdx.x & 31));
}

enum G1Op : int { G_ADD_AFFINE, G_ADD, G_DOUBLE, G_COUNT };

// a[i], b[i], out[i] are XYZZ points (X, Y, ZZ, ZZZ; Fq Montgomery). G_ADD_AFFINE adds the affine point
// (b.X, b.Y), negated when neg[i] != 0; G_ADD adds b; G_DOUBLE doubles a.
__global__ void __launch_bounds__(BLOCK) g1_kernel(int op, const uint64_t* a, const uint64_t* b, const uint32_t* neg,
                                                   uint64_t* out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * BLOCK) {
        XYZZ acc = ld_xyzz(a, i);
        const XYZZ o = ld_xyzz(b, i);
        switch (op) {
            case G_ADD_AFFINE: xyzz_add_affine(acc, o.x, o.y, neg[i] != 0); break;
            case G_ADD: xyzz_add(acc, o); break;
            case G_DOUBLE: xyzz_double(acc); break;
        }
        st_xyzz(out, i, acc);
    }
}

#define TRY(x)                                     \
    do {                                           \
        const cudaError_t e_ = (x);                \
        if (e_ != cudaSuccess) return (int)e_;     \
    } while (0)

// Device buffer, freed on every return path.
struct Buf {
    void* p = nullptr;
    ~Buf() {
        if (p) cudaFree(p);
    }
    // allocate `bytes`; copy from `host`, or zero-fill when host is null
    cudaError_t init(const void* host, size_t bytes) {
        cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
        if (e != cudaSuccess) return e;
        return host ? cudaMemcpy(p, host, bytes, cudaMemcpyHostToDevice) : cudaMemset(p, 0, bytes);
    }
    template <class T>
    T* as() const {
        return (T*)p;
    }
};

int finish(void* host_out, const Buf& d, size_t bytes) {
    TRY(cudaGetLastError());
    TRY(cudaMemcpy(host_out, d.p, bytes, cudaMemcpyDeviceToHost));
    TRY(cudaDeviceSynchronize());
    return 0;
}

}  // namespace

extern "C" {

int ph_field_op(int fld, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
    if ((fld != 0 && fld != 1) || op < 0 || op >= OP_COUNT || (op == OP_INVERSE && fld != 1))
        return (int)cudaErrorInvalidValue;
    Buf da, db, dout;
    TRY(da.init(a, n * 32));
    TRY(db.init(b, n * 32));
    TRY(dout.init(nullptr, n * 32));
    if (fld == 0)
        field_op_kernel<FrParams><<<grid_for(n), BLOCK>>>(op, da.as<uint64_t>(), db.as<uint64_t>(), dout.as<uint64_t>(), n);
    else
        field_op_kernel<FqParams><<<grid_for(n), BLOCK>>>(op, da.as<uint64_t>(), db.as<uint64_t>(), dout.as<uint64_t>(), n);
    return finish(out, dout, n * 32);
}

// seed, out: n x 17 u32 words; a, b: n x count elements of 8 u32 words.
int ph_wide_acc(int mode, const uint32_t* seed, const uint32_t* a, const uint32_t* b, int count, int reps,
                uint32_t* out, size_t n) {
    if (mode < 0 || mode >= W_COUNT || count < 0 || reps < 0) return (int)cudaErrorInvalidValue;
    const int block = 64;  // the shared-memory form's stride
    Buf dseed, da, db, dout;
    TRY(dseed.init(seed, n * 17 * 4));
    TRY(da.init(a, n * count * 32));
    TRY(db.init(b, n * count * 32));
    TRY(dout.init(nullptr, n * 17 * 4));
    wide_acc_kernel<<<(unsigned)((n + block - 1) / block), block, 17 * block * 4>>>(
        mode, dseed.as<uint32_t>(), da.as<uint32_t>(), db.as<uint32_t>(), count, reps, dout.as<uint32_t>(), n);
    return finish(out, dout, n * 17 * 4);
}

// acc: 17 x n u32 words (word k of value i at k * n + i).
int ph_reduce_wide17(int fld, const uint32_t* acc, uint64_t* out, size_t n) {
    if (fld != 0 && fld != 1) return (int)cudaErrorInvalidValue;
    Buf dacc, dout;
    TRY(dacc.init(acc, n * 17 * 4));
    TRY(dout.init(nullptr, n * 32));
    if (fld == 0) reduce_kernel<FrParams><<<grid_for(n), BLOCK>>>(dacc.as<uint32_t>(), dout.as<uint64_t>(), n);
    else reduce_kernel<FqParams><<<grid_for(n), BLOCK>>>(dacc.as<uint32_t>(), dout.as<uint64_t>(), n);
    return finish(out, dout, n * 32);
}

// lanes: n bins of 8 u64 lanes -> n Fr elements, through the header's own kernel.
int ph_bins_to_fr(const uint64_t* lanes, uint64_t* out, size_t n) {
    Buf dl, dout;
    TRY(dl.init(lanes, n * 64));
    TRY(dout.init(nullptr, n * 32));
    const size_t g = (n + BINS_BLOCK - 1) / BINS_BLOCK;
    bins_to_fr_kernel<<<(unsigned)(g < 1 ? 1 : g > 512 ? 512 : g), BINS_BLOCK>>>(
        dl.as<unsigned long long>(), n, dout.as<uint64_t>());
    return finish(out, dout, n * 32);
}

// n (a multiple of 32) lanes flush into nbins zeroed bins of 8 u64 lanes; bins receives them.
int ph_pf_flush(const uint32_t* emit, const uint32_t* key, const uint64_t* val, size_t n, uint64_t* bins,
                size_t nbins) {
    if (n % 32) return (int)cudaErrorInvalidValue;
    Buf de, dk, dv, db;
    TRY(de.init(emit, n * 4));
    TRY(dk.init(key, n * 4));
    TRY(dv.init(val, n * 32));
    TRY(db.init(nullptr, nbins * 64));
    flush_kernel<<<grid_for(n), BLOCK>>>(de.as<uint32_t>(), dk.as<uint32_t>(), dv.as<uint64_t>(), n,
                                         db.as<unsigned long long>());
    return finish(bins, db, nbins * 64);
}

// a, b, out: n XYZZ points of 4 Fq elements; neg: n flags (G_ADD_AFFINE only).
int ph_g1(int op, const uint64_t* a, const uint64_t* b, const uint32_t* neg, uint64_t* out, size_t n) {
    if (op < 0 || op >= G_COUNT) return (int)cudaErrorInvalidValue;
    Buf da, db, dn, dout;
    TRY(da.init(a, n * 128));
    TRY(db.init(b, n * 128));
    TRY(dn.init(neg, n * 4));
    TRY(dout.init(nullptr, n * 128));
    g1_kernel<<<grid_for(n), BLOCK>>>(op, da.as<uint64_t>(), db.as<uint64_t>(), dn.as<uint32_t>(),
                                      dout.as<uint64_t>(), n);
    return finish(out, dout, n * 128);
}

}  // extern "C"
