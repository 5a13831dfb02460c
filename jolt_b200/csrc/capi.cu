// C ABI of the H100 backend (see include/jolt_b200.h for the per-function reference citations).
// The context mirrors ProofSession (crates/jolt-kernels/src/backend.rs:283-286): it owns the
// stream, the stream-ordered device pool, and the small reduction / staging buffers.
// This unit: library / context, tables, bind, eq expansion, element-wise harness, diagnostics.
// Members and the round scheduler live in member.cu, the resident kernel service in resident.cu.
#include "../../include/jolt_b200.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "member.hpp"

using namespace jb;
using namespace jbi;
using Guard = CtxGuard;

namespace {

template <typename K>
int blocks_per_sm(K kernel) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, 256, 0) != cudaSuccess || nb < 1) nb = 1;
    return nb;
}

int grid_for(jb_ctx* c, size_t items, int per_sm) {
    size_t need = (items + 255) / 256;
    size_t cap = (size_t)c->sm_count * per_sm;
    size_t g = need < cap ? need : cap;
    return g < 1 ? 1 : (int)g;
}

template <int ORDER, bool HI4>
int launch_bind(jb_ctx* c, const uint64_t* in, uint64_t* out, size_t half, const BindScalar& s) {
    static int per_sm = blocks_per_sm(bind_kernel<ORDER, HI4>);
    int grid = grid_for(c, half, per_sm);
    int tix = c->timing_begin(1, half, 1);
    bind_kernel<ORDER, HI4><<<grid, 256, 0, c->stream>>>(in, out, half, s);
    c->timing_end(tix);
    c->launches++;
    return c->check(cudaGetLastError(), "bind_kernel launch");
}

}  // namespace

// Halves one table under `r` (Polynomial::bind_with_order).
int jbi::bind_table(jb_ctx* c, Table& t, const uint64_t r[4], int order) {
    if (t.len < 2 || (t.len & (t.len - 1))) return c->fail(JB_ERR_INVALID, "bind: table length must be a power of two >= 2");
    if (!canonical_fr(r)) return c->fail(JB_ERR_INVALID, "bind: challenge limbs not canonical (>= r)");
    bool hi4;
    BindScalar s = make_scalar(r, &hi4);
    size_t half = t.len / 2;
    int st;
    if (order == JB_HIGH_TO_LOW) {
        st = hi4 ? launch_bind<ORDER_HIGH_TO_LOW, true>(c, t.buf, t.buf, half, s)
                 : launch_bind<ORDER_HIGH_TO_LOW, false>(c, t.buf, t.buf, half, s);
    } else if (order == JB_LOW_TO_HIGH) {
        if ((st = c->ensure_alt(t, half)) != JB_OK) return st;
        st = hi4 ? launch_bind<ORDER_LOW_TO_HIGH, true>(c, t.buf, t.alt, half, s)
                 : launch_bind<ORDER_LOW_TO_HIGH, false>(c, t.buf, t.alt, half, s);
        if (st == JB_OK) t.swap_buffers();
    } else {
        return c->fail(JB_ERR_INVALID, "bind: unknown binding order");
    }
    if (st == JB_OK) t.len = half;
    return st;
}


namespace {
// eq table for `nvars` variables (HOST limbs r, optional host scale); recursive prefix for n > 11.
EqVars eq_vars(const uint64_t* r, size_t count, const uint64_t* scale) {
    EqVars v;
    std::memset(&v, 0, sizeof v);
    for (size_t j = 0; j < count; ++j)
        for (int w = 0; w < 4; ++w) {
            v.r[j][2 * w] = (uint32_t)r[4 * j + w];
            v.r[j][2 * w + 1] = (uint32_t)(r[4 * j + w] >> 32);
        }
    if (scale) {
        v.has_scale = 1;
        for (int w = 0; w < 4; ++w) {
            v.scale[2 * w] = (uint32_t)scale[w];
            v.scale[2 * w + 1] = (uint32_t)(scale[w] >> 32);
        }
    }
    return v;
}

}  // namespace

int jbi::eq_build(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, uint64_t* d_out) {
    if (nvars <= (size_t)EQ_BLOCK_VARS) {
        eq_expand_kernel<<<1, 256, 0, c->stream>>>(nullptr, eq_vars(r, nvars, scale), (int)nvars, d_out);
        c->launches++;
        return c->check(cudaGetLastError(), "eq_expand_kernel launch");
    }
    // n > 11: prefix table over the leading n-11 variables (recursively), the block-independent table
    // over the trailing 8, and one streaming pass that writes every output exactly once.
    size_t hi_vars = nvars - EQ_BLOCK_VARS;
    uint64_t *d_prefix = nullptr, *d_low8 = nullptr;
    int st = c->dev_alloc((void**)&d_prefix, ((size_t)1 << hi_vars) * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&d_low8, 256 * 32);
    if (st == JB_OK) st = eq_build(c, r, hi_vars, scale, d_prefix);
    // layout (JB_EQ_LAYOUT: 0 (default) = the 3 register variables FIRST in the block, a warp's store covers 1 KiB;
    // 1 = LAST: 8 consecutive outputs per thread; both write the same DRAM bytes whatever the store flavour)
    const bool low3 = c->eq_layout != 0;
    if (st == JB_OK) st = eq_build(c, r + 4 * (hi_vars + (low3 ? 0 : 3)), 8, nullptr, d_low8);
    if (st == JB_OK) {
        int tix = c->timing_begin(3, (uint64_t)1 << nvars, 1);
        const uint64_t* r3 = r + 4 * (hi_vars + (low3 ? 8 : 0));
        bool hi4 = true;  // all three register-stage variables are 125-bit challenges [0,0,lo,hi]
        for (int j = 0; j < 3; ++j) hi4 = hi4 && r3[4 * j] == 0 && r3[4 * j + 1] == 0;
        const unsigned g = (unsigned)((size_t)1 << hi_vars);
        // tables beyond what L2 can usefully keep are streamed out with evict-first stores (JB_EQ_STORE=0/1 forces)
        const bool cs = c->eq_store_mode < 0 ? nvars >= 22 : c->eq_store_mode == 1;
        const EqVars v3 = eq_vars(r3, 3, nullptr);
#define JB_EQ_LAUNCH(H, C, L) eq_stream_kernel<H, C, L><<<g, 256, 0, c->stream>>>(d_prefix, v3, d_low8, d_out)
        if (low3) {
            if (hi4 && cs) JB_EQ_LAUNCH(true, true, true);
            else if (hi4) JB_EQ_LAUNCH(true, false, true);
            else if (cs) JB_EQ_LAUNCH(false, true, true);
            else JB_EQ_LAUNCH(false, false, true);
        } else {
            if (hi4 && cs) JB_EQ_LAUNCH(true, true, false);
            else if (hi4) JB_EQ_LAUNCH(true, false, false);
            else if (cs) JB_EQ_LAUNCH(false, true, false);
            else JB_EQ_LAUNCH(false, false, false);
        }
#undef JB_EQ_LAUNCH
        c->timing_end(tix);
        c->launches++;
        st = c->check(cudaGetLastError(), "eq_stream_kernel launch");
    }
    if (d_prefix) c->dev_free(d_prefix);
    if (d_low8) c->dev_free(d_low8);
    return st;
}

// ------------------------------------------------------------------------------------------
extern "C" {

const char* jb_version(void) { return "jolt_b200 0.1 (sm_90a)"; }

const char* jb_status_str(int status) {
    switch (status) {
        case JB_OK: return "ok";
        case JB_ERR_NO_DEVICE: return "no CUDA device (this backend has no CPU fallback)";
        case JB_ERR_CUDA: return "CUDA error";
        case JB_ERR_INVALID: return "invariant violation";
        case JB_ERR_OOM: return "device out of memory";
        case JB_ERR_ROUND_CHECK: return "sumcheck round check failed: s(0)+s(1) != previous_claim";
        case JB_ERR_UNSUPPORTED: return "unsupported";
        case JB_ERR_LENGTH: return "msm: bases/scalars length mismatch";
        default: return "unknown status";
    }
}

int jb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

static int ctx_create_impl(int device, bool borrow, void* cuda_stream, jb_ctx** out) {
    if (!out) return JB_ERR_INVALID;
    *out = nullptr;
    int n = jb_device_count();
    if (n <= 0) return JB_ERR_NO_DEVICE;
    if (device < 0 || device >= n) return JB_ERR_INVALID;
    jb_ctx* c = new (std::nothrow) jb_ctx();
    if (!c) return JB_ERR_OOM;
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete c; return JB_ERR_CUDA; }
    if (borrow) {  // a null handle is the legacy default stream
        c->stream = (cudaStream_t)cuda_stream;
        c->owns_stream = false;
    } else {
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return JB_ERR_CUDA; }
        c->owns_stream = true;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    c->sm_count = prop.multiProcessorCount;
    if (const char* sh = std::getenv("JB_FUSED_SHAPE")) c->fused_shape = std::atoi(sh);  // tuning knob
    if (std::getenv("JB_NO_TAIL")) c->use_tail = false;  // diagnostics: one launch per round all the way down
    if (const char* ml = std::getenv("JB_RESIDENT_MAX_LOG")) c->resident_max_log = std::atoi(ml);
    if (const char* sp = std::getenv("JB_STATIC_PCT")) c->resident_static_pct = std::max(0, std::min(100, std::atoi(sp)));
    if (const char* ts = std::getenv("JB_RESIDENT_TIMEOUT_S")) c->resident_timeout_cycles = (long long)(std::atof(ts) * 1.9e9);
    if (const char* rs = std::getenv("JB_RES_STAGED")) c->res_staged = std::atoi(rs) != 0;
    if (std::getenv("JB_EVAL_TMA")) c->eval_tma = true;
    if (std::getenv("JB_NO_LOOKAHEAD")) c->lookahead = false;
    if (const char* es = std::getenv("JB_EQ_STORE")) c->eq_store_mode = std::atoi(es);
    if (const char* el = std::getenv("JB_EQ_LAYOUT")) c->eq_layout = std::atoi(el);  // diagnostics: every round waits for its own answer
    // A kernel-replaying profiler (ncu) or a serialising tool (compute-sanitizer, nsys CUDA trace) cannot
    // run a kernel that waits for host commands; under CUDA injection keep one launch per round.
    {
        extern char** environ;
        for (char** e = environ; e && *e; ++e) {
            if (!std::strncmp(*e, "CUDA_INJECTION64_PATH=", 22) || !std::strncmp(*e, "NV_NSIGHT_INJECTION", 19) ||
                !std::strncmp(*e, "NV_COMPUTE_PROFILER", 19) || !std::strncmp(*e, "NSYS_PROFILING_SESSION_ID=", 26))
                c->use_tail = false;
        }
    }
    if (std::getenv("JB_FORCE_RESIDENT")) c->use_tail = true;  // debugging: keep the resident kernel under a tool
    // keep freed blocks in the pool (ProofSession "device memory pools")
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thresh = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);
    }
    bool ok = cudaMalloc((void**)&c->d_small, JB_SMALL_BYTES) == cudaSuccess &&
              cudaMallocHost((void**)&c->h_small, JB_SMALL_BYTES) == cudaSuccess &&
              cudaHostAlloc((void**)&c->h_result, 1024 * JB_RESULT_SLOTS, cudaHostAllocMapped) == cudaSuccess &&
              cudaHostGetDevicePointer((void**)&c->d_result_alias, c->h_result, 0) == cudaSuccess &&
              cudaMalloc((void**)&c->d_counter, 64) == cudaSuccess && cudaMemset(c->d_counter, 0, 64) == cudaSuccess;
    if (ok) std::memset(c->h_result, 0, 1024 * JB_RESULT_SLOTS);
    if (!ok) {
        jb_ctx_destroy(c);
        return JB_ERR_OOM;
    }
    *out = c;
    return JB_OK;
}

int jb_ctx_create(int device, jb_ctx** out) { return ctx_create_impl(device, false, nullptr, out); }

int jb_ctx_create_on_stream(int device, void* cuda_stream, jb_ctx** out) {
    return ctx_create_impl(device, true, cuda_stream, out);
}

void jb_ctx_destroy(jb_ctx* c) {
    if (!c) return;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        cudaSetDevice(c->device);
        c->quiesce_resident(true);
    }
    jb_comm_destroy(c);
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    for (auto& kv : c->tables) c->release(kv.second);
    c->tables.clear();
    for (auto& r : c->tail_pool) {
        if (r.stream) { cudaStreamSynchronize(r.stream); cudaStreamDestroy(r.stream); }
        if (r.event) cudaEventDestroy(r.event);
        if (r.mb_host) cudaFreeHost(r.mb_host);
        if (r.d_state) cudaFree(r.d_state);
    }
    c->tail_pool.clear();
    for (auto& kv : c->srs) {
        if (kv.second.xy) cudaFreeAsync(kv.second.xy, c->stream);
        if (kv.second.pre) cudaFreeAsync(kv.second.pre, c->stream);
        if (kv.second.pre_small) cudaFreeAsync(kv.second.pre_small, c->stream);
    }
    c->srs.clear();
    c->msm_release();
    if (c->d_partial) cudaFreeAsync(c->d_partial, c->stream);
    if (c->d_small) cudaFree(c->d_small);
    if (c->h_small) cudaFreeHost(c->h_small);
    if (c->h_result) cudaFreeHost(c->h_result);
    if (c->d_lanes) cudaFree(c->d_lanes);
    if (c->d_counter) cudaFree(c->d_counter);
    if (c->owns_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

const char* jb_last_error(jb_ctx* c) { return c ? c->err.c_str() : "null context"; }

int jb_ctx_synchronize(jb_ctx* c) {
    if (!c) return JB_ERR_INVALID;
    Guard g(c);
    return c->check(cudaStreamSynchronize(c->stream), "stream synchronize");
}

uint64_t jb_ctx_launch_count(jb_ctx* c) { return c ? c->launches : 0; }

int jb_ctx_diag(jb_ctx* c, double out[4]) {
    if (!c || !out) return JB_ERR_INVALID;
    out[0] = (double)c->diag_wait_ns;
    out[1] = (double)c->diag_waits;
    out[2] = out[3] = 0;
    c->diag_wait_ns = 0;
    c->diag_waits = 0;
    return JB_OK;
}

int jb_ctx_run_log(jb_ctx* c, uint64_t* out, size_t cap_rounds, size_t* rounds) {
    if (!c || !out || !rounds) return JB_ERR_INVALID;
    Guard g(c, true);
    const size_t n = c->last_run_rounds < cap_rounds ? c->last_run_rounds : cap_rounds;
    std::memcpy(out, c->last_run_log, n * 64);
    *rounds = n;
    return JB_OK;
}

int jb_ctx_timing_enable(jb_ctx* c, int on, uint64_t min_items) {
    if (!c) return JB_ERR_INVALID;
    Guard g(c);
    c->timing = on != 0;
    c->timing_min_items = min_items;
    return JB_OK;
}

int jb_ctx_timing_collect(jb_ctx* c, int* kinds, uint64_t* items, int* ms_m, double* ms, size_t cap, size_t* count) {
    if (!c || !count) return JB_ERR_INVALID;
    Guard g(c);
    int st = c->check(cudaStreamSynchronize(c->stream), "timing sync");
    if (st != JB_OK) return st;
    size_t n = 0;
    for (auto& t : c->timed) {
        float f = (float)t.ms_direct;
        if (t.e0) cudaEventElapsedTime(&f, t.e0, t.e1);
        if (n < cap) {
            if (kinds) kinds[n] = t.kind;
            if (items) items[n] = t.items;
            if (ms_m) ms_m[n] = t.m;
            if (ms) ms[n] = f;
            ++n;
        }
        if (t.e0) {
            cudaEventDestroy(t.e0);
            cudaEventDestroy(t.e1);
        }
    }
    c->timed.clear();
    *count = n;
    return JB_OK;
}

// ---- tables ------------------------------------------------------------------------------
int jb_table_alloc(jb_ctx* c, size_t len, jb_table* out) {
    if (!c || !out || len == 0) return JB_ERR_INVALID;
    Guard g(c);
    Table t;
    int st = c->dev_alloc((void**)&t.buf, len * 32);
    if (st != JB_OK) return st;
    t.cap = t.len = len;
    t.buf_owned = true;
    *out = c->next_id++;
    c->tables[*out] = t;
    return JB_OK;
}

int jb_table_upload(jb_ctx* c, const uint64_t* limbs, size_t len, jb_table* out) {
    if (!c || !limbs) return JB_ERR_INVALID;
    int st = jb_table_alloc(c, len, out);
    if (st != JB_OK) return st;
    Guard g(c);
    Table& t = c->tables[*out];
    st = c->check(cudaMemcpyAsync(t.buf, limbs, len * 32, cudaMemcpyHostToDevice, c->stream), "table upload");
    // the host buffer is borrowed for the duration of the call only: with pinned / registered memory the copy is
    // truly asynchronous, so wait for it (pageable memory is staged before cudaMemcpyAsync returns anyway)
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "table upload sync");
    return st;
}

int jb_table_wrap_device(jb_ctx* c, void* dptr, size_t len, jb_table* out) {
    if (!c || !dptr || !out || len == 0 || ((uintptr_t)dptr & 31)) return JB_ERR_INVALID;
    Guard g(c);
    Table t;
    t.buf = (uint64_t*)dptr;
    t.cap = t.len = len;
    t.buf_owned = false;
    *out = c->next_id++;
    c->tables[*out] = t;
    return JB_OK;
}

int jb_table_len(jb_ctx* c, jb_table h, size_t* len) {
    if (!c || !len) return JB_ERR_INVALID;
    Guard g(c);
    Table* t = c->find(h);
    if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
    *len = t->len;
    return JB_OK;
}

int jb_table_device_ptr(jb_ctx* c, jb_table h, void** p) {
    if (!c || !p) return JB_ERR_INVALID;
    Guard g(c);
    Table* t = c->find(h);
    if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
    *p = t->buf;
    return JB_OK;
}

int jb_table_download(jb_ctx* c, jb_table h, uint64_t* out, size_t len) {
    if (!c || !out) return JB_ERR_INVALID;
    Guard g(c);
    Table* t = c->find(h);
    if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
    if (len > t->len) return c->fail(JB_ERR_INVALID, "download: len exceeds table length");
    int st = c->check(cudaMemcpyAsync(out, t->buf, len * 32, cudaMemcpyDeviceToHost, c->stream), "table download");
    if (st != JB_OK) return st;
    return c->check(cudaStreamSynchronize(c->stream), "table download sync");
}

int jb_table_clone(jb_ctx* c, jb_table h, jb_table* out) {
    if (!c || !out) return JB_ERR_INVALID;
    size_t len;
    {
        Guard g(c);
        Table* t = c->find(h);
        if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
        len = t->len;
    }
    int st = jb_table_alloc(c, len, out);
    if (st != JB_OK) return st;
    Guard g(c);
    return c->check(cudaMemcpyAsync(c->tables[*out].buf, c->tables[h].buf, len * 32, cudaMemcpyDeviceToDevice, c->stream),
                    "table clone");
}

int jb_table_free(jb_ctx* c, jb_table h) {
    if (!c) return JB_ERR_INVALID;
    Guard g(c);
    auto it = c->tables.find(h);
    if (it == c->tables.end()) return c->fail(JB_ERR_INVALID, "unknown table handle");
    c->release(it->second);
    c->tables.erase(it);
    return JB_OK;
}

int jb_table_bind(jb_ctx* c, jb_table h, const uint64_t r[4], int order) {
    if (!c || !r) return JB_ERR_INVALID;
    Guard g(c);
    Table* t = c->find(h);
    if (!t) return c->fail(JB_ERR_INVALID, "unknown table handle");
    return bind_table(c, *t, r, order);
}

// ---- eq ----------------------------------------------------------------------------------
int jb_eq_evals(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, jb_table* out) {
    if (!c || !out || (nvars && !r) || nvars > 40) return JB_ERR_INVALID;
    for (size_t i = 0; i < nvars; ++i)
        if (!canonical_fr(r + 4 * i)) return c->fail(JB_ERR_INVALID, "eq: point limbs not canonical");
    if (scale && !canonical_fr(scale)) return c->fail(JB_ERR_INVALID, "eq: scale limbs not canonical");
    int st = jb_table_alloc(c, (size_t)1 << nvars, out);
    if (st != JB_OK) return st;
    Guard g(c);
    return eq_build(c, r, nvars, scale, c->tables[*out].buf);
}

int jb_eq_evals_aligned_block(jb_ctx* c, const uint64_t* r, size_t nvars, size_t start_index, size_t block_size,
                              jb_table* out) {
    if (!c || !out || !r) return JB_ERR_INVALID;
    if (block_size == 0 || (block_size & (block_size - 1)) || start_index % block_size)
        return c->fail(JB_ERR_INVALID, "eq aligned block: block_size must be a power of two dividing start_index");
    size_t block_vars = 0;
    while (((size_t)1 << block_vars) < block_size) ++block_vars;
    if (block_vars > nvars) return c->fail(JB_ERR_INVALID, "eq aligned block: block larger than the domain");
    size_t prefix_len = nvars - block_vars;
    size_t prefix_value = start_index >> block_vars;
    // prefix scale = prod_i (bit ? r_i : 1 - r_i): O(log G) host multiplications (eq.rs:252-260)
    HostFr scale = HostFr::one();
    for (size_t i = 0; i < prefix_len; ++i) {
        if (!canonical_fr(r + 4 * i)) return c->fail(JB_ERR_INVALID, "eq: point limbs not canonical");
        HostFr ri = HostFr::from_limbs(r + 4 * i);
        bool bit = (prefix_value >> (prefix_len - 1 - i)) & 1;
        scale = scale * (bit ? ri : HostFr::one() - ri);
    }
    return jb_eq_evals(c, r + 4 * prefix_len, block_vars, scale.l, out);
}


// ---- element-wise parity harness ---------------------------------------------------------------
int jb_vec_op(jb_ctx* c, int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
    if (!c || !a || !b || !out || op < 0 || op > 5 || (field != 0 && field != 1)) return JB_ERR_INVALID;
    if (n == 0) return JB_OK;
    Guard g(c);
    uint64_t *da = nullptr, *db = nullptr, *dd = nullptr;
    int st = c->dev_alloc((void**)&da, n * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&db, n * 32);
    if (st == JB_OK) st = c->dev_alloc((void**)&dd, n * 32);
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(da, a, n * 32, cudaMemcpyHostToDevice, c->stream), "vec H2D");
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(db, b, n * 32, cudaMemcpyHostToDevice, c->stream), "vec H2D");
    if (st == JB_OK) {
        unsigned grid = (unsigned)((n + 255) / 256);
        if (field == 0) vec_op_kernel<Fr><<<grid, 256, 0, c->stream>>>(da, db, dd, n, op);
        else vec_op_kernel<Fq><<<grid, 256, 0, c->stream>>>(da, db, dd, n, op);
        c->launches++;
        st = c->check(cudaGetLastError(), "vec_op launch");
    }
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(out, dd, n * 32, cudaMemcpyDeviceToHost, c->stream), "vec D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "vec sync");
    if (da) c->dev_free(da);
    if (db) c->dev_free(db);
    if (dd) c->dev_free(dd);
    return st;
}

}  // extern "C"

// ---- diagnostics: ALU ceiling of the Montgomery product (DESIGN.md roofline evidence) ------------
namespace {
template <class F, int VARIANT>
__global__ void __launch_bounds__(256) mul_chain_kernel(uint64_t* io, int iters) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    F x0 = ld_elem_rw<F>(io, 4 * i), x1 = ld_elem_rw<F>(io, 4 * i + 1);
    F b0 = ld_elem_rw<F>(io, 4 * i + 2), b1 = ld_elem_rw<F>(io, 4 * i + 3);
    for (int k = 0; k < iters; ++k) {
        if (VARIANT == 0) {  // full 8x8 product + reduction
            x0 = fp_mul(x0, b0);
            x1 = fp_mul(x1, b1);
        } else if (VARIANT == 1) {  // 125-bit challenge multiplier (4 rows)
            x0 = fp_mul_hi4(x0, b0.v + 4);
            x1 = fp_mul_hi4(x1, b1.v + 4);
        } else {  // add/sub only
            x0 = fp_add(x0, b0);
            x1 = fp_sub(x1, b1);
        }
    }
    st_elem(io, 4 * i, x0);
    st_elem(io, 4 * i + 1, x1);
}
}  // namespace

extern "C" int jb_diag_mul_throughput(jb_ctx* c, int field, int variant, int iters, int blocks, double* out_gops) {
    if (!c || !out_gops || iters < 1 || blocks < 1 || variant < 0 || variant > 2) return JB_ERR_INVALID;
    Guard g(c);
    size_t threads = (size_t)blocks * 256;
    uint64_t* d = nullptr;
    int st = c->dev_alloc((void**)&d, threads * 4 * 32);
    if (st != JB_OK) return st;
    std::vector<uint64_t> h(threads * 16);
    uint64_t sm = 0x1234;
    for (auto& v : h) { sm += 0x9E3779B97F4A7C15ULL; uint64_t z = sm; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; v = z ^ (z >> 31); }
    for (size_t i = 0; i < threads * 4; ++i) h[4 * i + 3] &= 0x0fffffffffffffffULL;  // < p
    st = c->check(cudaMemcpyAsync(d, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c->stream), "diag H2D");
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 5 && st == JB_OK; ++rep) {
        cudaEventRecord(e0, c->stream);
#define JB_DIAG_LAUNCH(F, V) mul_chain_kernel<F, V><<<blocks, 256, 0, c->stream>>>(d, iters)
        if (field == 0) { if (variant == 0) JB_DIAG_LAUNCH(Fr, 0); else if (variant == 1) JB_DIAG_LAUNCH(Fr, 1); else JB_DIAG_LAUNCH(Fr, 2); }
        else { if (variant == 0) JB_DIAG_LAUNCH(Fq, 0); else if (variant == 1) JB_DIAG_LAUNCH(Fq, 1); else JB_DIAG_LAUNCH(Fq, 2); }
#undef JB_DIAG_LAUNCH
        c->launches++;
        cudaEventRecord(e1, c->stream);
        st = c->check(cudaEventSynchronize(e1), "diag sync");
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 0 && ms < best) best = ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    c->dev_free(d);
    if (st == JB_OK) *out_gops = (double)threads * 2.0 * iters / (best * 1e-3) / 1e9;
    return st;
}
