// Witness columns in their own formats, decided once for every entry point that reads them:
//   * compact columns: primitive integers of a jb_scalar_kind other than JB_SCALAR_FR (small_scalar.cuh);
//   * one-hot address columns: u8, u16 or u32 addresses of T cycles into K addresses, the all-ones value of the width
//     meaning "no address" (the cycle touched none; for u32 that is NO_ADDRESS itself). K and T are powers of two,
//     T < 2^31, K <= 2^16 for u8 / u16 and K <= ONE_HOT_MAX_K_U32 = 2^24 for u32; an address >= K that is not the
//     none value is found on the device, raises the call's flag and fails the call. u32 columns are for address spaces
//     as large as RAM's (word addresses of a guest's memory), and only the entry points that pass SK_U32 as the widest
//     kind they accept take them: jb_one_hot_evaluate / jb_one_hot_pushforward, product members over one-hot sources
//     and read-write checking. The others (booleanity, commitments, linear combinations, the vector-matrix product,
//     expression members over sources) keep u8 / u16. 2^24 bounds the K-entry field tables those entry points build
//     (512 MiB each at 2^24); above it the eq gathers and the read-write address phase would have to be chunked.
// A column is in host memory (on_device = 0: copied to the device for the call, or for the owner that keeps it) or in
// device memory (on_device = 1: read in place, so it must be aligned to its entry, at most to 8 bytes).
#pragma once
#include <algorithm>
#include <string>

#include "ctx.hpp"
#include "small_scalar.cuh"

namespace jb {

constexpr uint32_t NO_ADDRESS = 0xffffffffu;
constexpr size_t ONE_HOT_MAX_K = (size_t)1 << 16;      // u8 / u16 address columns
constexpr size_t ONE_HOT_MAX_K_U32 = (size_t)1 << 24;  // u32 address columns

// The largest K a one-hot column of `kind` may address.
inline size_t one_hot_max_k(int kind) { return kind == SK_U32 ? ONE_HOT_MAX_K_U32 : ONE_HOT_MAX_K; }

// Address i of a one-hot column of `kind`, NO_ADDRESS for the none value. WIDEST is the widest kind the caller accepts
// (SK_U16: u8 / u16, SK_U32: u8 / u16 / u32); a caller that accepts u32 pays one more uniform branch, the others none.
template <int WIDEST = SK_U16>
__device__ __forceinline__ uint32_t ld_address(const void* col, size_t i, int kind) {
    static_assert(WIDEST == SK_U16 || WIDEST == SK_U32, "one-hot columns are u8, u16 or u32");
    if (WIDEST == SK_U32 && kind == SK_U32) return static_cast<const uint32_t*>(col)[i];  // none = NO_ADDRESS already
    const uint32_t a = kind == SK_U8 ? (uint32_t)static_cast<const uint8_t*>(col)[i] : (uint32_t)static_cast<const uint16_t*>(col)[i];
    return a == (kind == SK_U8 ? 0xffu : 0xffffu) ? NO_ADDRESS : a;
}

inline bool pow2(size_t x) { return x != 0 && (x & (x - 1)) == 0; }
inline int log2_of(size_t x) {
    int l = 0;
    while (x >> (l + 1)) ++l;
    return l;
}

inline bool compact_kind(int kind) { return kind >= SK_U8 && kind <= SK_LAST; }

inline int fail_column(jb_ctx* c, int status, const char* what, const char* why) {
    return c->fail(status, (std::string(what) + ": " + why).c_str());
}

// One compact column of `kind` (its length is the caller's to check).
inline int check_compact_column(jb_ctx* c, const char* what, int kind, const void* values, int on_device) {
    if (!compact_kind(kind)) return fail_column(c, JB_ERR_INVALID, what, "unknown scalar kind");
    if (!values) return fail_column(c, JB_ERR_INVALID, what, "null column");
    if (on_device != 0 && on_device != 1) return fail_column(c, JB_ERR_INVALID, what, "on_device must be 0 or 1");
    if (on_device && (uintptr_t)values % (size_t)std::min(8, small_kind_bytes(kind)))
        return fail_column(c, JB_ERR_INVALID, what, "misaligned device column");
    return JB_OK;
}

// Whether an entry point that accepts address kinds up to `widest` (SK_U16 or SK_U32) takes `kind`.
inline bool one_hot_kind(int kind, int widest) { return kind == SK_U8 || kind == SK_U16 || (widest == SK_U32 && kind == SK_U32); }

// `count` one-hot address columns of T cycles into K addresses (a layout, where there is one, is the caller's), for
// an entry point that accepts address kinds up to `widest`.
inline int check_one_hot_columns(jb_ctx* c, const char* what, int kind, size_t T, size_t K, int on_device,
                                 const void* const* columns, size_t count, int widest = SK_U16) {
    if (!one_hot_kind(kind, widest))
        return fail_column(c, JB_ERR_INVALID, what,
                           widest == SK_U32 ? "addresses must be JB_SCALAR_U8, JB_SCALAR_U16 or JB_SCALAR_U32"
                                            : "addresses must be JB_SCALAR_U8 or JB_SCALAR_U16");
    if (!pow2(T) || !pow2(K)) return fail_column(c, JB_ERR_INVALID, what, "K and T must be powers of two");
    if (on_device != 0 && on_device != 1) return fail_column(c, JB_ERR_INVALID, what, "on_device must be 0 or 1");
    if (T >= ((size_t)1 << 31)) return fail_column(c, JB_ERR_UNSUPPORTED, what, "T must be < 2^31");
    if (K > one_hot_max_k(kind))
        return fail_column(c, JB_ERR_UNSUPPORTED, what, kind == SK_U32 ? "K must be <= 2^24" : "K must be <= 2^16");
    if (count && !columns) return fail_column(c, JB_ERR_INVALID, what, "null pointer");
    for (size_t p = 0; p < count; ++p) {
        if (!columns[p]) return fail_column(c, JB_ERR_INVALID, what, "null column");
        if (on_device && (uintptr_t)columns[p] % (size_t)small_kind_bytes(kind))
            return fail_column(c, JB_ERR_INVALID, what, "misaligned device column");
    }
    return JB_OK;
}

// The failure of a call whose kernels raised the bad-address flag.
inline int fail_bad_address(jb_ctx* c) {
    return c->fail(JB_ERR_INVALID, "one-hot: an address >= K that is not the none value");
}

// A device copy of a column in host or device memory, owned by the caller (dev_free).
inline int copy_column(jb_ctx* c, const void* values, size_t bytes, int on_device, void** out) {
    int st = c->dev_alloc(out, bytes);
    if (st != JB_OK) return st;
    return c->check(cudaMemcpyAsync(*out, values, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                                    c->stream),
                    "column copy");
}

// A column a call reads in place: a host column is copied to device memory owned by the call's scratch, a device
// column is used as it is.
inline int get_column(Scratch& scratch, const void* src, size_t bytes, int on_device, const void** dst) {
    if (on_device) {
        *dst = src;
        return JB_OK;
    }
    void* d = nullptr;
    int st = scratch.alloc(bytes, &d);
    if (st == JB_OK)
        st = scratch.c->check(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, scratch.c->stream), "column copy");
    *dst = d;
    return st;
}

}  // namespace jb
