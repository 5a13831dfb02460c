// The term descriptors of the batched-polynomial entry points (jb_table_linear_combination,
// jb_lc_vector_matrix_product): one device record per jb_lc_term, and the checks that build it, so both entry points
// read the same descriptor format and validate it the same way. Internal to the translation units that include it.
#pragma once
#include <cstring>
#include <vector>

#include "columns.cuh"
#include "member.hpp"

namespace {

using namespace jb;
using namespace jbi;

struct LcTerm {
    const void* ptr;  // TABLE: entries; COMPACT: values; ONE_HOT: addresses
    uint64_t len;     // entries of the term: a prefix of the output (ONE_HOT: K T)
    uint32_t c[8];    // TABLE / ONE_HOT: c~; COMPACT: (c R)~
    uint32_t nc[8];   // COMPACT: p - (c R)~, for negative values
    uint32_t type, kind, layout;
    uint32_t log_k, log_t, pad;
};
static_assert(sizeof(LcTerm) % 8 == 0, "LcTerm is staged as u64 words");

// The checks of one term that need no allocation; fills its descriptor except the column pointer of a host column.
int check_term(jb_ctx* c, const jb_lc_term& in, size_t len, LcTerm& t) {
    std::memset(&t, 0, sizeof t);
    if (!canonical_fr(in.coeff)) return c->fail(JB_ERR_INVALID, "linear_combination: coefficient limbs not canonical");
    t.type = (uint32_t)in.type;
    HostFr cf = HostFr::from_limbs(in.coeff);
    if (in.type == JB_LC_TABLE) {
        Table* tab = c->find(in.table);
        if (!tab) return c->fail(JB_ERR_INVALID, "unknown table handle");
        if (!pow2(tab->len)) return c->fail(JB_ERR_INVALID, "linear_combination: a table's length is not a power of two");
        t.ptr = tab->buf;
        t.len = tab->len;
    } else if (in.type == JB_LC_COMPACT) {
        const int st = check_compact_column(c, "linear_combination", in.kind, in.values, in.on_device);
        if (st != JB_OK) return st;
        if (!pow2(in.len)) return c->fail(JB_ERR_INVALID, "linear_combination: a compact length is not a power of two");
        t.kind = (uint32_t)in.kind;
        t.len = in.len;
        const HostFr r2{{HostFr::R2[0], HostFr::R2[1], HostFr::R2[2], HostFr::R2[3]}};
        cf = cf * r2;  // (c R)~: times a plain integer |v| it is c v R^2
        uint64_t neg[4];
        std::memcpy(neg, HostFr::P, 32);
        uint64_t borrow = 0;
        for (int k = 0; k < 4; ++k) {  // p - (c R)~ (= p for c = 0: still a multiple of p)
            const unsigned __int128 d = (unsigned __int128)neg[k] - cf.l[k] - borrow;
            neg[k] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
        for (int k = 0; k < 4; ++k) {
            t.nc[2 * k] = (uint32_t)neg[k];
            t.nc[2 * k + 1] = (uint32_t)(neg[k] >> 32);
        }
    } else if (in.type == JB_LC_ONE_HOT) {
        if (in.layout != JB_ONE_HOT_CYCLE_MAJOR && in.layout != JB_ONE_HOT_ADDRESS_MAJOR)
            return c->fail(JB_ERR_INVALID, "linear_combination: unknown one-hot layout");
        const int st = check_one_hot_columns(c, "linear_combination", in.kind, in.len, in.K, in.on_device, &in.values, 1);
        if (st != JB_OK) return st;
        t.kind = (uint32_t)in.kind;
        t.layout = (uint32_t)in.layout;
        t.log_k = log2_of(in.K);
        t.log_t = log2_of(in.len);
        t.len = in.K * in.len;
    } else {
        return c->fail(JB_ERR_INVALID, "linear_combination: unknown term type");
    }
    if (t.len > len) return c->fail(JB_ERR_INVALID, "linear_combination: a term is longer than the output");
    for (int k = 0; k < 4; ++k) {
        t.c[2 * k] = (uint32_t)cf.l[k];
        t.c[2 * k + 1] = (uint32_t)(cf.l[k] >> 32);
    }
    return JB_OK;
}

// Every term's checks, before anything is allocated (count and len are the caller's to check): desc[i] is term i's.
int check_terms(jb_ctx* c, const jb_lc_term* terms, size_t count, size_t len, std::vector<LcTerm>& desc) {
    desc.resize(count);
    for (size_t i = 0; i < count; ++i) {
        const int st = check_term(c, terms[i], len, desc[i]);
        if (st != JB_OK) return st;
    }
    return JB_OK;
}

// The column pointers of the checked descriptors: host columns are copied to the device for the call (owned by scratch).
int load_columns(Scratch& scratch, const jb_lc_term* terms, size_t count, std::vector<LcTerm>& desc) {
    int st = JB_OK;
    for (size_t i = 0; i < count && st == JB_OK; ++i) {
        const jb_lc_term& in = terms[i];
        if (in.type == JB_LC_TABLE) continue;
        const size_t bytes = in.len * (size_t)small_kind_bytes(in.kind);
        st = get_column(scratch, in.values, bytes, in.on_device, &desc[i].ptr);
    }
    return st;
}

}  // namespace
