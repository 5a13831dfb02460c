// Read-write checking member (jb_member_create_read_write): the cycle phase over the sparse K x T memory matrix.
//
// The bound matrix is a list of entries sorted by (row, key), one per address k a block of cycles touched. An entry
// holds ra_a for every access, the bound Val, and Val before (vs) and after (ve) the row's block of cycles. A cycle
// round pairs rows 2i and 2i+1 and matches their keys; a key present on one side only takes the other side from its
// own boundary value (ra = 0, Val = ve of the lo row or vs of the hi row), which is exact because Val is constant
// over a block that never touches k. Every round is O(live entries): one thread per entry finds its partner by
// binary search in the sibling row. The entries that speak for a key of the pair (every entry of the even row, the
// unmatched ones of the odd row) are flagged, and the exclusive scan of the flags gives each its slot: the pair's base
// plus its rank among the pair's keys, i.e. the flagged entries of either row with smaller keys (a merge-path rank).
//
// With p = cycle_rounds_first < t the cycle phase stops after p binds and the address phase runs on the same entries
// re-sorted by (key, row): the pairing, the flags, the scan and the slots are the cycle phase's with the roles of key
// and row swapped (template parameter AM, address-major). An address round pairs keys 2k' and 2k' + 1 and matches
// their rows; a side a key does not hold at a row takes Val from that key's own history: the ve of its last entry at
// an earlier row, or its bound init value when there is none (Val(k, .) is constant between the rows that touch k).
// Each owner's pair is weighted by eq(w[0 .. t - p), row). After the last address bind the one remaining key becomes
// dense T / 2^p-entry tables ra_a, Val (and the bound inc) for the expression pass of the remaining cycle rounds.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "columns.cuh"
#include "member.hpp"

using namespace jb;
using namespace jbi;

namespace {

constexpr int RW_BLOCK = 256;
constexpr unsigned RW_BAD_ADDRESS = 1, RW_BAD_INC = 2;

// One entry buffer (structure of arrays): key[i], row[i] and the A + 3 field arrays ra_0 .. ra_{A-1}, val, vs, ve.
struct RwView {
    uint32_t* key;
    uint32_t* row;
    uint64_t* f;
    size_t cap;
    __device__ __forceinline__ uint64_t* fld(int j) const { return f + (size_t)j * cap * 4; }
};

// The columns of the creation pass (device pointers; val_kind SK_FR = a field table).
struct RwCols {
    const void* addr[RW_MAX_ACCESSES];
    const void* val[RW_MAX_ACCESSES];
    int val_kind[RW_MAX_ACCESSES];
    int addr_kind;
    int w;
};

struct RwCoef {
    Fr c[RW_MAX_ACCESSES];
    unsigned d_mask;  // bit a: d_a = 1
};

struct RwTabs {
    uint64_t* t[RW_MAX_ACCESSES + 2];  // ra_0 .. ra_{A-1}, Val, inc
};

template <int A>
struct Side {
    Fr ra[A];
    Fr val, vs, ve;
};

template <int A>
__device__ __forceinline__ void load_side(const RwView& v, size_t i, Side<A>& s) {
#pragma unroll
    for (int a = 0; a < A; ++a) s.ra[a] = ld_elem<Fr>(v.fld(a), i);
    s.val = ld_elem<Fr>(v.fld(A), i);
    s.vs = ld_elem<Fr>(v.fld(A + 1), i);
    s.ve = ld_elem<Fr>(v.fld(A + 2), i);
}

// The side of a key its row does not hold: no access, Val constant at the boundary value b.
template <int A>
__device__ __forceinline__ void absent_side(const Fr& b, Side<A>& s) {
#pragma unroll
    for (int a = 0; a < A; ++a) s.ra[a] = Fr::zero();
    s.val = b;
    s.vs = b;
    s.ve = b;
}

// The index entries are grouped by (major) and ordered by within a group (minor): the row and the key in the cycle
// phase, the key and the row in the address phase (AM).
template <bool AM>
__device__ __forceinline__ uint32_t* major_of(const RwView& v) { return AM ? v.key : v.row; }
template <bool AM>
__device__ __forceinline__ uint32_t* minor_of(const RwView& v) { return AM ? v.row : v.key; }

struct RwPair {
    uint32_t maj;   // the entry's row (key when AM)
    uint32_t lb;    // the first entry of the sibling group whose minor is not below the entry's
    int64_t mate;   // the sibling group's entry of the same minor, or -1
    bool owner;     // the entry speaks for its minor: in the even group, or unmatched in the odd group
};

template <bool AM>
__device__ __forceinline__ RwPair rw_pair(const RwView& v, const uint32_t* off, uint32_t e) {
    const uint32_t* mn = minor_of<AM>(v);
    RwPair p;
    p.maj = major_of<AM>(v)[e];
    const uint32_t x = mn[e], sib = p.maj ^ 1u, beg = off[sib], end = off[sib + 1];
    uint32_t lo = beg, hi = end;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (mn[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    const bool matched = lo < end && mn[lo] == x;
    p.lb = lo;
    p.mate = matched ? (int64_t)lo : -1;
    p.owner = !(p.maj & 1u) || !matched;
    return p;
}

// Address phase: Val of the sibling key at the entry's row when the sibling holds no entry there - the ve of its last
// entry at an earlier row (the one before lb), else its bound init value.
__device__ __forceinline__ Fr key_boundary(const RwView& v, int A, const uint32_t* off, const uint64_t* init,
                                           const RwPair& p) {
    const uint32_t sib = p.maj ^ 1u;
    return p.lb > off[sib] ? ld_elem<Fr>(v.fld(A + 2), p.lb - 1) : ld_elem<Fr>(init, sib);
}

template <int A>
__device__ __forceinline__ void pair_sides(const RwView& v, uint32_t e, const RwPair& p, Side<A>& lo, Side<A>& hi) {
    if (!(p.maj & 1u)) {
        load_side<A>(v, e, lo);
        if (p.mate >= 0) load_side<A>(v, (size_t)p.mate, hi);
        else absent_side<A>(lo.ve, hi);
    } else {
        load_side<A>(v, e, hi);
        absent_side<A>(hi.vs, lo);
    }
}

// Where an owner's folded entry goes: the pair's base (the owners of the earlier pairs) plus the owners of the pair
// with smaller minors - in its own group before it, and in the sibling group before lb.
__device__ __forceinline__ size_t rw_slot(const uint32_t* off, const uint32_t* base, uint32_t e, const RwPair& p) {
    const uint32_t ev = off[p.maj & ~1u], od = off[p.maj | 1u];
    return (p.maj & 1u) ? (size_t)base[ev] + (p.lb - ev) + (base[e] - base[od])
                        : (size_t)base[ev] + (e - ev) + (base[p.lb] - base[od]);
}

// R = sum_a c_a ra_a and W = sum_{a: d_a = 1} c_a ra_a of one side.
template <int A>
__device__ __forceinline__ void side_sums(const Side<A>& s, const RwCoef& cf, Fr& R, Fr& W) {
    R = Fr::zero();
    W = Fr::zero();
#pragma unroll
    for (int a = 0; a < A; ++a) {
        const Fr t = fp_mul(cf.c[a], s.ra[a]);
        R = fp_add(R, t);
        if (cf.d_mask >> a & 1u) W = fp_add(W, t);
    }
}

// q(0) and q(inf) of a cycle round, over the owners: per pair y the weight eq_out[y >> in_bits] * eq_in[y & mask] times
//   q(0)   = R_lo val_lo + W_lo inc_lo,
//   q(inf) = (R_hi - R_lo)(val_hi - val_lo) + (W_hi - W_lo)(inc_hi - inc_lo).
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_eval_kernel(RwView v, const uint32_t* off, uint32_t n, const uint64_t* inc,
                                                           RwCoef cf, EqWeights eqw, RoundOut out) {
    __shared__ uint32_t smem[RW_BLOCK / 32 * 2 * 8];
    Fr acc[2] = {Fr::zero(), Fr::zero()};
    const size_t mask = ((size_t)1 << eqw.in_bits) - 1;
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const RwPair p = rw_pair<false>(v, off, e);
        if (!p.owner) continue;
        Side<A> lo, hi;
        pair_sides<A>(v, e, p, lo, hi);
        const size_t y = p.maj >> 1;
        Fr Rl, Wl, Rh, Wh;
        side_sums<A>(lo, cf, Rl, Wl);
        side_sums<A>(hi, cf, Rh, Wh);
        const Fr il = ld_elem<Fr>(inc, 2 * y), ih = ld_elem<Fr>(inc, 2 * y + 1);
        const Fr q0 = fp_add(fp_mul(Rl, lo.val), fp_mul(Wl, il));
        const Fr qi = fp_add(fp_mul(fp_sub(Rh, Rl), fp_sub(hi.val, lo.val)), fp_mul(fp_sub(Wh, Wl), fp_sub(ih, il)));
        const Fr wt = fp_mul(ld_elem<Fr>(eqw.e_out, y >> eqw.in_bits), ld_elem<Fr>(eqw.e_in, y & mask));
        acc[0] = fp_add(acc[0], fp_mul(wt, q0));
        acc[1] = fp_add(acc[1], fp_mul(wt, qi));
    }
    block_sum<2>(acc, smem);
    round_epilogue<2>(acc, smem, out);
}

// R = sum_a c_a ra_a, W = sum_{a: d_a = 1} c_a ra_a and val of entry i, or of an absent side (i < 0: ra = 0, val = b),
// read field by field (the address pass keeps no whole sides in registers).
template <int A>
__device__ __forceinline__ void side_terms(const RwView& v, int64_t i, const Fr& b, const RwCoef& cf, Fr& R, Fr& W, Fr& val) {
    R = Fr::zero();
    W = Fr::zero();
    if (i < 0) {
        val = b;
        return;
    }
#pragma unroll
    for (int a = 0; a < A; ++a) {
        const Fr t = fp_mul(cf.c[a], ld_elem<Fr>(v.fld(a), (size_t)i));
        R = fp_add(R, t);
        if (cf.d_mask >> a & 1u) W = fp_add(W, t);
    }
    val = ld_elem<Fr>(v.fld(A), (size_t)i);
}

// q(0), q(1) and q(inf) of an address round over the owners, unscaled (the host multiplies the eq scalar in): per
// owner the weight eq(w[0 .. t - p), row) = eq_out[y >> in_bits] * eq_in[y & mask] * lin[row & 1] (y = row >> 1, lin
// the factor of the row's lowest variable) times
//   q(0) = R_lo val_lo + W_lo inc,   q(1) = R_hi val_hi + W_hi inc,   q(inf) = (R_hi - R_lo)(val_hi - val_lo),
// inc = inc(row) being the same on both sides of an address pair.
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_key_eval_kernel(RwView v, const uint32_t* off, uint32_t n,
                                                               const uint64_t* inc, const uint64_t* init, RwCoef cf,
                                                               EqWeights eqw, Fr lin0, Fr lin1, RoundOut out) {
    __shared__ uint32_t smem[RW_BLOCK / 32 * 3 * 8];
    Fr acc[3] = {Fr::zero(), Fr::zero(), Fr::zero()};
    const size_t mask = ((size_t)1 << eqw.in_bits) - 1;
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const RwPair p = rw_pair<true>(v, off, e);
        if (!p.owner) continue;
        const int64_t li = (p.maj & 1u) ? -1 : (int64_t)e, hi = (p.maj & 1u) ? (int64_t)e : p.mate;
        const Fr b = li < 0 || hi < 0 ? key_boundary(v, A, off, init, p) : Fr::zero();
        Fr Rl, Wl, vl, Rh, Wh, vh;
        side_terms<A>(v, li, b, cf, Rl, Wl, vl);
        side_terms<A>(v, hi, b, cf, Rh, Wh, vh);
        const uint32_t row = v.row[e];
        const size_t y = row >> 1;
        const Fr ic = ld_elem<Fr>(inc, row);
        Fr lin;  // (selected limb by limb: a select of the whole parameter would go through local memory)
#pragma unroll
        for (int w = 0; w < 8; ++w) lin.v[w] = (row & 1u) ? lin1.v[w] : lin0.v[w];
        const Fr wt = fp_mul(fp_mul(ld_elem<Fr>(eqw.e_out, y >> eqw.in_bits), ld_elem<Fr>(eqw.e_in, y & mask)), lin);
        acc[0] = fp_add(acc[0], fp_mul(wt, fp_add(fp_mul(Rl, vl), fp_mul(Wl, ic))));
        acc[1] = fp_add(acc[1], fp_mul(wt, fp_add(fp_mul(Rh, vh), fp_mul(Wh, ic))));
        acc[2] = fp_add(acc[2], fp_mul(wt, fp_mul(fp_sub(Rh, Rl), fp_sub(vh, vl))));
    }
    block_sum<3>(acc, smem);
    round_epilogue<3>(acc, smem, out);
}

// flag[e] = 1 for the entries that become an entry of the bound matrix (the owners).
template <bool AM>
__global__ void __launch_bounds__(RW_BLOCK) rw_flag_kernel(RwView v, const uint32_t* off, uint32_t n, uint32_t* flag) {
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x)
        flag[e] = rw_pair<AM>(v, off, e).owner ? 1u : 0u;
}

// The bind of a round: each owner writes its minor's folded entry at rw_slot, with major >> 1. ra_a and val are bound
// in both phases; the cycle phase keeps vs of the lo side and ve of the hi side (the pair's block of cycles), the
// address phase binds ve (Val after the row, at the bound address).
template <int A, bool AM>
__global__ void __launch_bounds__(RW_BLOCK) rw_bind_kernel(RwView in, const uint32_t* off, uint32_t n,
                                                           const uint32_t* base, const uint64_t* init, BindScalar s,
                                                           RwView out) {
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const RwPair p = rw_pair<AM>(in, off, e);
        if (!p.owner) continue;
        const size_t o = rw_slot(off, base, e, p);
        minor_of<AM>(out)[o] = minor_of<AM>(in)[e];
        major_of<AM>(out)[o] = p.maj >> 1;
        // the two sides field by field (as pair_sides, one field at a time): an absent side has ra = 0 and the
        // boundary value b for val, vs and ve
        const int64_t li = (p.maj & 1u) ? -1 : (int64_t)e, hi = (p.maj & 1u) ? (int64_t)e : p.mate;
        Fr b = Fr::zero();
        if (AM) {
            if (li < 0 || hi < 0) b = key_boundary(in, A, off, init, p);
        } else {
            b = (p.maj & 1u) ? ld_elem<Fr>(in.fld(A + 1), e) : hi < 0 ? ld_elem<Fr>(in.fld(A + 2), e) : Fr::zero();
        }
        auto side = [&](int j, int64_t i) { return i >= 0 ? ld_elem<Fr>(in.fld(j), (size_t)i) : j < A ? Fr::zero() : b; };
#pragma unroll
        for (int j = 0; j <= A; ++j) st_elem(out.fld(j), o, bind_pair<false>(side(j, li), side(j, hi), s));
        if (AM) {
            st_elem(out.fld(A + 2), o, bind_pair<false>(side(A + 2, li), side(A + 2, hi), s));
        } else {
            st_elem(out.fld(A + 1), o, side(A + 1, li));
            st_elem(out.fld(A + 2), o, side(A + 2, hi));
        }
    }
}

// Row offsets of the bound matrix: new_off[y] = base[off[2y]] for y <= rows / 2 (off[rows] = n, base[n] = total).
__global__ void __launch_bounds__(RW_BLOCK) rw_rows_kernel(const uint32_t* off, const uint32_t* base, size_t half,
                                                           uint32_t* new_off) {
    for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y <= half; y += (size_t)gridDim.x * blockDim.x)
        new_off[y] = base[off[2 * y]];
}

__global__ void __launch_bounds__(RW_BLOCK) rw_iota_kernel(uint32_t n, uint32_t* out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = i;
}

// The entries in (key, row) order: out's keys are already sorted (a stable sort by key of entries sorted by (row,
// key)); entry i takes the row, ra_a, val and ve of in's entry perm[i] (vs is not needed by the address phase).
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_gather_kernel(RwView in, const uint32_t* perm, uint32_t n, RwView out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t s = perm[i];
        out.row[i] = in.row[s];
#pragma unroll 1
        for (int j = 0; j < A + 3; ++j)
            if (j != A + 1) st_elem(out.fld(j), i, ld_elem<Fr>(in.fld(j), s));
    }
}

// Key offsets of sorted keys: off[k] = the first entry whose key is not below k, k <= K.
__global__ void __launch_bounds__(RW_BLOCK) rw_key_offsets_kernel(const uint32_t* key, uint32_t n, size_t K, uint32_t* off) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k <= K; k += (size_t)gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (key[mid] < k) lo = mid + 1;
            else hi = mid;
        }
        off[k] = lo;
    }
}

// The one remaining key's entries (sorted by row) as dense tables over the rows: ra_a = the entry's, or 0 where the
// row has none; Val = the entry's val, else the ve of the last entry at an earlier row, else the bound init value.
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_dense_kernel(RwView v, uint32_t n, size_t rows, const uint64_t* init,
                                                            RwTabs tb) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (v.row[mid] < i) lo = mid + 1;
            else hi = mid;
        }
        const bool hit = lo < n && v.row[lo] == i;
#pragma unroll
        for (int a = 0; a < A; ++a) st_elem(tb.t[a], i, hit ? ld_elem<Fr>(v.fld(a), lo) : Fr::zero());
        st_elem(tb.t[A], i, hit ? ld_elem<Fr>(v.fld(A), lo) : lo > 0 ? ld_elem<Fr>(v.fld(A + 2), lo - 1) : ld_elem<Fr>(init, 0));
    }
}

__device__ __forceinline__ Fr ld_value(const void* p, int kind, size_t i) {
    if (kind == SK_FR) return ld_elem<Fr>(static_cast<const uint64_t*>(p), i);
    uint32_t mag[4];
    const bool neg = ld_small(p, i, kind, mag);
    return promote_small(mag, neg);
}

// A field table of n entries from a field table or a compact column.
__global__ void __launch_bounds__(RW_BLOCK) rw_load_kernel(const void* src, int kind, size_t n, uint64_t* out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        st_elem(out, i, ld_value(src, kind, i));
}

// The addresses of cycle j's accesses (NO_ADDRESS for none and, raising RW_BAD_ADDRESS, for an address >= K), the
// write's address aw, and which accesses speak for their address (lead[a]: the first access to it).
template <int A>
__device__ __forceinline__ int cycle_keys(const RwCols& cols, size_t j, uint32_t K, uint32_t (&ad)[A], bool (&lead)[A],
                                          uint32_t& aw, unsigned* bad) {
    int nk = 0;
    aw = NO_ADDRESS;
#pragma unroll
    for (int a = 0; a < A; ++a) {
        ad[a] = ld_address<SK_U32>(cols.addr[a], j, cols.addr_kind);
        if (ad[a] != NO_ADDRESS && ad[a] >= K) {
            if (bad) atomicOr(bad, RW_BAD_ADDRESS);
            ad[a] = NO_ADDRESS;
        }
        if (a == cols.w) aw = ad[a];
        lead[a] = ad[a] != NO_ADDRESS;
#pragma unroll
        for (int b = 0; b < a; ++b) lead[a] = lead[a] && ad[b] != ad[a];
        nk += lead[a] ? 1 : 0;
    }
    return nk;
}

// Entries per cycle, and the checks of the columns: an address >= K that is not none, a nonzero increment at a
// cycle whose write address is none.
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_count_kernel(RwCols cols, size_t T, uint32_t K, const uint64_t* inc,
                                                            uint32_t* count, unsigned* bad) {
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < T; j += (size_t)gridDim.x * blockDim.x) {
        uint32_t ad[A], aw;
        bool lead[A];
        count[j] = (uint32_t)cycle_keys<A>(cols, j, K, ad, lead, aw, bad);
        if (aw == NO_ADDRESS && !ld_elem<Fr>(inc, j).is_zero()) atomicOr(bad, RW_BAD_INC);
    }
}

// The unbound matrix: row j holds one entry per address k cycle j touches, in ascending order, with
// ra_a = [addr_a(j) = k], val = vs = v_a(j) of the first access to k (they all agree: v_a(j) = Val(k, j)) and
// ve = val + [addr_w(j) = k] inc(j).
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_fill_kernel(RwCols cols, size_t T, uint32_t K, const uint64_t* inc,
                                                           const uint32_t* off, RwView v) {
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < T; j += (size_t)gridDim.x * blockDim.x) {
        uint32_t ad[A], aw;
        bool lead[A];
        cycle_keys<A>(cols, j, K, ad, lead, aw, nullptr);
#pragma unroll
        for (int a = 0; a < A; ++a) {
            if (!lead[a]) continue;
            int rank = 0;
#pragma unroll
            for (int b = 0; b < A; ++b) rank += (lead[b] && ad[b] < ad[a]) ? 1 : 0;
            const size_t o = (size_t)off[j] + rank;
#pragma unroll
            for (int b = 0; b < A; ++b) st_elem(v.fld(b), o, ad[b] == ad[a] ? Fr::one() : Fr::zero());
            const Fr val = ld_value(cols.val[a], cols.val_kind[a], j);
            v.key[o] = ad[a];
            v.row[o] = (uint32_t)j;
            st_elem(v.fld(A), o, val);
            st_elem(v.fld(A + 1), o, val);
            st_elem(v.fld(A + 2), o, aw == ad[a] ? fp_add(val, ld_elem<Fr>(inc, j)) : val);
        }
    }
}

// The address phase's tables before the scatter: ra_a = 0, Val = init, inc = the bound inc(r_cycle) everywhere.
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_tables_kernel(RwTabs tb, size_t K, const uint64_t* init, const uint64_t* inc1) {
    const Fr ir = ld_elem<Fr>(inc1, 0);
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < K; k += (size_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < A; ++a) st_elem(tb.t[a], k, Fr::zero());
        st_elem(tb.t[A], k, ld_elem<Fr>(init, k));
        st_elem(tb.t[A + 1], k, ir);
    }
}

// The one remaining row's entries into the address tables.
template <int A>
__global__ void __launch_bounds__(RW_BLOCK) rw_scatter_kernel(RwView v, uint32_t n, RwTabs tb) {
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const uint32_t k = v.key[e];
#pragma unroll
        for (int a = 0; a < A; ++a) st_elem(tb.t[a], k, ld_elem<Fr>(v.fld(a), e));
        st_elem(tb.t[A], k, ld_elem<Fr>(v.fld(A), e));
    }
}

RwView view(const RwState& rw, int b) { return RwView{rw.key[b], rw.row[b], rw.f[b], rw.cap}; }

unsigned grid_for(const jb_ctx* c, size_t items) { return launch_grid(c, items, RW_BLOCK, 8); }

// Kernel templates by access count (A = 1 .. 4).
template <template <int> class K, class... Args>
void by_a(int A, Args&&... args) {
    switch (A) {
        case 1: K<1>::run(args...); break;
        case 2: K<2>::run(args...); break;
        case 3: K<3>::run(args...); break;
        default: K<4>::run(args...); break;
    }
}
template <int A>
struct EvalL {
    static void run(jb_ctx* c, const RwState& rw, const RwCoef& cf, const EqWeights& eqw, RoundOut ro, int* st) {
        *st = launch_round(c, rw_eval_kernel<A>, RW_BLOCK, 0, 8, rw.n, 2, 2, 3, "rw_eval_kernel launch", ro,
                           view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n, (const uint64_t*)rw.inc.buf, cf, eqw);
    }
};
template <int A>
struct KeyEvalL {
    static void run(jb_ctx* c, const RwState& rw, const RwCoef& cf, const EqWeights& eqw, const Fr& l0, const Fr& l1,
                    RoundOut ro, int* st) {
        *st = launch_round(c, rw_key_eval_kernel<A>, RW_BLOCK, 0, 8, rw.n, 3, 2, 2, "rw_key_eval_kernel launch", ro,
                           view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n, (const uint64_t*)rw.inc.buf,
                           (const uint64_t*)rw.init.buf, cf, eqw, l0, l1);
    }
};
template <int A>
struct BindL {
    static void run(jb_ctx* c, const RwState& rw, const BindScalar& s) {
        const unsigned g = grid_for(c, rw.n);
        if (rw.by_key)
            rw_bind_kernel<A, true><<<g, RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n,
                                                                  rw.base, rw.init.buf, s, view(rw, rw.cur ^ 1));
        else
            rw_bind_kernel<A, false><<<g, RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n,
                                                                   rw.base, nullptr, s, view(rw, rw.cur ^ 1));
    }
};
template <int A>
struct GatherL {
    static void run(jb_ctx* c, const RwState& rw) {
        rw_gather_kernel<A><<<grid_for(c, rw.n), RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), rw.base, (uint32_t)rw.n,
                                                                          view(rw, rw.cur ^ 1));
    }
};
template <int A>
struct DenseL {
    static void run(jb_ctx* c, const RwState& rw, size_t rows, const RwTabs& tb) {
        rw_dense_kernel<A><<<grid_for(c, rows), RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), (uint32_t)rw.n, rows,
                                                                         rw.init.buf, tb);
    }
};
template <int A>
struct CountL {
    static void run(jb_ctx* c, const RwCols& cols, const RwState& rw, unsigned* bad) {
        rw_count_kernel<A><<<grid_for(c, rw.T), RW_BLOCK, 0, c->stream>>>(cols, rw.T, (uint32_t)rw.K, rw.inc.buf, rw.flag, bad);
    }
};
template <int A>
struct FillL {
    static void run(jb_ctx* c, const RwCols& cols, const RwState& rw) {
        rw_fill_kernel<A><<<grid_for(c, rw.T), RW_BLOCK, 0, c->stream>>>(cols, rw.T, (uint32_t)rw.K, rw.inc.buf,
                                                                        rw.off[0], view(rw, 0));
    }
};
template <int A>
struct TablesL {
    static void run(jb_ctx* c, const RwState& rw, const RwTabs& tb) {
        rw_tables_kernel<A><<<grid_for(c, rw.K), RW_BLOCK, 0, c->stream>>>(tb, rw.K, rw.init.buf, rw.inc.buf);
    }
};
template <int A>
struct ScatterL {
    static void run(jb_ctx* c, const RwState& rw, const RwTabs& tb) {
        rw_scatter_kernel<A><<<grid_for(c, rw.n), RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), (uint32_t)rw.n, tb);
    }
};

// base = exclusive scan of flag over `items` entries.
int scan(jb_ctx* c, RwState& rw, size_t items) {
    size_t bytes = rw.scan_bytes;
    return c->check(cub::DeviceScan::ExclusiveSum(rw.scan_tmp, bytes, rw.flag, rw.base, (int)items, c->stream),
                    "read-write: scan");
}

// Reads the live entry count (the last row offset) back.
int read_count(jb_ctx* c, RwState& rw) {
    int st = c->check(cudaMemcpyAsync(c->h_small, rw.off[rw.cur] + rw.rows, sizeof(uint32_t), cudaMemcpyDeviceToHost,
                                      c->stream), "read-write: count D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "read-write: count sync");
    if (st == JB_OK) rw.n = *(const uint32_t*)c->h_small;
    return st;
}

int load_field(jb_ctx* c, const jb_source& s, size_t n, uint64_t* out) {
    if (s.type == JB_SOURCE_TABLE)
        return c->check(cudaMemcpyAsync(out, c->find(s.table)->buf, n * 32, cudaMemcpyDeviceToDevice, c->stream),
                        "read-write: table copy");
    Scratch scratch(c);
    const void* d = nullptr;
    int st = get_column(scratch, s.values, n * (size_t)small_kind_bytes(s.kind), s.on_device, &d);
    if (st != JB_OK) return st;
    rw_load_kernel<<<grid_for(c, n), RW_BLOCK, 0, c->stream>>>(d, s.kind, n, out);
    return c->check(cudaGetLastError(), "rw_load_kernel launch");
}

// A value, increment or initial-value source: a field table of n entries or a compact column.
int check_rw_source(jb_ctx* c, const jb_source& s, size_t n, const char* what) {
    if (s.type == JB_SOURCE_TABLE) {
        const Table* t = c->find(s.table);
        if (!t) return fail_column(c, JB_ERR_INVALID, what, "unknown table handle");
        if (t->len != n) return fail_column(c, JB_ERR_INVALID, what, "a table of another length");
        return JB_OK;
    }
    if (s.type != JB_SOURCE_COMPACT) return fail_column(c, JB_ERR_INVALID, what, "a field table or a compact column");
    return check_compact_column(c, what, s.kind, s.values, s.on_device);
}

RwCoef coefficients(const RwState& rw) {
    RwCoef cf;
    std::memset(&cf, 0, sizeof cf);
    for (int a = 0; a < rw.A; ++a) {
        for (int w = 0; w < 4; ++w) {
            cf.c[a].v[2 * w] = (uint32_t)rw.coeff[a][w];
            cf.c[a].v[2 * w + 1] = (uint32_t)(rw.coeff[a][w] >> 32);
        }
        if (rw.d[a]) cf.d_mask |= 1u << a;
    }
    return cf;
}

Fr device_fr(const HostFr& x) {
    uint64_t l[4];
    x.store(l);
    Fr f;
    for (int w = 0; w < 4; ++w) {
        f.v[2 * w] = (uint32_t)l[w];
        f.v[2 * w + 1] = (uint32_t)(l[w] >> 32);
    }
    return f;
}

// One bind of the bound matrix (either phase): flag the owners, scan, write the folded entries and the new group
// offsets; the other buffer becomes the current one with half the groups. The caller reads the new count back.
int bind_entries(jb_ctx* c, RwState& rw, const uint64_t r[4]) {
    bool hi4;
    const BindScalar s = make_scalar(r, &hi4);
    const unsigned g = grid_for(c, rw.n);
    if (rw.by_key) rw_flag_kernel<true><<<g, RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n, rw.flag);
    else rw_flag_kernel<false><<<g, RW_BLOCK, 0, c->stream>>>(view(rw, rw.cur), rw.off[rw.cur], (uint32_t)rw.n, rw.flag);
    int st = c->check(cudaMemsetAsync(rw.flag + rw.n, 0, sizeof(uint32_t), c->stream), "read-write: memset");
    if (st == JB_OK) st = scan(c, rw, rw.n + 1);
    if (st != JB_OK) return st;
    by_a<BindL>(rw.A, c, rw, s);
    const size_t half = rw.rows / 2;
    rw_rows_kernel<<<grid_for(c, half + 1), RW_BLOCK, 0, c->stream>>>(rw.off[rw.cur], rw.base, half, rw.off[rw.cur ^ 1]);
    c->launches += 4;
    if ((st = c->check(cudaGetLastError(), "read-write: bind launch")) != JB_OK) return st;
    rw.cur ^= 1;
    rw.rows = half;
    return JB_OK;
}

}  // namespace


void rw_release(jb_member* mem) {
    RwState* rw = mem->rw;
    if (!rw) return;
    jb_ctx* c = mem->ctx;
    for (int b = 0; b < 2; ++b) {
        c->dev_free(rw->key[b]);
        c->dev_free(rw->row[b]);
        c->dev_free(rw->f[b]);
        c->dev_free(rw->off[b]);
        rw->key[b] = rw->row[b] = nullptr;
        rw->f[b] = nullptr;
        rw->off[b] = nullptr;
    }
    c->dev_free(rw->flag);
    c->dev_free(rw->base);
    c->dev_free(rw->scan_tmp);
    rw->flag = rw->base = nullptr;
    rw->scan_tmp = nullptr;
    c->release(rw->init);
    c->release(rw->inc);
}

int rw_create(jb_ctx* c, const jb_rw_access* acc, size_t A, size_t w, int addr_kind, int addr_on_device, size_t T,
              size_t K, const jb_source* inc, const jb_source* init, const uint64_t* w_cycle, size_t nvars,
              const uint64_t* scale, size_t cycle_rounds_first, int order, jb_member** out) {
    const char* what = "read-write";
    if (!acc || !inc || !init || !out || (nvars && !w_cycle)) return c->fail(JB_ERR_INVALID, "read-write: null pointer");
    if (order == JB_HIGH_TO_LOW)
        return c->fail(JB_ERR_UNSUPPORTED, "read-write: HighToLow (a cycle round pairs adjacent cycles)");
    if (order != JB_LOW_TO_HIGH) return c->fail(JB_ERR_INVALID, "read-write: unknown binding order");
    if (A > RW_MAX_ACCESSES) return c->fail(JB_ERR_UNSUPPORTED, "read-write: at most 4 accesses");
    if (A == 0) return c->fail(JB_ERR_INVALID, "read-write: no accesses");
    if (w >= A) return c->fail(JB_ERR_INVALID, "read-write: the write access is not an access");
    if (!pow2(T) || T < 2 || T > ((size_t)1 << 30))
        return c->fail(JB_ERR_INVALID, "read-write: T must be a power of two in [2, 2^30]");
    if (!pow2(K) || (one_hot_kind(addr_kind, SK_U32) && K > one_hot_max_k(addr_kind)))
        return c->fail(JB_ERR_INVALID, addr_kind == SK_U32 ? "read-write: K must be a power of two in [1, 2^24]"
                                                           : "read-write: K must be a power of two in [1, 2^16]");
    const void* cols[RW_MAX_ACCESSES];
    for (size_t a = 0; a < A; ++a) cols[a] = acc[a].addr;
    int st = check_one_hot_columns(c, what, addr_kind, T, K, addr_on_device, cols, A, SK_U32);
    if (st != JB_OK) return st;
    size_t ncols = 0;  // distinct address columns: a cycle has at most that many entries
    for (size_t a = 0; a < A; ++a) {
        if ((st = check_rw_source(c, acc[a].value, T, "read-write value")) != JB_OK) return st;
        if (!canonical_fr(acc[a].coeff)) return c->fail(JB_ERR_INVALID, "read-write: coefficient limbs not canonical");
        if (acc[a].write_flag != 0 && acc[a].write_flag != 1) return c->fail(JB_ERR_INVALID, "read-write: write_flag must be 0 or 1");
        bool seen = false;
        for (size_t b = 0; b < a; ++b) seen = seen || cols[b] == cols[a];
        ncols += seen ? 0 : 1;
    }
    if (std::min(ncols, K) * T >= ((size_t)1 << 31))
        return c->fail(JB_ERR_INVALID, "read-write: min(K, address columns) * T must be below 2^31");
    if ((st = check_rw_source(c, *inc, T, "read-write inc")) != JB_OK) return st;
    if ((st = check_rw_source(c, *init, K, "read-write init")) != JB_OK) return st;
    const size_t t = (size_t)log2_of(T);
    if (nvars != t) return c->fail(JB_ERR_INVALID, "read-write: the eq point must have log2(T) coordinates");
    for (size_t i = 0; i < nvars; ++i)
        if (!canonical_fr(w_cycle + 4 * i)) return c->fail(JB_ERR_INVALID, "read-write: point limbs not canonical");
    if (scale && !canonical_fr(scale)) return c->fail(JB_ERR_INVALID, "read-write: scale not canonical");
    if (cycle_rounds_first > t) return c->fail(JB_ERR_INVALID, "read-write: cycle_rounds_first must be at most log2(T)");

    // everything the rounds need is allocated here
    jb_member* mem = new_member(c, MemberKind::ReadWrite, 2, 1, JB_LOW_TO_HIGH, K * T);
    if (!mem) return JB_ERR_OOM;
    RwState* rw = new (std::nothrow) RwState();
    if (!rw) {
        delete mem;
        return JB_ERR_OOM;
    }
    mem->rw = rw;
    rw->A = (int)A;
    rw->w = (int)w;
    rw->T = T;
    rw->K = K;
    rw->rows = T;
    rw->cap = std::min(ncols, K) * T;
    rw->p = K == 1 ? t : cycle_rounds_first;  // (K = 1: no address rounds, every order is the same)
    rw->kappa = (size_t)log2_of(K);
    const bool mixed = rw->p < t;
    for (size_t a = 0; a < A; ++a) {
        std::memcpy(rw->coeff[a], acc[a].coeff, 32);
        rw->d[a] = acc[a].write_flag;
    }
    const size_t nf = A + 3;
    for (int b = 0; b < 2 && st == JB_OK; ++b) {
        st = c->dev_alloc((void**)&rw->key[b], rw->cap * 4);
        if (st == JB_OK) st = c->dev_alloc((void**)&rw->row[b], rw->cap * 4);
        if (st == JB_OK) st = c->dev_alloc((void**)&rw->f[b], rw->cap * nf * 32);
        // row offsets, and key offsets (K + 1) in the address phase
        const size_t offs = std::max(b == 0 ? T + 1 : T / 2 + 1, mixed ? K + 1 : 0);
        if (st == JB_OK) st = c->dev_alloc((void**)&rw->off[b], offs * 4);
    }
    if (st == JB_OK) st = c->dev_alloc((void**)&rw->flag, (rw->cap + 1) * 4);
    if (st == JB_OK) st = c->dev_alloc((void**)&rw->base, (rw->cap + 1) * 4);
    if (st == JB_OK) {
        const size_t items = std::max(rw->cap, T) + 1;
        st = c->check(cub::DeviceScan::ExclusiveSum(nullptr, rw->scan_bytes, rw->flag, rw->base, (int)items, c->stream),
                      "read-write: scan size");
        size_t sort_bytes = 0;  // the address phase's sort by key shares the scan's workspace
        if (st == JB_OK && mixed)
            st = c->check(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, rw->key[0], rw->key[1], rw->flag, rw->base,
                                                          (int)rw->cap, 0, (int)rw->kappa, c->stream),
                          "read-write: sort size");
        rw->scan_bytes = std::max(rw->scan_bytes, sort_bytes);
        if (st == JB_OK) st = c->dev_alloc(&rw->scan_tmp, rw->scan_bytes);
    }
    if (st == JB_OK) st = c->dev_alloc((void**)&rw->init.buf, K * 32);
    if (st == JB_OK) {
        rw->init.cap = rw->init.len = K;
        if (mixed) st = c->ensure_alt(rw->init, K / 2);  // bound by the address rounds
    }
    if (st == JB_OK) st = c->dev_alloc((void**)&rw->inc.buf, T * 32);
    if (st == JB_OK) {
        rw->inc.cap = rw->inc.len = T;
        st = c->ensure_alt(rw->inc, T / 2);
    }
    // the tables of the expression pass: A + 2 over the K addresses, or (mixed) ra_a and Val over the T / 2^p rows
    // that remain after the address rounds, inc being the bound inc table itself
    const size_t tab_len = mixed ? T >> rw->p : K;
    mem->tables.resize(A + 2);
    for (size_t j = 0; j < (mixed ? A + 1 : A + 2) && st == JB_OK; ++j) {
        Table& tb = mem->tables[j];
        st = c->dev_alloc((void**)&tb.buf, tab_len * 32);
        tb.cap = tb.len = tab_len;
        if (st == JB_OK) st = c->ensure_alt(tb, std::max<size_t>(tab_len / 2, 1));
    }
    // the rows of the unbound matrix, straight from the borrowed columns
    unsigned* d_bad = nullptr;
    Scratch scratch(c);
    RwCols rc;
    std::memset(&rc, 0, sizeof rc);
    rc.addr_kind = addr_kind;
    rc.w = (int)w;
    if (st == JB_OK) st = scratch.alloc(sizeof(unsigned), &d_bad);
    if (st == JB_OK) st = c->check(cudaMemsetAsync(d_bad, 0, sizeof(unsigned), c->stream), "read-write: flag memset");
    if (st == JB_OK) st = load_field(c, *inc, T, rw->inc.buf);
    if (st == JB_OK) st = load_field(c, *init, K, rw->init.buf);
    for (size_t a = 0; a < A && st == JB_OK; ++a) {
        size_t same = a;  // an address column shared with an earlier access is copied once
        for (size_t b = 0; b < a && same == a; ++b)
            if (acc[b].addr == acc[a].addr) same = b;
        if (same < a) rc.addr[a] = rc.addr[same];
        else st = get_column(scratch, acc[a].addr, T * (size_t)small_kind_bytes(addr_kind), addr_on_device, &rc.addr[a]);
        const jb_source& v = acc[a].value;
        rc.val_kind[a] = v.type == JB_SOURCE_TABLE ? SK_FR : v.kind;
        if (st == JB_OK && v.type == JB_SOURCE_TABLE) rc.val[a] = c->find(v.table)->buf;
        else if (st == JB_OK) st = get_column(scratch, v.values, T * (size_t)small_kind_bytes(v.kind), v.on_device, &rc.val[a]);
    }
    if (st == JB_OK) {
        by_a<CountL>((int)A, c, rc, *rw, d_bad);
        st = c->check(cudaGetLastError(), "rw_count_kernel launch");
    }
    if (st == JB_OK) st = c->check(cudaMemsetAsync(rw->flag + T, 0, sizeof(uint32_t), c->stream), "read-write: memset");
    if (st == JB_OK) {
        size_t bytes = rw->scan_bytes;
        st = c->check(cub::DeviceScan::ExclusiveSum(rw->scan_tmp, bytes, rw->flag, rw->off[0], (int)(T + 1), c->stream),
                      "read-write: row scan");
    }
    unsigned bad = 0;
    if (st == JB_OK) st = c->check(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, c->stream),
                                   "read-write: flag D2H");
    if (st == JB_OK) st = c->check(cudaStreamSynchronize(c->stream), "read-write: check sync");
    if (st == JB_OK && (bad & RW_BAD_ADDRESS)) st = fail_bad_address(c);
    if (st == JB_OK && (bad & RW_BAD_INC))
        st = c->fail(JB_ERR_INVALID, "read-write: a nonzero increment at a cycle whose write address is none");
    if (st == JB_OK) {
        by_a<FillL>((int)A, c, rc, *rw);
        st = c->check(cudaGetLastError(), "rw_fill_kernel launch");
    }
    if (st == JB_OK) st = read_count(c, *rw);  // (also: the borrowed columns have been read when this returns)
    if (st != JB_OK) {  // (the caller holds the context lock: no jb_member_destroy here)
        rw_release(mem);
        for (auto& tb : mem->tables) c->release(tb);
        delete rw;
        delete mem;
        return st;
    }
    *out = mem;
    return JB_OK;
}

int rw_cycle_round(jb_member* mem, const uint64_t* bind, const EqWeights& eqw, RoundOut ro) {
    jb_ctx* c = mem->ctx;
    RwState& rw = *mem->rw;
    if (bind) {
        const int st = rw_cycle_bind(mem, bind);
        if (st != JB_OK) return st;
    }
    int st = JB_OK;
    by_a<EvalL>(rw.A, c, rw, coefficients(rw), eqw, ro, &st);
    return st;
}

int rw_cycle_bind(jb_member* mem, const uint64_t r[4]) {
    jb_ctx* c = mem->ctx;
    RwState& rw = *mem->rw;
    int st = bind_entries(c, rw, r);
    if (st != JB_OK) return st;
    mem->len /= 2;
    if ((st = bind_table(c, rw.inc, r, JB_LOW_TO_HIGH)) != JB_OK) return st;
    if ((st = read_count(c, rw)) != JB_OK) return st;
    if (rw.rows > 1) return JB_OK;
    // the last cycle variable is bound: the one remaining row becomes the address phase's K-entry tables
    RwTabs tb;
    for (int j = 0; j < rw.A + 2; ++j) tb.t[j] = mem->tables[j].buf;
    by_a<TablesL>(rw.A, c, rw, tb);
    by_a<ScatterL>(rw.A, c, rw, tb);
    c->launches += 2;
    st = c->check(cudaGetLastError(), "read-write: scatter launch");
    rw_release(mem);  // (stream-ordered: freed after the scatter has read the entries)
    return st;
}

int rw_begin_keys(jb_member* mem) {
    jb_ctx* c = mem->ctx;
    RwState& rw = *mem->rw;
    const unsigned g = grid_for(c, rw.n);
    rw_iota_kernel<<<g, RW_BLOCK, 0, c->stream>>>((uint32_t)rw.n, rw.flag);
    size_t bytes = rw.scan_bytes;
    int st = c->check(cub::DeviceRadixSort::SortPairs(rw.scan_tmp, bytes, rw.key[rw.cur], rw.key[rw.cur ^ 1], rw.flag,
                                                      rw.base, (int)rw.n, 0, (int)rw.kappa, c->stream),
                      "read-write: sort by key");
    if (st != JB_OK) return st;
    by_a<GatherL>(rw.A, c, rw);
    rw_key_offsets_kernel<<<grid_for(c, rw.K + 1), RW_BLOCK, 0, c->stream>>>(rw.key[rw.cur ^ 1], (uint32_t)rw.n, rw.K,
                                                                            rw.off[rw.cur ^ 1]);
    c->launches += 3;
    if ((st = c->check(cudaGetLastError(), "read-write: address phase launch")) != JB_OK) return st;
    rw.cur ^= 1;
    rw.rows = rw.K;
    rw.by_key = true;
    return JB_OK;
}

int rw_key_pass(jb_member* mem, const EqWeights& eqw, const uint64_t* w_low, RoundOut ro) {
    RwState& rw = *mem->rw;
    const HostFr l1 = HostFr::from_limbs(w_low), l0 = HostFr::one() - l1;
    int st = JB_OK;
    by_a<KeyEvalL>(rw.A, mem->ctx, rw, coefficients(rw), eqw, device_fr(l0), device_fr(l1), ro, &st);
    return st;
}

int rw_key_bind(jb_member* mem, const uint64_t r[4]) {
    jb_ctx* c = mem->ctx;
    RwState& rw = *mem->rw;
    int st = bind_entries(c, rw, r);
    if (st != JB_OK) return st;
    mem->len /= 2;
    if ((st = bind_table(c, rw.init, r, JB_LOW_TO_HIGH)) != JB_OK) return st;
    if ((st = read_count(c, rw)) != JB_OK) return st;
    if (rw.rows > 1) return JB_OK;
    // the last address variable is bound: the one remaining key becomes dense tables over the T / 2^p rows
    const size_t rows = rw.T >> rw.p;
    RwTabs tb;
    for (int j = 0; j <= rw.A; ++j) tb.t[j] = mem->tables[j].buf;
    by_a<DenseL>(rw.A, c, rw, rows, tb);
    c->launches++;
    st = c->check(cudaGetLastError(), "rw_dense_kernel launch");
    std::swap(mem->tables[rw.A + 1], rw.inc);
    rw_release(mem);  // (stream-ordered: freed after the dense pass has read the entries)
    return st;
}
