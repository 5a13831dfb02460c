/* ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C CPU restatement of the a16z/jolt hot path over BN254 Fr/Fq, used as
 * (1) the bit-exact checker for the CUDA path at sizes Python cannot reach and
 * (2) the "port" CPU baseline timed by bench.py (all host threads via OpenMP,
 * chunk grain >= 1024 mirroring PAR_THRESHOLD, crates/jolt-poly/src/dense.rs:17).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library.
 *
 * The reference's arithmetic lives in the third-party arkworks fork
 * (a16z/arkworks-algebra @ 76bb3a45, Cargo.lock:883-885), which is absent from
 * /root/reference and cannot be built here (no Rust). This file restates the
 * published algorithms: CIOS Montgomery over 4 x u64 with R = 2^256, Jacobian
 * G1 on y^2 = x^3 + 3, Pippenger with arkworks' window heuristic. It is pinned
 * by tests/test_oracle_c.py against oracle/bn254.py, which is itself pinned by
 * the reference's golden vectors (crates/jolt-field/tests/golden_bytes.rs).
 * G1/MSM: parity unpinned by golden vectors (the reference holds none).
 *
 * All field elements are 4 x u64 little-endian Montgomery limbs, fully reduced
 * (crates/jolt-field/src/bn254/mod.rs:33-42).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef unsigned __int128 u128;
typedef uint64_t u64;

typedef struct {
    u64 p[4];    /* modulus */
    u64 inv;     /* -p^-1 mod 2^64 */
    u64 r1[4];   /* R mod p   (Montgomery one) */
    u64 r2[4];   /* R^2 mod p */
} field_t;

static const field_t FR = {
    {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
    0xc2e1f593efffffffULL,
    {0xac96341c4ffffffbULL, 0x36fc76959f60cd29ULL, 0x666ea36f7879462eULL, 0x0e0a77c19a07df2fULL},
    {0x1bb8e645ae216da7ULL, 0x53fe3ab1e35c59e3ULL, 0x8c49833d53bb8085ULL, 0x0216d0b17f4e44a5ULL}};

static const field_t FQ = {
    {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
    0x87d20782e4866389ULL,
    {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL},
    {0xf32cfc5b538afa89ULL, 0xb5e71911d44501fbULL, 0x47ab1eff0a417ff6ULL, 0x06d89f71cab8351fULL}};

static inline int geq(const u64 a[4], const u64 b[4]) {
    for (int i = 3; i >= 0; --i) {
        if (a[i] != b[i]) return a[i] > b[i];
    }
    return 1;
}

static inline u64 sub4(u64 o[4], const u64 a[4], const u64 b[4]) {
    u64 borrow = 0;
    for (int i = 0; i < 4; ++i) {
        u128 t = (u128)a[i] - b[i] - borrow;
        o[i] = (u64)t;
        borrow = (u64)(t >> 64) & 1;
    }
    return borrow;
}

static inline u64 add4(u64 o[4], const u64 a[4], const u64 b[4]) {
    u64 carry = 0;
    for (int i = 0; i < 4; ++i) {
        u128 t = (u128)a[i] + b[i] + carry;
        o[i] = (u64)t;
        carry = (u64)(t >> 64);
    }
    return carry;
}

static inline void f_add(const field_t *F, u64 o[4], const u64 a[4], const u64 b[4]) {
    u64 t[4];
    add4(t, a, b); /* p < 2^254 so no carry out */
    if (geq(t, F->p)) sub4(o, t, F->p); else memcpy(o, t, 32);
}

static inline void f_sub(const field_t *F, u64 o[4], const u64 a[4], const u64 b[4]) {
    u64 t[4];
    if (sub4(t, a, b)) add4(o, t, F->p); else memcpy(o, t, 32);
}

static inline void f_neg(const field_t *F, u64 o[4], const u64 a[4]) {
    static const u64 z[4] = {0, 0, 0, 0};
    f_sub(F, o, z, a);
}

/* CIOS Montgomery multiplication, R = 2^256. */
static inline void f_mul(const field_t *F, u64 o[4], const u64 a[4], const u64 b[4]) {
    u64 t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        u64 c = 0;
        for (int j = 0; j < 4; ++j) {
            u128 x = (u128)a[j] * b[i] + t[j] + c;
            t[j] = (u64)x;
            c = (u64)(x >> 64);
        }
        u128 x = (u128)t[4] + c;
        t[4] = (u64)x;
        t[5] = (u64)(x >> 64);
        u64 m = t[0] * F->inv;
        x = (u128)m * F->p[0] + t[0];
        c = (u64)(x >> 64);
        for (int j = 1; j < 4; ++j) {
            x = (u128)m * F->p[j] + t[j] + c;
            t[j - 1] = (u64)x;
            c = (u64)(x >> 64);
        }
        x = (u128)t[4] + c;
        t[3] = (u64)x;
        t[4] = t[5] + (u64)(x >> 64);
    }
    if (t[4] || geq(t, F->p)) sub4(o, t, F->p); else memcpy(o, t, 32);
}

static inline int f_is_zero(const u64 a[4]) { return (a[0] | a[1] | a[2] | a[3]) == 0; }
static inline int f_eq(const u64 a[4], const u64 b[4]) { return memcmp(a, b, 32) == 0; }

static void f_pow(const field_t *F, u64 o[4], const u64 a[4], const u64 e[4]) {
    u64 acc[4], base[4];
    memcpy(acc, F->r1, 32);
    memcpy(base, a, 32);
    for (int i = 0; i < 256; ++i) {
        if ((e[i / 64] >> (i % 64)) & 1) f_mul(F, acc, acc, base);
        f_mul(F, base, base, base);
    }
    memcpy(o, acc, 32);
}

static void f_inv(const field_t *F, u64 o[4], const u64 a[4]) {
    u64 e[4], two[4] = {2, 0, 0, 0};
    sub4(e, F->p, two);
    f_pow(F, o, a, e);
}

/* ---- exported field helpers (sel: 0 = Fr, 1 = Fq) -------------------------------- */
static const field_t *pick(int sel) { return sel ? &FQ : &FR; }

void orc_f_add(int sel, u64 *o, const u64 *a, const u64 *b) { f_add(pick(sel), o, a, b); }
void orc_f_sub(int sel, u64 *o, const u64 *a, const u64 *b) { f_sub(pick(sel), o, a, b); }
void orc_f_mul(int sel, u64 *o, const u64 *a, const u64 *b) { f_mul(pick(sel), o, a, b); }
void orc_f_neg(int sel, u64 *o, const u64 *a) { f_neg(pick(sel), o, a); }
void orc_f_inv(int sel, u64 *o, const u64 *a) { f_inv(pick(sel), o, a); }
/* canonical integer limbs -> Montgomery limbs and back */
void orc_f_to_mont(int sel, u64 *o, const u64 *a) { f_mul(pick(sel), o, a, pick(sel)->r2); }
void orc_f_from_mont(int sel, u64 *o, const u64 *a) {
    static const u64 one[4] = {1, 0, 0, 0};
    f_mul(pick(sel), o, a, one);
}

/* element-wise vector ops (bn254_differential.rs:75-99 mirrored at scale); op: 0 add 1 sub 2 mul */
void orc_f_vec(int sel, int op, u64 *o, const u64 *a, const u64 *b, size_t n) {
    const field_t *F = pick(sel);
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) {
        if (op == 0) f_add(F, o + 4 * i, a + 4 * i, b + 4 * i);
        else if (op == 1) f_sub(F, o + 4 * i, a + 4 * i, b + 4 * i);
        else f_mul(F, o + 4 * i, a + 4 * i, b + 4 * i);
    }
}

int orc_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ---- bind (crates/jolt-poly/src/dense.rs:188-263) ---------------------------------
 * order 0 = HighToLow: out[i] = e[i] + s*(e[i+half]-e[i]);
 * order 1 = LowToHigh: out[i] = e[2i] + s*(e[2i+1]-e[2i]). out may alias in for order 0
 * (the reference binds HighToLow in place, :196-199). threads<=1 -> serial loop. */
void orc_bind(u64 *out, const u64 *in, size_t n, const u64 s[4], int order, int threads) {
    size_t half = n / 2;
    (void)threads;
#pragma omp parallel for schedule(static, 1024) if (threads > 1 && half >= 1024) num_threads(threads > 1 ? threads : 1)
    for (size_t i = 0; i < half; ++i) {
        const u64 *lo = order == 0 ? in + 4 * i : in + 8 * i;
        const u64 *hi = order == 0 ? in + 4 * (i + half) : in + 8 * i + 4;
        u64 d[4], m[4], l[4];
        memcpy(l, lo, 32);
        f_sub(&FR, d, hi, l);
        f_mul(&FR, m, s, d);
        f_add(&FR, out + 4 * i, l, m);
    }
}

/* ---- eq table (crates/jolt-poly/src/eq.rs:299-315), r[0] <-> MSB -------------------- */
void orc_eq_evals(u64 *out, const u64 *r, int nvars, const u64 *scale_or_null) {
    size_t N = (size_t)1 << nvars;
    const u64 *sc = scale_or_null ? scale_or_null : FR.r1;
    for (size_t i = 0; i < N; ++i) memcpy(out + 4 * i, sc, 32);
    size_t size = 1;
    for (int j = 0; j < nvars; ++j) {
        size *= 2;
        for (size_t i = size - 1; i >= 1; i -= 2) {
            u64 scalar[4];
            memcpy(scalar, out + 4 * (i / 2), 32);
            f_mul(&FR, out + 4 * i, scalar, r + 4 * j);
            f_sub(&FR, out + 4 * (i - 1), scalar, out + 4 * i);
            if (i == 1) break;
        }
    }
}

/* Parallel eq for the CPU baseline: same values; top `split` variables expanded serially,
 * each prefix's suffix block expanded independently (eq.rs:238-263 decomposition). */
void orc_eq_evals_par(u64 *out, const u64 *r, int nvars, const u64 *scale_or_null, int threads) {
    int split = nvars > 10 ? 6 : 0;
    if (threads <= 1 || split == 0) { orc_eq_evals(out, r, nvars, scale_or_null); return; }
    size_t P = (size_t)1 << split;
    u64 *prefix = (u64 *)malloc(P * 32);
    orc_eq_evals(prefix, r, split, scale_or_null);
    size_t block = (size_t)1 << (nvars - split);
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
    for (size_t b = 0; b < P; ++b) orc_eq_evals(out + 4 * b * block, r + 4 * split, nvars - split, prefix + 4 * b);
    free(prefix);
}

/* ---- univariate-evaluation sweep (jolt-kernels/src/reference/naive.rs:260-299,
 *      jolt-sumcheck/tests/roundtrip.rs:44-62): s(t) = sum_y prod_j (lo_j + t (hi_j - lo_j)) */
void orc_product_round_evals(u64 *out, const u64 *const *tables, int m, size_t n, int degree, int order,
                             int threads) {
    size_t half = n / 2;
    int nt = threads > 1 ? threads : 1;
    int D = degree + 1;
    u64 *partial = (u64 *)calloc((size_t)nt * D * 4, 8);
#pragma omp parallel num_threads(nt)
    {
#ifdef _OPENMP
        int tid = omp_get_thread_num();
#else
        int tid = 0;
#endif
        u64 *acc = partial + (size_t)tid * D * 4;
#pragma omp for schedule(static)
        for (size_t y = 0; y < half; ++y) {
            u64 cur[8][4], dlt[8][4];
            for (int j = 0; j < m; ++j) {
                const u64 *lo = order == 0 ? tables[j] + 4 * y : tables[j] + 8 * y;
                const u64 *hi = order == 0 ? tables[j] + 4 * (y + half) : tables[j] + 8 * y + 4;
                memcpy(cur[j], lo, 32);
                f_sub(&FR, dlt[j], hi, lo);
            }
            for (int t = 0; t < D; ++t) {
                u64 prod[4];
                memcpy(prod, cur[0], 32);
                for (int j = 1; j < m; ++j) f_mul(&FR, prod, prod, cur[j]);
                f_add(&FR, acc + 4 * t, acc + 4 * t, prod);
                for (int j = 0; j < m; ++j) f_add(&FR, cur[j], cur[j], dlt[j]);
            }
        }
    }
    memset(out, 0, (size_t)D * 32);
    for (int t = 0; t < nt; ++t)
        for (int k = 0; k < D; ++k) f_add(&FR, out + 4 * k, out + 4 * k, partial + ((size_t)t * D + k) * 4);
    free(partial);
}

/* ---- BN254 G1, Jacobian over Fq (Montgomery). Identity: Z == 0. -------------------- */
typedef struct { u64 x[4], y[4], z[4]; } jac_t;

static void jac_set_inf(jac_t *p) { memset(p, 0, sizeof *p); memcpy(p->x, FQ.r1, 32); memcpy(p->y, FQ.r1, 32); }
static int jac_is_inf(const jac_t *p) { return f_is_zero(p->z); }

static void jac_double(jac_t *o, const jac_t *p) {
    if (jac_is_inf(p)) { *o = *p; return; }
    u64 a[4], b[4], c[4], d[4], e[4], f[4], t[4], x3[4], y3[4], z3[4];
    f_mul(&FQ, a, p->x, p->x);
    f_mul(&FQ, b, p->y, p->y);
    f_mul(&FQ, c, b, b);
    f_add(&FQ, t, p->x, b);
    f_mul(&FQ, t, t, t);
    f_sub(&FQ, t, t, a);
    f_sub(&FQ, t, t, c);
    f_add(&FQ, d, t, t);
    f_add(&FQ, e, a, a);
    f_add(&FQ, e, e, a);
    f_mul(&FQ, f, e, e);
    f_sub(&FQ, x3, f, d);
    f_sub(&FQ, x3, x3, d);
    f_mul(&FQ, z3, p->y, p->z);
    f_add(&FQ, z3, z3, z3);
    f_sub(&FQ, t, d, x3);
    f_mul(&FQ, y3, e, t);
    f_add(&FQ, c, c, c);
    f_add(&FQ, c, c, c);
    f_add(&FQ, c, c, c);
    f_sub(&FQ, y3, y3, c);
    memcpy(o->x, x3, 32); memcpy(o->y, y3, 32); memcpy(o->z, z3, 32);
}

/* mixed add: Jacobian + affine (ax, ay); handles P == Q and P == -Q explicitly. */
static void jac_add_affine(jac_t *o, const jac_t *p, const u64 ax[4], const u64 ay[4]) {
    if (jac_is_inf(p)) {
        memcpy(o->x, ax, 32); memcpy(o->y, ay, 32); memcpy(o->z, FQ.r1, 32);
        return;
    }
    u64 z2[4], u2[4], s2[4], h[4], rr[4], h2[4], h3[4], v[4], t[4], x3[4], y3[4], z3[4];
    f_mul(&FQ, z2, p->z, p->z);
    f_mul(&FQ, u2, ax, z2);
    f_mul(&FQ, s2, ay, p->z);
    f_mul(&FQ, s2, s2, z2);
    f_sub(&FQ, h, u2, p->x);
    f_sub(&FQ, rr, s2, p->y);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) { jac_double(o, p); return; }
        jac_set_inf(o); memset(o->z, 0, 32);
        return;
    }
    f_mul(&FQ, h2, h, h);
    f_mul(&FQ, h3, h2, h);
    f_mul(&FQ, v, p->x, h2);
    f_mul(&FQ, x3, rr, rr);
    f_sub(&FQ, x3, x3, h3);
    f_sub(&FQ, x3, x3, v);
    f_sub(&FQ, x3, x3, v);
    f_sub(&FQ, t, v, x3);
    f_mul(&FQ, y3, rr, t);
    f_mul(&FQ, t, p->y, h3);
    f_sub(&FQ, y3, y3, t);
    f_mul(&FQ, z3, p->z, h);
    memcpy(o->x, x3, 32); memcpy(o->y, y3, 32); memcpy(o->z, z3, 32);
}

static void jac_add(jac_t *o, const jac_t *p, const jac_t *q) {
    if (jac_is_inf(p)) { *o = *q; return; }
    if (jac_is_inf(q)) { *o = *p; return; }
    u64 z1z1[4], z2z2[4], u1[4], u2[4], s1[4], s2[4], h[4], rr[4], h2[4], h3[4], v[4], t[4], x3[4], y3[4], z3[4];
    f_mul(&FQ, z1z1, p->z, p->z);
    f_mul(&FQ, z2z2, q->z, q->z);
    f_mul(&FQ, u1, p->x, z2z2);
    f_mul(&FQ, u2, q->x, z1z1);
    f_mul(&FQ, s1, p->y, q->z); f_mul(&FQ, s1, s1, z2z2);
    f_mul(&FQ, s2, q->y, p->z); f_mul(&FQ, s2, s2, z1z1);
    f_sub(&FQ, h, u2, u1);
    f_sub(&FQ, rr, s2, s1);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) { jac_double(o, p); return; }
        jac_set_inf(o); memset(o->z, 0, 32);
        return;
    }
    f_mul(&FQ, h2, h, h);
    f_mul(&FQ, h3, h2, h);
    f_mul(&FQ, v, u1, h2);
    f_mul(&FQ, x3, rr, rr);
    f_sub(&FQ, x3, x3, h3);
    f_sub(&FQ, x3, x3, v);
    f_sub(&FQ, x3, x3, v);
    f_sub(&FQ, t, v, x3);
    f_mul(&FQ, y3, rr, t);
    f_mul(&FQ, t, s1, h3);
    f_sub(&FQ, y3, y3, t);
    f_mul(&FQ, z3, p->z, q->z);
    f_mul(&FQ, z3, z3, h);
    memcpy(o->x, x3, 32); memcpy(o->y, y3, 32); memcpy(o->z, z3, 32);
}

/* Jacobian -> affine (x, y) Montgomery limbs; returns 1 if identity (out zeroed). */
static int jac_to_affine(u64 out_xy[8], const jac_t *p) {
    if (jac_is_inf(p)) { memset(out_xy, 0, 64); return 1; }
    u64 zi[4], zi2[4], zi3[4];
    f_inv(&FQ, zi, p->z);
    f_mul(&FQ, zi2, zi, zi);
    f_mul(&FQ, zi3, zi2, zi);
    f_mul(&FQ, out_xy, p->x, zi2);
    f_mul(&FQ, out_xy + 4, p->y, zi3);
    return 0;
}

/* affine bases are 8 x u64 (x, y) Montgomery; the identity is encoded as x = y = 0
 * (not on the curve since b = 3), matching the product's C ABI (include/jolt_b200.h). */
static int aff_is_inf(const u64 *b) { return f_is_zero(b) && f_is_zero(b + 4); }

/* out = k * base, k given as a canonical 4-limb integer. */
static void jac_scalar_mul_affine(jac_t *o, const u64 *base, const u64 k[4]) {
    jac_t acc;
    jac_set_inf(&acc); memset(acc.z, 0, 32);
    if (aff_is_inf(base)) { *o = acc; return; }
    for (int i = 255; i >= 0; --i) {
        jac_double(&acc, &acc);
        if ((k[i / 64] >> (i % 64)) & 1) jac_add_affine(&acc, &acc, base, base + 4);
    }
    *o = acc;
}

int orc_g1_scalar_mul(u64 out_xy[8], const u64 base_xy[8], const u64 scalar_mont[4]) {
    u64 k[4];
    orc_f_from_mont(0, k, scalar_mont);
    jac_t r;
    jac_scalar_mul_affine(&r, base_xy, k);
    return jac_to_affine(out_xy, &r);
}

int orc_g1_add(u64 out_xy[8], const u64 a_xy[8], const u64 b_xy[8]) {
    jac_t p;
    jac_set_inf(&p); memset(p.z, 0, 32);
    if (!aff_is_inf(a_xy)) jac_add_affine(&p, &p, a_xy, a_xy + 4);
    if (!aff_is_inf(b_xy)) jac_add_affine(&p, &p, b_xy, b_xy + 4);
    return jac_to_affine(out_xy, &p);
}

int orc_g1_on_curve(const u64 xy[8]) {
    if (aff_is_inf(xy)) return 1;
    u64 y2[4], x3[4], three[4] = {3, 0, 0, 0}, b[4];
    orc_f_to_mont(1, b, three);
    f_mul(&FQ, y2, xy + 4, xy + 4);
    f_mul(&FQ, x3, xy, xy);
    f_mul(&FQ, x3, x3, xy);
    f_add(&FQ, x3, x3, b);
    return f_eq(y2, x3);
}

/* SRS-like bases: out[i] = beta^i * g  (jolt-hyperkzg/src/scheme.rs:54-73), affine. */
void orc_g1_powers(u64 *out_xy, size_t n, const u64 g_xy[8], const u64 beta_mont[4]) {
    u64 k[4];
    orc_f_from_mont(0, k, beta_mont);
    u64 cur[8];
    memcpy(cur, g_xy, 64);
    for (size_t i = 0; i < n; ++i) {
        memcpy(out_xy + 8 * i, cur, 64);
        jac_t r;
        jac_scalar_mul_affine(&r, cur, k);
        jac_to_affine(cur, &r);
    }
}

/* The same powers, fast enough for 2^24 points: tau^i on the host, then each tau^i * g as a sum of
 * one precomputed multiple per c-bit window of tau^i (a fixed-base table of g: table[w][d - 1] =
 * d * 2^(c w) * g, affine), mixed additions in parallel, and one inversion per chunk of points
 * (Montgomery's batch trick) back to affine. Identity points (tau = 0) come out as x = y = 0. */
#define POW_CHUNK 1024

/* Jacobian -> affine for m points with one inversion; identities (Z = 0) become x = y = 0. */
static void jac_batch_to_affine(u64 *out_xy, const jac_t *p, size_t m, u64 (*scratch)[4]) {
    u64 acc[4];
    memcpy(acc, FQ.r1, 32);
    for (size_t i = 0; i < m; ++i) {  /* scratch[i] = prod of the non-zero Z's before i */
        memcpy(scratch[i], acc, 32);
        if (!jac_is_inf(&p[i])) f_mul(&FQ, acc, acc, p[i].z);
    }
    u64 inv[4];
    f_inv(&FQ, inv, acc);
    for (size_t i = m; i-- > 0;) {
        if (jac_is_inf(&p[i])) { memset(out_xy + 8 * i, 0, 64); continue; }
        u64 zi[4], zi2[4], zi3[4];
        f_mul(&FQ, zi, inv, scratch[i]);
        f_mul(&FQ, inv, inv, p[i].z);
        f_mul(&FQ, zi2, zi, zi);
        f_mul(&FQ, zi3, zi2, zi);
        f_mul(&FQ, out_xy + 8 * i, p[i].x, zi2);
        f_mul(&FQ, out_xy + 8 * i + 4, p[i].y, zi3);
    }
}

static u64 window_digit(const u64 k[4], int bit, int c) {
    int limb = bit / 64, off = bit % 64;
    u64 d = k[limb] >> off;
    if (off + c > 64 && limb < 3) d |= k[limb + 1] << (64 - off);
    return d & (((u64)1 << c) - 1);
}

void orc_g1_powers_fast(u64 *out_xy, size_t n, const u64 g_xy[8], const u64 tau_mont[4], int threads) {
    if (n == 0) return;
    const int nt = threads > 1 ? threads : 1;
    const int c = n >= ((size_t)1 << 16) ? 16 : 8;
    const int nwin = (254 + c - 1) / c;
    const size_t nd = ((size_t)1 << c) - 1;
    /* the table: window w starts from 2^(c w) * g and adds it nd - 1 times */
    u64 *table = (u64 *)malloc((size_t)nwin * nd * 64);
    jac_t base;
    jac_set_inf(&base); memset(base.z, 0, 32);
    jac_add_affine(&base, &base, g_xy, g_xy + 4);
    u64 *bases = (u64 *)malloc((size_t)nwin * 64);
    for (int w = 0; w < nwin; ++w) {
        jac_to_affine(bases + 8 * w, &base);
        for (int k = 0; k < c; ++k) jac_double(&base, &base);
    }
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt)
    for (size_t job = 0; job < (size_t)nwin * ((nd + POW_CHUNK - 1) / POW_CHUNK); ++job) {
        const size_t per = (nd + POW_CHUNK - 1) / POW_CHUNK;
        const int w = (int)(job / per);
        const size_t lo = (job % per) * POW_CHUNK, hi = lo + POW_CHUNK < nd ? lo + POW_CHUNK : nd;
        const u64 *b = bases + 8 * w;
        jac_t *pts = (jac_t *)malloc(sizeof(jac_t) * POW_CHUNK);
        u64(*scratch)[4] = malloc(32 * POW_CHUNK);
        u64 k[4] = {lo + 1, 0, 0, 0}, km[4];
        orc_f_to_mont(0, km, k);
        jac_scalar_mul_affine(&pts[0], b, k);  /* (lo + 1) * b, then + b per entry */
        for (size_t d = lo + 1; d < hi; ++d) jac_add_affine(&pts[d - lo], &pts[d - lo - 1], b, b + 4);
        jac_batch_to_affine(table + ((size_t)w * nd + lo) * 8, pts, hi - lo, scratch);
        free(scratch);
        free(pts);
    }
    free(bases);
    /* tau^i: the first power of each chunk by exponentiation, the rest by one multiplication each */
    u64 tau[4];
    memcpy(tau, tau_mont, 32);
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt)
    for (size_t lo = 0; lo < n; lo += POW_CHUNK) {
        const size_t hi = lo + POW_CHUNK < n ? lo + POW_CHUNK : n;
        jac_t *pts = (jac_t *)malloc(sizeof(jac_t) * POW_CHUNK);
        u64(*scratch)[4] = malloc(32 * POW_CHUNK);
        u64 e[4] = {lo, 0, 0, 0}, pw[4];
        f_pow(&FR, pw, tau, e);
        for (size_t i = lo; i < hi; ++i) {
            u64 k[4];
            orc_f_from_mont(0, k, pw);
            jac_t *acc = &pts[i - lo];
            jac_set_inf(acc); memset(acc->z, 0, 32);
            for (int w = 0; w < nwin; ++w) {
                const u64 d = window_digit(k, w * c, c);
                if (d) {
                    const u64 *t = table + ((size_t)w * nd + d - 1) * 8;
                    jac_add_affine(acc, acc, t, t + 4);
                }
            }
            f_mul(&FR, pw, pw, tau);
        }
        jac_batch_to_affine(out_xy + 8 * lo, pts, hi - lo, scratch);
        free(scratch);
        free(pts);
    }
    free(table);
}

/* naive MSM: sum_i s_i * P_i (jolt-crypto/tests/group_laws.rs:69-79). */
int orc_g1_msm_naive(u64 out_xy[8], const u64 *bases_xy, const u64 *scalars_mont, size_t n) {
    jac_t acc;
    jac_set_inf(&acc); memset(acc.z, 0, 32);
    for (size_t i = 0; i < n; ++i) {
        u64 k[4];
        orc_f_from_mont(0, k, scalars_mont + 4 * i);
        jac_t t;
        jac_scalar_mul_affine(&t, bases_xy + 8 * i, k);
        jac_add(&acc, &acc, &t);
    }
    return jac_to_affine(out_xy, &acc);
}

/* Pippenger bucket MSM on canonical scalars (jolt-crypto/src/ec/bn254/mod.rs:195-212 ->
 * ark_ec msm_bigint): window c = 3 if n < 32 else ln(n) + 2; windows processed in
 * parallel (one OpenMP task per window, as arkworks does with Rayon). c <= 0 -> heuristic. */
int orc_g1_msm_pippenger(u64 out_xy[8], const u64 *bases_xy, const u64 *scalars_mont, size_t n, int c,
                         int threads) {
    if (n == 0) { memset(out_xy, 0, 64); return 1; }
    if (c <= 0) c = n < 32 ? 3 : (int)(log((double)n)) + 2;
    int nwin = (254 + c - 1) / c;
    u64 *canon = (u64 *)malloc(n * 32);
#pragma omp parallel for schedule(static) num_threads(threads > 1 ? threads : 1)
    for (size_t i = 0; i < n; ++i) orc_f_from_mont(0, canon + 4 * i, scalars_mont + 4 * i);
    jac_t *wsum = (jac_t *)malloc(sizeof(jac_t) * nwin);
    size_t nb = ((size_t)1 << c) - 1;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 1 ? threads : 1)
    for (int w = 0; w < nwin; ++w) {
        jac_t *buckets = (jac_t *)malloc(sizeof(jac_t) * nb);
        for (size_t b = 0; b < nb; ++b) { jac_set_inf(&buckets[b]); memset(buckets[b].z, 0, 32); }
        int bit = w * c;
        for (size_t i = 0; i < n; ++i) {
            const u64 *k = canon + 4 * i;
            int limb = bit / 64, off = bit % 64;
            u64 d = k[limb] >> off;
            if (off + c > 64 && limb < 3) d |= k[limb + 1] << (64 - off);
            d &= ((u64)1 << c) - 1;
            if (d && !aff_is_inf(bases_xy + 8 * i))
                jac_add_affine(&buckets[d - 1], &buckets[d - 1], bases_xy + 8 * i, bases_xy + 8 * i + 4);
        }
        jac_t run, acc;
        jac_set_inf(&run); memset(run.z, 0, 32);
        acc = run;
        for (size_t b = nb; b-- > 0;) {
            jac_add(&run, &run, &buckets[b]);
            jac_add(&acc, &acc, &run);
        }
        wsum[w] = acc;
        free(buckets);
    }
    jac_t total = wsum[nwin - 1];
    for (int w = nwin - 2; w >= 0; --w) {
        for (int k = 0; k < c; ++k) jac_double(&total, &total);
        jac_add(&total, &total, &wsum[w]);
    }
    free(wsum);
    free(canon);
    return jac_to_affine(out_xy, &total);
}

/* ---- HyperKZG host-side scalar pieces (jolt-hyperkzg/src/kzg.rs:34-59) --------------- */
void orc_witness_polynomial(u64 *h, const u64 *f, size_t d, const u64 u[4]) {
    if (d <= 1) return;
    u64 acc[4] = {0, 0, 0, 0};
    for (size_t i = d - 1; i >= 1; --i) {
        u64 t[4];
        f_mul(&FR, t, acc, u);
        f_add(&FR, acc, f + 4 * i, t);
        memcpy(h + 4 * (i - 1), acc, 32);
    }
}

void orc_eval_univariate(u64 out[4], const u64 *coeffs, size_t n, const u64 u[4]) {
    u64 res[4] = {0, 0, 0, 0}, power[4];
    memcpy(power, FR.r1, 32);
    for (size_t i = 0; i < n; ++i) {
        u64 t[4];
        f_mul(&FR, t, coeffs + 4 * i, power);
        f_add(&FR, res, res, t);
        f_mul(&FR, power, power, u);
    }
    memcpy(out, res, 32);
}
