/* ORACLE (test infrastructure, NOT product code): a threaded C restatement of jb_table_linear_combination on the C
 * oracle's field arithmetic (oracle/oracle.c, included whole), for sizes the big-int reference cannot reach and as the
 * host route tools/lincomb_bench.py times:
 *   P[x] = sum_i c_i p_i[x] for x < len_i (0 beyond), Montgomery product by Montgomery product, no deferred reduction.
 * A term has the layout of jb_lc_term, except that a TABLE term carries host limbs in `values` and its length in
 * `len`. Compact values are promoted as jb_table_upload_small does (F::from(v), negatives r - |v|, -0 = 0); a one-hot
 * term of T = len addresses is the K T polynomial with coefficient (k, j) = 1 iff addr[j] == k. Built and loaded by
 * tests/lincomb_cref.py. */
#include "../../oracle/oracle.c"

typedef struct {
    int type, kind, on_device, layout;
    u64 table;
    const void *values;
    size_t len, K;
    u64 coeff[4];
} lc_term;

/* |v| as two u64 words; returns v < 0 (kinds of include/jolt_b200.h: 1 u8 .. 9 s128) */
static int lc_small(const void *values, size_t i, int kind, u64 mag[2]) {
    const u64 *w = (const u64 *)values;
    int neg = 0;
    mag[0] = mag[1] = 0;
    switch (kind) {
        case 1: mag[0] = ((const uint8_t *)values)[i]; break;
        case 2: mag[0] = ((const uint16_t *)values)[i]; break;
        case 3: mag[0] = ((const uint32_t *)values)[i]; break;
        case 4: mag[0] = w[i]; break;
        case 5: mag[0] = w[2 * i]; mag[1] = w[2 * i + 1]; break;
        case 6: neg = (w[i] >> 63) != 0; mag[0] = neg ? 0 - w[i] : w[i]; break;
        case 7: {
            u128 v = ((u128)w[2 * i + 1] << 64) | w[2 * i];
            neg = (w[2 * i + 1] >> 63) != 0;
            if (neg) v = 0 - v;
            mag[0] = (u64)v;
            mag[1] = (u64)(v >> 64);
            break;
        }
        case 8: mag[0] = w[2 * i]; neg = (w[2 * i + 1] & 0xff) == 0; break;
        case 9: mag[0] = w[3 * i]; mag[1] = w[3 * i + 1]; neg = (w[3 * i + 2] & 0xff) == 0; break;
        default: break;
    }
    if ((mag[0] | mag[1]) == 0) neg = 0;
    return neg;
}

void lc_linear_combination(u64 *out, const lc_term *terms, size_t count, size_t len) {
#pragma omp parallel for schedule(static, 4096)
    for (size_t x = 0; x < len; ++x) {
        u64 acc[4] = {0, 0, 0, 0}, v[4], m[4];
        for (size_t t = 0; t < count; ++t) {
            const lc_term *tm = &terms[t];
            if (tm->type == 0) {
                if (x >= tm->len) continue;
                memcpy(v, (const u64 *)tm->values + 4 * x, 32);
            } else if (tm->type == 1) {
                if (x >= tm->len) continue;
                u64 mag[2], k[4] = {0, 0, 0, 0};
                const int neg = lc_small(tm->values, x, tm->kind, mag);
                k[0] = mag[0];
                k[1] = mag[1];
                f_mul(&FR, v, k, FR.r2);
                if (neg) f_neg(&FR, v, v);
            } else {
                const size_t T = tm->len, K = tm->K;
                if (x >= K * T) continue;
                const size_t j = tm->layout == 0 ? x / K : x % T, k = tm->layout == 0 ? x % K : x / T;
                const u64 a = tm->kind == 1 ? ((const uint8_t *)tm->values)[j] : ((const uint16_t *)tm->values)[j];
                const u64 none = tm->kind == 1 ? 0xff : 0xffff;
                if (a == none || a != k) continue;
                memcpy(v, FR.r1, 32);
            }
            f_mul(&FR, m, tm->coeff, v);
            f_add(&FR, acc, acc, m);
        }
        memcpy(out + 4 * x, acc, 32);
    }
}
