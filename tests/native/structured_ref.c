/* ORACLE (test infrastructure, NOT product code): threaded C builds of the LT and eq+1 tables on the C oracle's field
 * arithmetic (oracle/oracle.c, included whole), for sizes the big-int reference cannot reach and as the host route
 * tools/structured_bench.py times. Both start from the eq table E = orc_eq_evals_par(r, scale):
 *   LT[j] = sum_{t > j} E[t]: a suffix sum, per chunk in parallel, then each chunk offset by the sum of the chunks
 *           after it;
 *   E1[j] = E[j - 1], E1[0] = 0.
 * Built and loaded by tests/structured_ref.py. */
#include "../../oracle/oracle.c"

void orc_lt_evals(u64 *out, const u64 *r, int nvars, const u64 *scale_or_null, int threads) {
    size_t N = (size_t)1 << nvars;
    orc_eq_evals_par(out, r, nvars, scale_or_null, threads);
    size_t chunks = threads > 1 && N >= 4096 ? (size_t)threads * 4 : 1;
    size_t len = (N + chunks - 1) / chunks;
    u64 *tot = (u64 *)calloc(chunks + 1, 32);
    /* in place: out[j] <- the sum of the chunk's entries after j; tot[c] <- the chunk's whole sum */
#pragma omp parallel for schedule(static, 1) num_threads(threads > 1 ? threads : 1)
    for (size_t c = 0; c < chunks; ++c) {
        size_t lo = c * len, hi = lo + len < N ? lo + len : N;
        u64 acc[4] = {0, 0, 0, 0}, e[4];
        for (size_t j = hi; j-- > lo;) {
            memcpy(e, out + 4 * j, 32);
            memcpy(out + 4 * j, acc, 32);
            f_add(&FR, acc, acc, e);
        }
        memcpy(tot + 4 * c, acc, 32);
    }
    /* tot[c] <- the sum of the chunks after c */
    u64 acc[4] = {0, 0, 0, 0}, e[4];
    for (size_t c = chunks; c-- > 0;) {
        memcpy(e, tot + 4 * c, 32);
        memcpy(tot + 4 * c, acc, 32);
        f_add(&FR, acc, acc, e);
    }
#pragma omp parallel for schedule(static, 1) num_threads(threads > 1 ? threads : 1)
    for (size_t c = 0; c < chunks; ++c) {
        size_t lo = c * len, hi = lo + len < N ? lo + len : N;
        if (f_is_zero(tot + 4 * c)) continue;
        for (size_t j = lo; j < hi; ++j) f_add(&FR, out + 4 * j, out + 4 * j, tot + 4 * c);
    }
    free(tot);
}

void orc_eq_plus_one_evals(u64 *out, const u64 *r, int nvars, const u64 *scale_or_null, int threads) {
    size_t N = (size_t)1 << nvars;
    orc_eq_evals_par(out, r, nvars, scale_or_null, threads);
    memmove(out + 4, out, (N - 1) * 32);
    memset(out, 0, 32);
}
