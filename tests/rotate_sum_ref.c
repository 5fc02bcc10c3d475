/* rotate_sum_ref.c — the summed rotations of DESIGN.md §2.17 restated on the oracle (TEST INFRASTRUCTURE ONLY).
 *
 * Compiles the oracle's own translation unit in (its mod-up and its division by P are static there) and adds the one new
 * step, the summed multiply-accumulate:
 *     acc   = sum_m sum_g perm_m(U_g) o gk_m[g]            over all L limbs, c = 0 and 1, exact mod q_i
 *     (k0, k1) = dpo_mod_down_special(acc, t_plain)
 *     out   = (c0 + sum_m perm_m(c0) + k0,  c1 + k1)
 * The carried terms are added after the division, not carried through it as the kernel does (the same bits, DESIGN.md §2.17).
 * Shares no code with deeppowers_b200/csrc.  Built into tests/_emu/ by tests/rotate_sum_ref.py. */
#include "../oracle/dpfhe_oracle.c"

/* ct, out: [batch][2][Lq][N]; gks: [n_rot][dnum][2][L][N]; galois: [n_rot].  mode 1 drops the carried c1 term (a deliberately
 * wrong variant the tests tell apart). */
int rsr_rotate_sum_grouped(unsigned logn, unsigned L, const uint64_t *moduli, unsigned K, const uint64_t *ct, size_t n_rot, const uint64_t *galois,
                           const uint64_t *gks, uint64_t t_plain, uint64_t *out, size_t batch, int mode) {
    dpo_ctx *c = dpo_create(logn, L, moduli);
    if (!c) return -1;
    if (K < 1 || 2 * K > L || n_rot < 1) {
        dpo_destroy(c);
        return -1;
    }
    const unsigned Lq = L - K, dnum = dpo_grouped_digits(c, K);
    const size_t N = c->N, P = (size_t)Lq * N, PK = (size_t)L * N, key_words = (size_t)dnum * 2 * PK;
    uint32_t *perm = (uint32_t *)malloc(n_rot * N * 4);
    for (size_t r = 0; r < n_rot; r++) dpo_galois_perm(c, galois[r], perm + r * N);
#pragma omp parallel for schedule(dynamic, 1)
    for (long b = 0; b < (long)batch; b++) {
        const uint64_t *src = ct + 2 * P * b;
        uint64_t *dst = out + 2 * P * b;
        uint64_t *U = (uint64_t *)malloc((size_t)dnum * PK * 8), *acc = (uint64_t *)calloc(2 * PK, 8), *k = (uint64_t *)malloc(2 * P * 8);
        grouped_mod_up(c, K, src + P, U);
        for (size_t r = 0; r < n_rot; r++) {
            const uint32_t *pr = perm + r * N;
            const uint64_t *key = gks + r * key_words;
            for (unsigned g = 0; g < dnum; g++)
                for (unsigned i = 0; i < L; i++) {
                    const uint64_t q = c->q[i], r0 = c->br0[i], r1 = c->br1[i];
                    const uint64_t *u = U + ((size_t)g * L + i) * N;
                    const uint64_t *kb = key + ((size_t)g * 2 + 0) * PK + i * N, *ka = key + ((size_t)g * 2 + 1) * PK + i * N;
                    for (size_t n = 0; n < N; n++) {
                        acc[i * N + n] = addmod(acc[i * N + n], barrett_mul(u[pr[n]], kb[n], q, r0, r1), q);
                        acc[PK + i * N + n] = addmod(acc[PK + i * N + n], barrett_mul(u[pr[n]], ka[n], q, r0, r1), q);
                    }
                }
        }
        dpo_mod_down_special(c, K, acc, t_plain, k, 2);
        for (unsigned l = 0; l < Lq; l++) {
            const uint64_t q = c->q[l];
            for (size_t n = 0; n < N; n++) {
                const size_t o = l * N + n;
                uint64_t s = addmod(src[o], k[o], q);
                for (size_t r = 0; r < n_rot; r++) s = addmod(s, src[l * N + perm[r * N + n]], q);
                dst[o] = s;
                dst[P + o] = mode == 1 ? k[P + o] : addmod(src[P + o], k[P + o], q);
            }
        }
        free(U); free(acc); free(k);
    }
    free(perm);
    dpo_destroy(c);
    return 0;
}
