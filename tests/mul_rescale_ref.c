/* mul_rescale_ref.c — multiply-and-rescale of DESIGN.md §2.19 restated on the oracle (TEST INFRASTRUCTURE ONLY).
 *
 * Compiles the oracle's own translation unit in (its tensor product over a limb prefix, its mod-up and its helpers are static
 * there) and writes the definition out step by step:
 *     D_c   = sum_t ct_tensor(a_t, b_t)_c                     c = 0, 1, 2, over the Lq ciphertext moduli
 *     acc_c = P * D_c on the Lq ciphertext rows (0 on the special rows) + sum_g U_g o evk[g][c]     over all L limbs, exact mod q_i
 *     out   = dpo_mod_down_special(K + 1, acc, t_plain)       the last K + 1 limbs {q_{Lq-1}, p_0 .. p_{K-1}} divided out
 * Shares no code with deeppowers_b200/csrc.  Built into tests/_emu/ by tests/mul_rescale_ref.py. */
#include "../oracle/dpfhe_oracle.c"

/* acc [2][L][N] of one output ciphertext; a, b: the n_terms operands of this ciphertext, pair t at a + t * stride */
static void msr_acc_one(const dpo_ctx *c, unsigned K, size_t n_terms, const uint64_t *a, const uint64_t *b, size_t stride, const uint64_t *evk,
                        uint64_t *acc) {
    const unsigned L = c->L, Lq = L - K, dnum = dpo_grouped_digits(c, K);
    const size_t N = c->N, P = (size_t)Lq * N, PK = (size_t)L * N;
    uint64_t *D = (uint64_t *)calloc(3 * P, 8), *d = (uint64_t *)malloc(3 * P * 8), *U = (uint64_t *)malloc((size_t)dnum * PK * 8);
    for (size_t t = 0; t < n_terms; t++) {
        ct_tensor_limbs(c, Lq, a + t * stride, b + t * stride, d);
        for (unsigned k = 0; k < 3; k++)
            for (unsigned l = 0; l < Lq; l++)
                for (size_t n = 0; n < N; n++) {
                    const size_t o = k * P + l * N + n;
                    D[o] = addmod(D[o], d[o], c->q[l]);
                }
    }
    grouped_mod_up(c, K, D + 2 * P, U);
    memset(acc, 0, 2 * PK * 8);
    for (unsigned g = 0; g < dnum; g++)
        for (unsigned i = 0; i < L; i++) {
            const uint64_t q = c->q[i], r0 = c->br0[i], r1 = c->br1[i];
            const uint64_t *u = U + ((size_t)g * L + i) * N;
            const uint64_t *kb = evk + ((size_t)g * 2 + 0) * PK + i * N, *ka = evk + ((size_t)g * 2 + 1) * PK + i * N;
            for (size_t n = 0; n < N; n++) {
                acc[i * N + n] = addmod(acc[i * N + n], barrett_mul(u[n], kb[n], q, r0, r1), q);
                acc[PK + i * N + n] = addmod(acc[PK + i * N + n], barrett_mul(u[n], ka[n], q, r0, r1), q);
            }
        }
    for (unsigned i = 0; i < Lq; i++) {
        const uint64_t q = c->q[i], Pm = prod_mod(c, Lq, L, L, q);
        for (size_t n = 0; n < N; n++) {
            acc[i * N + n] = addmod(acc[i * N + n], mulmod(D[i * N + n], Pm, q), q);
            acc[PK + i * N + n] = addmod(acc[PK + i * N + n], mulmod(D[P + i * N + n], Pm, q), q);
        }
    }
    free(D); free(d); free(U);
}

/* a, b: [n_terms][batch][2][Lq][N]; evk: [dnum][2][L][N].  want_acc = 0: out [batch][2][Lq-1][N], the result; want_acc = 1: out
 * [batch][2][L][N], the accumulator before the division (the tests check the division against integers). */
int msr_mul_rescale(unsigned logn, unsigned L, const uint64_t *moduli, unsigned K, size_t n_terms, const uint64_t *a, const uint64_t *b,
                    const uint64_t *evk, uint64_t t_plain, uint64_t *out, size_t batch, int want_acc) {
    dpo_ctx *c = dpo_create(logn, L, moduli);
    if (!c) return -1;
    if (K < 1 || 2 * K > L || L - K < 2 || n_terms < 1) {
        dpo_destroy(c);
        return -1;
    }
    const unsigned Lq = L - K;
    const size_t N = c->N, P = (size_t)Lq * N, PK = (size_t)L * N;
#pragma omp parallel for schedule(dynamic, 1)
    for (long i = 0; i < (long)batch; i++) {
        uint64_t *acc = want_acc ? out + (size_t)i * 2 * PK : (uint64_t *)malloc(2 * PK * 8);
        msr_acc_one(c, K, n_terms, a + (size_t)i * 2 * P, b + (size_t)i * 2 * P, batch * 2 * P, evk, acc);
        if (!want_acc) {
            dpo_mod_down_special(c, K + 1, acc, t_plain, out + (size_t)i * 2 * (P - N), 2);
            free(acc);
        }
    }
    dpo_destroy(c);
    return 0;
}
