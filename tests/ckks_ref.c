/*
 * ckks_ref.c — C11 restatement of the CKKS slot encoding of DESIGN.md §2.12 (TEST INFRASTRUCTURE ONLY).
 *
 * It shares no code with deeppowers_b200/csrc/: the twiddles are computed on their own (124-bit fixed point, first quadrant),
 * and so are the slot permutation, the exact reduction and the Garner digits.  It works on coefficient-form residues; the
 * transforms of §2.3 around it are the oracle's (tests/ckks_ref.py composes the two).  Built by tests/ckks_ref.py with
 * -ffp-contract=off: every product and sum is rounded on its own, as the specification requires.
 */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;

#define CKR_MAX_L 16

static uint64_t mulmod(uint64_t a, uint64_t b, uint64_t q) { return (uint64_t)(((u128)a * b) % q); }
static uint64_t submod(uint64_t a, uint64_t b, uint64_t q) { return a >= b ? a - b : a + q - b; }
static uint64_t powmod(uint64_t a, uint64_t e, uint64_t q) {
    uint64_t r = 1 % q, b = a % q;
    for (; e; e >>= 1, b = mulmod(b, b, q))
        if (e & 1) r = mulmod(r, b, q);
    return r;
}
static uint32_t bitrev(uint32_t x, unsigned bits) {
    uint32_t r = 0;
    for (unsigned i = 0; i < bits; ++i, x >>= 1) r = (r << 1) | (x & 1);
    return r;
}

/* floor(a * b / 2^124) for a, b < 2^127 with a * b < 2^252 */
static u128 fx124_mul(u128 a, u128 b) {
    const uint64_t al = (uint64_t)a, ah = (uint64_t)(a >> 64), bl = (uint64_t)b, bh = (uint64_t)(b >> 64);
    const u128 ll = (u128)al * bl, lh = (u128)al * bh, hl = (u128)ah * bl, hh = (u128)ah * bh;
    const u128 m = (ll >> 64) + (uint64_t)lh + (uint64_t)hl;       /* bits 64.. of the product */
    const u128 top = hh + (lh >> 64) + (hl >> 64) + (m >> 64);      /* bits 128.. */
    return (top << 4) | ((uint64_t)m >> 60);
}

/* nearest double (ties to even) of v / 2^124, 0 <= v <= 2^124: built from its bits */
static double fx124_round(u128 v) {
    if (!v) return 0.0;
    int top = 0;
    for (u128 t = v; t >>= 1;) ++top;
    uint64_t mant;
    int e2 = top - 124;   /* v / 2^124 in [2^e2, 2^(e2+1)) */
    if (top <= 52) {
        mant = (uint64_t)v << (52 - top);
    } else {
        const int sh = top - 52;
        const u128 rest = v & (((u128)1 << sh) - 1), mid = (u128)1 << (sh - 1);
        mant = (uint64_t)(v >> sh);
        if (rest > mid || (rest == mid && (mant & 1))) ++mant;
        if (mant >> 53) { mant >>= 1; ++e2; }
    }
    const uint64_t bits = ((uint64_t)(e2 + 1023) << 52) | (mant & ((1ull << 52) - 1));
    double d;
    memcpy(&d, &bits, 8);
    return d;
}

/* (cos, sin) of pi a / 2^b, 0 <= a / 2^b < 1/2, by the Taylor series in 124-bit fixed point */
static void cos_sin_fx(uint64_t a, unsigned b, double *c, double *s) {
    const u128 pi124 = ((u128)0x3243F6A8885A308Dull << 64) | 0x313198A2E0370734ull;   /* floor(pi * 2^124) */
    const u128 x = (pi124 >> b) * a + (((pi124 & (((u128)1 << b) - 1)) * a) >> b);
    u128 even = 0, odd = 0, even_neg = 0, odd_neg = 0, term = (u128)1 << 124;
    for (unsigned k = 0; term != 0; ++k) {
        u128 *acc = (k & 1) ? ((k & 2) ? &odd_neg : &odd) : ((k & 2) ? &even_neg : &even);
        *acc += term;
        term = fx124_mul(term, x) / (k + 1);
    }
    *c = fx124_round(even - even_neg);
    *s = fx124_round(odd - odd_neg);
}

/* tw: N pairs (cos, sin)(pi k / N), correctly rounded */
void ckr_twiddles(unsigned logn, double *tw) {
    const uint64_t N = (uint64_t)1 << logn;
    for (uint64_t k = 0; k < N; ++k) {
        double c, s;
        if (k == N / 2) {   /* cos(pi/2) = +0 exactly; the series would leave the truncation error of pi */
            c = 0.0;
            s = 1.0;
        } else if (k < N / 2) {
            cos_sin_fx(k, logn, &c, &s);
        } else {   /* angle pi - pi (N - k) / N */
            cos_sin_fx(N - k, logn, &c, &s);
            c = -c;
        }
        tw[2 * k] = c;
        tw[2 * k + 1] = s;
    }
}

typedef struct { double re, im; } cplx;

static cplx cx_mul(cplx a, cplx b) {
    cplx r;
    r.re = a.re * b.re - a.im * b.im;
    r.im = a.re * b.im + a.im * b.re;
    return r;
}

/* slot j is the value at exp(i pi e_j / N), e_j = 5^j mod 2N = 4 t_j + 1: the DFT output t_j */
static void slot_table(uint32_t *tj, uint64_t N) {
    uint64_t e = 1;
    for (uint64_t j = 0; j < N / 2; ++j, e = e * 5 % (2 * N)) tj[j] = (uint32_t)((e - 1) / 4);
}

/* radix-2 decimation in time over S = N/2 points, input bit-reversed: a[t] <- sum_k a[k] W^(+-tk), W = tw[4] */
static void special_fft(cplx *a, const cplx *tw, unsigned logn, int inverse) {
    const size_t S = (size_t)1 << (logn - 1);
    for (unsigned s = 0; (size_t)1 << s < S; ++s) {
        const size_t h = (size_t)1 << s;
        for (size_t blk = 0; blk < S; blk += 2 * h)
            for (size_t j = 0; j < h; ++j) {
                cplx w = tw[j << (logn - s)];
                if (inverse) w.im = -w.im;
                const cplx x = a[blk + j], y = cx_mul(a[blk + j + h], w);
                a[blk + j].re = x.re + y.re;
                a[blk + j].im = x.im + y.im;
                a[blk + j + h].re = x.re - y.re;
                a[blk + j + h].im = x.im - y.im;
            }
    }
}

/* x mod q for an integral double x = +-M 2^e, |M| < 2^53 */
static uint64_t double_mod(double x, uint64_t q) {
    uint64_t b;
    memcpy(&b, &x, 8);
    const int ex = (int)((b >> 52) & 0x7ff);
    uint64_t m = b & ((1ull << 52) - 1);
    int e;
    if (ex) { m |= 1ull << 52; e = ex - 1075; } else { e = -1074; }
    uint64_t r;
    if (e >= 0) r = mulmod(m % q, powmod(2, (uint64_t)e, q), q);
    else r = (e > -64 ? m >> -e : 0) % q;
    return (b >> 63) && r ? q - r : r;
}

/* slots [n_vec][N/2][2] -> res [n_vec][L][N]: the rounded coefficients reduced into every limb (coefficient form);
 * coeffs (may be NULL): the rounded coefficients [n_vec][N] themselves */
void ckr_encode(unsigned logn, unsigned L, const uint64_t *q, const double *slots, size_t n_vec, double scale, uint64_t *res, double *coeffs) {
    const size_t N = (size_t)1 << logn, S = N / 2;
    cplx *tw = malloc(N * sizeof(cplx)), *a = malloc(S * sizeof(cplx));
    uint32_t *tj = malloc(S * sizeof(uint32_t));
    double *x = malloc(N * sizeof(double));
    ckr_twiddles(logn, (double *)tw);
    slot_table(tj, N);
    const double sc = scale * (2.0 / (double)N);
    for (size_t v = 0; v < n_vec; ++v) {
        const cplx *z = (const cplx *)(slots + v * N);
        for (size_t j = 0; j < S; ++j) a[bitrev(tj[j], logn - 1)] = z[j];
        special_fft(a, tw, logn, 1);
        for (size_t k = 0; k < S; ++k) {
            cplx w = tw[k];
            w.im = -w.im;
            const cplx u = cx_mul(a[k], w);
            x[k] = __builtin_rint(sc * u.re);
            x[k + S] = __builtin_rint(sc * u.im);
        }
        if (coeffs) memcpy(coeffs + v * N, x, N * sizeof(double));
        for (unsigned l = 0; l < L; ++l)
            for (size_t k = 0; k < N; ++k) res[(v * L + l) * N + k] = double_mod(x[k], q[l]);
    }
    free(tw); free(a); free(tj); free(x);
}

/* res [n_vec][L][N] canonical coefficient-form residues -> slots [n_vec][N/2][2] */
void ckr_decode(unsigned logn, unsigned L, const uint64_t *q, const uint64_t *res, size_t n_vec, double scale, double *slots) {
    const size_t N = (size_t)1 << logn, S = N / 2;
    cplx *tw = malloc(N * sizeof(cplx)), *a = malloc(S * sizeof(cplx));
    uint32_t *tj = malloc(S * sizeof(uint32_t));
    double *cf = malloc(N * sizeof(double));
    ckr_twiddles(logn, (double *)tw);
    slot_table(tj, N);
    /* digits of (Q - 1) / 2 */
    uint64_t half[CKR_MAX_L], rem = 0;
    for (unsigned i = L; i-- > 0;) {
        const u128 t = (u128)rem * q[i] + (q[i] - 1);
        half[i] = (uint64_t)(t / 2);
        rem = (uint64_t)(t % 2);
    }
    uint64_t ginv[CKR_MAX_L][CKR_MAX_L];   /* [j][i] q_j^-1 mod q_i */
    for (unsigned i = 0; i < L; ++i)
        for (unsigned j = 0; j < i; ++j) ginv[j][i] = powmod(q[j] % q[i], q[i] - 2, q[i]);
    for (size_t v = 0; v < n_vec; ++v) {
        const uint64_t *poly = res + v * L * N;
        for (size_t k = 0; k < N; ++k) {
            uint64_t d[CKR_MAX_L];
            for (unsigned i = 0; i < L; ++i) {   /* Garner: X = d_0 + d_1 q_0 + d_2 q_0 q_1 + ... */
                uint64_t t = poly[i * N + k];
                for (unsigned j = 0; j < i; ++j) t = mulmod(submod(t, d[j] % q[i], q[i]), ginv[j][i], q[i]);
                d[i] = t;
            }
            int above = 0;
            for (unsigned i = L; i-- > 0;)
                if (d[i] != half[i]) { above = d[i] > half[i]; break; }
            if (above) {   /* Q - X, digit by digit */
                unsigned i = 0;
                for (; d[i] == 0; ++i) {}
                d[i] = q[i] - d[i];
                for (++i; i < L; ++i) d[i] = q[i] - 1 - d[i];
            }
            double r = (double)d[L - 1];
            for (unsigned i = L - 1; i-- > 0;) r = r * (double)q[i] + (double)d[i];
            cf[k] = (above ? -r : r) / scale;
        }
        for (size_t k = 0; k < S; ++k) {
            const cplx u = {cf[k], cf[k + S]};
            a[bitrev((uint32_t)k, logn - 1)] = cx_mul(u, tw[k]);
        }
        special_fft(a, tw, logn, 0);
        cplx *z = (cplx *)(slots + v * N);
        for (size_t j = 0; j < S; ++j) z[j] = a[tj[j]];
    }
    free(tw); free(a); free(tj); free(cf);
}
