// host_params.cpp — see host_params.hpp.  Plain C++17, compiled into libdpfhe.so.
#include "host_params.hpp"

namespace dpfhe {

typedef unsigned __int128 u128;

uint64_t host_mulmod(uint64_t a, uint64_t b, uint64_t q) { return (uint64_t)((u128)a * b % q); }

// seed words, the exact uniform reduction (2^64 mod q and its Shoup companion), the noise factor t (1 for t = 0) and the gadget
// factor of the digits (P mod q_l, the product of the last K limbs; 1 for per-limb digits)
KeyArgs build_key_args(const HostParams &hp, const uint8_t seed[32], unsigned K, uint64_t t_plain) {
    KeyArgs A = {};
    for (int i = 0; i < 8; ++i)
        A.seed[i] = (uint32_t)seed[4 * i] | (uint32_t)seed[4 * i + 1] << 8 | (uint32_t)seed[4 * i + 2] << 16 | (uint32_t)seed[4 * i + 3] << 24;
    const unsigned L = hp.L;
    A.K = K;
    A.Lq = L - K;
    A.ndig = K ? (A.Lq + K - 1) / K : L;
    A.pk_a = L << hp.log_n;
    for (unsigned l = 0; l < L; ++l) {
        const uint64_t q = hp.limbs[l].lp.q;
        const uint64_t r64 = (uint64_t)(((u128)1 << 64) % q);
        A.r64[l] = r64;
        A.r64_s[l] = (uint64_t)(((u128)r64 << 64) / q);
        A.tq[l] = t_plain ? t_plain % q : 1;
        uint64_t f = 1 % q;
        for (unsigned k = L - K; k < L; ++k) f = host_mulmod(f, hp.limbs[k].lp.q % q, q);
        A.fac[l] = f;
    }
    return A;
}

uint64_t host_powmod(uint64_t a, uint64_t e, uint64_t q) {
    uint64_t r = 1 % q, base = a % q;
    for (; e; e >>= 1) {
        if (e & 1) r = host_mulmod(r, base, q);
        base = host_mulmod(base, base, q);
    }
    return r;
}

// Miller-Rabin, exact for n < 2^64 with the first twelve prime witnesses.
bool host_is_prime(uint64_t n) {
    const uint64_t small[12] = {2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37};
    if (n < 2) return false;
    for (uint64_t s : small) {
        if (n == s) return true;
        if (n % s == 0) return false;
    }
    uint64_t odd = n - 1;
    int twos = 0;
    while ((odd & 1) == 0) {
        odd >>= 1;
        ++twos;
    }
    for (uint64_t a : small) {
        uint64_t y = host_powmod(a, odd, n);
        if (y == 1 || y == n - 1) continue;
        bool witness = true;
        for (int r = 1; r < twos && witness; ++r) {
            y = host_mulmod(y, y, n);
            if (y == n - 1) witness = false;
        }
        if (witness) return false;
    }
    return true;
}

static uint32_t rev_bits(uint32_t v, unsigned bits) {
    uint32_t r = 0;
    for (unsigned k = 0; k < bits; ++k) r |= ((v >> k) & 1u) << (bits - 1 - k);
    return r;
}

static uint64_t shoup_of(uint64_t w, uint64_t q) { return (uint64_t)(((u128)w << 64) / q); }

// smallest primitive 2N-th root of unity: find one, then scan its odd powers.
static uint64_t min_primitive_root(uint64_t q, uint64_t two_n) {
    const uint64_t cofactor = (q - 1) / two_n;
    uint64_t any = 0;
    for (uint64_t g = 2; !any; ++g) {
        uint64_t cand = host_powmod(g, cofactor, q);
        if (host_powmod(cand, two_n >> 1, q) == q - 1) any = cand;
    }
    const uint64_t step = host_mulmod(any, any, q);
    uint64_t least = any, walk = any;
    for (uint64_t k = 3; k < two_n; k += 2) {
        walk = host_mulmod(walk, step, q);
        if (walk < least) least = walk;
    }
    return least;
}

template <int LOGN>
static void layout_tables(HostLimb &hl) {
    const size_t N = (size_t)1 << LOGN;
    const uint64_t q = hl.lp.q;
    hl.tw.assign(N, U64x2{0, 0});
    hl.itw.assign(N, U64x2{0, 0});
    for (int s = 0; s < LOGN; ++s)
        for (int i = 0; i < (1 << s); ++i) {
            const size_t nat = ((size_t)1 << s) + i, pos = (size_t)tw_pos<LOGN>(s, i);
            hl.tw[pos] = U64x2{hl.root_powers[nat], shoup_of(hl.root_powers[nat], q)};
            hl.itw[pos] = U64x2{hl.inv_root_powers[nat], shoup_of(hl.inv_root_powers[nat], q)};
        }
}

std::string build_host_params(unsigned log_n, unsigned L, const uint64_t *moduli, HostParams &out) {
    if (log_n < 12 || log_n > 14) return "log_n must be 12, 13 or 14";
    if (L < 1 || L > 16) return "n_limbs must be in [1,16]";
    const uint64_t two_n = (uint64_t)2 << log_n;
    const size_t N = (size_t)1 << log_n;
    std::vector<uint64_t> qs;
    if (moduli) {
        for (unsigned l = 0; l < L; ++l) {
            const uint64_t q = moduli[l];
            if (q >= (1ull << 60) || q <= (1ull << 33)) return "modulus out of range (2^33, 2^60)";
            if ((q - 1) % two_n) return "modulus is not 1 mod 2N";
            if (!host_is_prime(q)) return "modulus is not prime";
            for (uint64_t prev : qs)
                if (prev == q) return "moduli must be distinct";
            qs.push_back(q);
        }
    } else {
        // default basis (DESIGN.md 2.1): the L largest primes below 2^60 of the form k * 2^32 + 1.  They are 1 mod 2N
        // for every supported N, and multiplying by such a modulus costs one 32-bit multiply-add (modarith.cuh, DPFHE_FAST).
        uint64_t cand = (1ull << 60) + 1;
        while (qs.size() < L) {
            cand -= 1ull << 32;
            if (host_is_prime(cand)) qs.push_back(cand);
        }
    }
    out.log_n = log_n;
    out.L = L;
    out.limbs.assign(L, HostLimb());
    for (unsigned l = 0; l < L; ++l) {
        HostLimb &hl = out.limbs[l];
        const uint64_t q = qs[l];
        hl.psi = min_primitive_root(q, two_n);
        std::vector<uint64_t> pw(N);
        pw[0] = 1;
        for (size_t k = 1; k < N; ++k) pw[k] = host_mulmod(pw[k - 1], hl.psi, q);
        hl.root_powers.resize(N);
        hl.inv_root_powers.resize(N);
        for (size_t k = 0; k < N; ++k) {
            const uint64_t w = pw[rev_bits((uint32_t)k, log_n)];
            hl.root_powers[k] = w;
            hl.inv_root_powers[k] = host_powmod(w, q - 2, q);
        }
        LimbParams &lp = hl.lp;
        lp.q = q;
        lp.q2 = 2 * q;
        lp.qsb = (uint64_t)SB * q;
        lp.q4 = 4 * q;
        lp.q8 = 8 * q;
        lp.nq = 0 - q;
        unsigned bits = 64 - (unsigned)__builtin_clzll(q);
        lp.bar_shift = bits - 2;
        lp.bar_mu = (uint64_t)(((u128)1 << (lp.bar_shift + 64)) / q);
        lp.mu32 = (uint32_t)(((u128)1 << 64) / q);
        lp.nqh = (uint32_t)q == 1u ? 0u - (uint32_t)(q >> 32) : 0u;
        lp.pad_ = 0;
        lp.ninv = host_powmod((uint64_t)N % q, q - 2, q);
        lp.ninv_s = shoup_of(lp.ninv, q);
        lp.wninv = host_mulmod(hl.inv_root_powers[1], lp.ninv, q);
        lp.wninv_s = shoup_of(lp.wninv, q);
        switch (log_n) {
            case 12: layout_tables<12>(hl); break;
            case 13: layout_tables<13>(hl); break;
            default: layout_tables<14>(hl); break;
        }
    }
    return "";
}

void build_ms_consts(const HostParams &hp, uint64_t t_plain, MsConsts &K) {
    typedef unsigned __int128 u128;
    auto shoup = [](uint64_t w, uint64_t q) { return (uint64_t)((((u128)w) << 64) / q); };
    const unsigned L = hp.L;
    const uint64_t ql = hp.limbs[L - 1].lp.q;
    K = MsConsts();
    K.half = ql >> 1;
    K.has_t = t_plain ? 1u : 0u;
    K.tinv = t_plain ? host_powmod(t_plain % ql, ql - 2, ql) : 1;
    K.tinv_s = shoup(K.tinv, ql);
    for (unsigned i = 0; i + 1 < L; ++i) {
        const uint64_t q = hp.limbs[i].lp.q;
        K.qlm[i] = ql % q;
        K.qlm_s[i] = shoup(K.qlm[i], q);
        K.inv[i] = host_powmod(K.qlm[i], q - 2, q);
        K.inv_s[i] = shoup(K.inv[i], q);
        K.sinv[i] = t_plain ? host_mulmod(t_plain % q, K.inv[i], q) : K.inv[i];
        K.sinv_s[i] = shoup(K.sinv[i], q);
    }
}

void build_group_consts(const HostParams &hp, unsigned K, uint64_t t_plain, GroupConsts &G, MsConsts &Km) {
    typedef unsigned __int128 u128;
    auto shoup = [](uint64_t w, uint64_t q) { return (uint64_t)((((u128)w) << 64) / q); };
    const unsigned L = hp.L, Lq = L - K;
    auto q_of = [&](unsigned l) { return hp.limbs[l].lp.q; };
    // product of the moduli lo .. hi-1 except `skip`, modulo q
    auto prod_mod = [&](unsigned lo, unsigned hi, unsigned skip, uint64_t q) {
        uint64_t r = 1 % q;
        for (unsigned m = lo; m < hi; ++m)
            if (m != skip) r = host_mulmod(r, q_of(m) % q, q);
        return r;
    };
    G = GroupConsts();
    G.Lq = Lq;
    G.K = K;
    G.dnum = (Lq + K - 1) / K;
    auto fold = [&](unsigned l, uint64_t f) {   // limb l with N^-1 replaced by N^-1 * f
        LimbParams p = hp.limbs[l].lp;
        p.ninv = host_mulmod(p.ninv, f, p.q);
        p.ninv_s = shoup(p.ninv, p.q);
        p.wninv = host_mulmod(p.wninv, f, p.q);
        p.wninv_s = shoup(p.wninv, p.q);
        return p;
    };
    for (unsigned j = 0; j < Lq; ++j) {
        const unsigned lo = j / K * K, hi = lo + K < Lq ? lo + K : Lq;
        const uint64_t qj = q_of(j);
        G.lp_up[j] = fold(j, host_powmod(prod_mod(lo, hi, j, qj), qj - 2, qj));
        for (unsigned i = 0; i < L; ++i) {
            G.up[j][i] = prod_mod(lo, hi, j, q_of(i));
            G.up_s[j][i] = shoup(G.up[j][i], q_of(i));
        }
    }
    for (unsigned k = 0; k < K; ++k) {
        const unsigned s = Lq + k;
        const uint64_t p = q_of(s);
        uint64_t f = prod_mod(Lq, L, s, p);
        if (t_plain) f = host_mulmod(f, t_plain % p, p);
        G.lp_up[s] = fold(s, host_powmod(f, p - 2, p));
        G.half[k] = p >> 1;
        for (unsigned i = 0; i < Lq; ++i) {
            G.dn[k][i] = prod_mod(Lq, L, s, q_of(i));
            G.dn_s[k][i] = shoup(G.dn[k][i], q_of(i));
        }
    }
    Km = MsConsts();
    Km.has_t = 0;   // t^-1 is folded into lp_up of the special limbs
    Km.tinv = 1;
    for (unsigned i = 0; i < Lq; ++i) {
        const uint64_t q = q_of(i), Pm = prod_mod(Lq, L, L, q);
        G.neg_p[i] = q - Pm;
        Km.qlm[i] = Pm;
        Km.qlm_s[i] = shoup(Pm, q);
        Km.inv[i] = host_powmod(Pm, q - 2, q);
        Km.inv_s[i] = shoup(Km.inv[i], q);
        Km.sinv[i] = t_plain ? host_mulmod(t_plain % q, Km.inv[i], q) : Km.inv[i];
        Km.sinv_s[i] = shoup(Km.sinv[i], q);
    }
}

void build_rescale_consts(const HostParams &hp, unsigned K, uint64_t t_plain, GroupConsts &G, MsConsts &Km, RescaleConsts &R) {
    typedef unsigned __int128 u128;
    auto shoup = [](uint64_t w, uint64_t q) { return (uint64_t)((((u128)w) << 64) / q); };
    build_group_consts(hp, K, t_plain, G, Km);
    const unsigned L = hp.L, Lq = L - K, d = Lq - 1;   // d: the dropped limb
    const uint64_t qbar = hp.limbs[d].lp.q;
    auto fold = [&](LimbParams p, uint64_t f) {   // N^-1 replaced by N^-1 * f
        p.ninv = host_mulmod(p.ninv, f, p.q);
        p.ninv_s = shoup(p.ninv, p.q);
        p.wninv = host_mulmod(p.wninv, f, p.q);
        p.wninv_s = shoup(p.wninv, p.q);
        return p;
    };
    // special k: Phat'_k = Phat_k * qbar, so its N^-1 takes a further qbar^-1
    for (unsigned k = 0; k < K; ++k) {
        const uint64_t p = hp.limbs[Lq + k].lp.q;
        G.lp_up[Lq + k] = fold(G.lp_up[Lq + k], host_powmod(qbar % p, p - 2, p));
    }
    // the dropped limb: Phat'_qbar = P, y_qbar = INTT(acc) * (t P)^-1 mod qbar
    uint64_t P_qbar = 1;
    for (unsigned k = 0; k < K; ++k) P_qbar = host_mulmod(P_qbar, hp.limbs[Lq + k].lp.q % qbar, qbar);
    const uint64_t f = t_plain ? host_mulmod(P_qbar, t_plain % qbar, qbar) : P_qbar;
    R = RescaleConsts();
    R.lp_drop = fold(hp.limbs[d].lp, host_powmod(f, qbar - 2, qbar));
    R.half = qbar >> 1;
    for (unsigned i = 0; i < 16; ++i) G.neg_p[i] = 0, Km.inv[i] = Km.inv_s[i] = Km.sinv[i] = Km.sinv_s[i] = 0;
    for (unsigned k = 0; k < K; ++k) G.dn[k][d] = G.dn_s[k][d] = 0;
    for (unsigned i = 0; i < d; ++i) {
        const uint64_t q = hp.limbs[i].lp.q, Pm = Km.qlm[i], Ppm = host_mulmod(Pm, qbar % q, q);   // P mod q_i, P' mod q_i
        for (unsigned k = 0; k < K; ++k) {
            G.dn[k][i] = host_mulmod(G.dn[k][i], qbar % q, q);
            G.dn_s[k][i] = shoup(G.dn[k][i], q);
        }
        R.dn[i] = Pm;
        R.dn_s[i] = shoup(Pm, q);
        G.neg_p[i] = q - Ppm;
        Km.inv[i] = host_powmod(Ppm, q - 2, q);
        Km.inv_s[i] = shoup(Km.inv[i], q);
        Km.sinv[i] = t_plain ? host_mulmod(t_plain % q, Km.inv[i], q) : Km.inv[i];
        Km.sinv_s[i] = shoup(Km.sinv[i], q);
    }
}

// ---- CKKS slot encoding (DESIGN.md §2.12) ----------------------------------------------------------------------
// cos and sin of pi k / N in fixed point with 126 fractional bits (Taylor series, error below 2^-120), rounded once to double.
namespace {
// floor(a * b / 2^126) for a, b <= 2^127
u128 fx126_mul(u128 a, u128 b) {
    const uint64_t a0 = (uint64_t)a, a1 = (uint64_t)(a >> 64), b0 = (uint64_t)b, b1 = (uint64_t)(b >> 64);
    const u128 p00 = (u128)a0 * b0, p01 = (u128)a0 * b1, p10 = (u128)a1 * b0, p11 = (u128)a1 * b1;
    const u128 mid = (p00 >> 64) + (uint64_t)p01 + (uint64_t)p10;
    const u128 hi = p11 + (p01 >> 64) + (p10 >> 64) + (mid >> 64);
    return (hi << 2) | ((uint64_t)mid >> 62);
}
// v / 2^126 (v <= 2^126) rounded to the nearest double, ties to even
double fx126_to_double(u128 v) {
    if (v == 0) return 0.0;
    int msb = 127;
    while (!((v >> msb) & 1)) --msb;
    if (msb <= 52) return (double)(uint64_t)v * 0x1p-126;   // exact
    const int sh = msb - 52;
    uint64_t m = (uint64_t)(v >> sh);
    const u128 rem = v & (((u128)1 << sh) - 1), half = (u128)1 << (sh - 1);
    if (rem > half || (rem == half && (m & 1))) ++m;
    return (double)m * 0x1p-126 * (double)((u128)1 << sh);   // m < 2^54 and a power of two: both products exact
}
// (cos, sin) of pi k / N for 0 <= k <= N/4 (the first octant)
Cplx cos_sin_octant(uint64_t k, unsigned log_n) {
    const u128 pi126 = ((u128)0xC90FDAA22168C234ull << 64) | 0xC4C6628B80DC1CD1ull;   // floor(pi * 2^126)
    const u128 x = (pi126 >> log_n) * k + (((pi126 & (((u128)1 << log_n) - 1)) * k) >> log_n);
    u128 c_pos = 0, c_neg = 0, s_pos = 0, s_neg = 0;
    u128 t = (u128)1 << 126;   // x^n / n!
    for (unsigned n = 0; t; ++n) {
        if (n % 2 == 0) ((n / 2) % 2 ? c_neg : c_pos) += t;
        else ((n / 2) % 2 ? s_neg : s_pos) += t;
        t = fx126_mul(t, x) / (n + 1);
    }
    return Cplx{fx126_to_double(c_pos - c_neg), fx126_to_double(s_pos - s_neg)};
}
}  // namespace

void build_ckks_tables(const HostParams &hp, std::vector<Cplx> &tw, std::vector<uint32_t> &tj, std::vector<uint64_t> &pow2) {
    const unsigned log_n = hp.log_n;
    const uint64_t N = (uint64_t)1 << log_n, quarter = N / 4, half = N / 2;
    tw.resize(N);
    for (uint64_t k = 0; k < N; ++k) {
        const uint64_t r = k % half;   // angle pi r / N in [0, pi/2)
        Cplx v = r <= quarter ? cos_sin_octant(r, log_n) : cos_sin_octant(half - r, log_n);
        if (r > quarter) v = Cplx{v.im, v.re};
        if (k >= half) v = Cplx{0.0 - v.im, v.re};   // (cos, sin)(a + pi/2) = (-sin a, cos a); cos(pi/2) is +0
        tw[k] = v;
    }
    tj.resize(half);
    uint64_t e = 1;
    for (uint64_t j = 0; j < half; ++j, e = e * 5 % (2 * N)) tj[j] = (uint32_t)((e - 1) / 4);
    pow2.resize((size_t)hp.L * CKKS_POW2_E);
    for (unsigned l = 0; l < hp.L; ++l) {
        const uint64_t q = hp.limbs[l].lp.q;
        uint64_t p = 1;
        for (int x = 0; x < CKKS_POW2_E; ++x, p = host_mulmod(p, 2, q)) pow2[(size_t)l * CKKS_POW2_E + x] = p;
    }
}

void build_ckks_consts(const HostParams &hp, double scale, CkksConsts &K) {
    K = CkksConsts();
    const unsigned L = hp.L;
    for (unsigned i = 0; i < L; ++i) {
        const uint64_t qi = hp.limbs[i].lp.q;
        K.qd[i] = (double)qi;
        for (unsigned j = 0; j < i; ++j) K.ginv[j][i] = host_powmod(hp.limbs[j].lp.q % qi, qi - 2, qi);
    }
    // (Q - 1) / 2 from the digits q_i - 1 of Q - 1, halved from the most significant digit
    uint64_t r = 0;
    for (unsigned i = L; i-- > 0;) {
        const uint64_t qi = hp.limbs[i].lp.q;
        const u128 v = (u128)r * qi + (qi - 1);
        K.half[i] = (uint64_t)(v >> 1);
        r = (uint64_t)(v & 1);
    }
    K.scale = scale;
}

// ---- BGV slot encoding (DESIGN.md §2.13) ----------------------------------------------------------------------
static uint32_t shoup32_of(uint64_t w, uint64_t t) { return (uint32_t)((w << 32) / t); }

Mod32 make_mod32(uint64_t t) {
    const uint64_t r32 = ((uint64_t)1 << 32) % t;
    return Mod32{(uint32_t)t, (uint32_t)r32, shoup32_of(r32, t), shoup32_of(1, t)};
}

bool bgv_plain_modulus_valid(unsigned log_n, uint64_t t) {
    const uint64_t two_n = (uint64_t)2 << log_n;
    return t < ((uint64_t)1 << 31) && t > two_n && (t - 1) % two_n == 0 && host_is_prime(t);
}

uint64_t bgv_zeta(unsigned log_n, uint64_t t) {
    const uint64_t two_n = (uint64_t)2 << log_n;
    uint64_t g = 2;
    while (host_powmod(g, (t - 1) / 2, t) != t - 1) ++g;   // the least quadratic non-residue
    return host_powmod(g, (t - 1) / two_n, t);             // zeta^N = g^((t-1)/2) = -1: a primitive 2N-th root of unity
}

bool build_bgv_tables(const HostParams &hp, uint64_t t, std::vector<uint32_t> &tab, BgvTables &T) {
    const unsigned log_n = hp.log_n;
    if (!bgv_plain_modulus_valid(log_n, t)) return false;
    const uint64_t N = (uint64_t)1 << log_n, two_n = 2 * N, zeta = bgv_zeta(log_n, t);
    std::vector<uint64_t> zp(two_n);   // zeta^k
    zp[0] = 1;
    for (uint64_t k = 1; k < two_n; ++k) zp[k] = zp[k - 1] * zeta % t;
    tab.assign(5 * N, 0);
    for (uint64_t k = 0; k < N; ++k) {
        const uint64_t e = rev_bits((uint32_t)k, log_n), w = zp[e], wi = zp[(two_n - e) % two_n];
        tab[k] = (uint32_t)w;
        tab[N + k] = shoup32_of(w, t);
        tab[2 * N + k] = (uint32_t)wi;
        tab[3 * N + k] = shoup32_of(wi, t);
    }
    // slot (0, c) holds m(zeta^e), slot (1, c) m(zeta^(2N - e)), e = 5^c mod 2N; the forward transform's output br(i) is m(zeta^(2i+1))
    uint64_t e = 1;
    for (uint64_t c = 0; c < N / 2; ++c, e = e * 5 % two_n) {
        tab[4 * N + c] = rev_bits((uint32_t)((e - 1) / 2), log_n);
        tab[4 * N + N / 2 + c] = rev_bits((uint32_t)((two_n - e - 1) / 2), log_n);
    }
    T = BgvTables();
    T.m = make_mod32(t);
    T.ninv = (uint32_t)host_powmod(N, t - 2, t);
    T.ninv_s = shoup32_of(T.ninv, t);
    return true;
}

void build_bgv_consts(const HostParams &hp, uint64_t t, BgvConsts &K) {
    K = BgvConsts();
    CkksConsts C;
    build_ckks_consts(hp, 1.0, C);
    for (unsigned i = 0; i < 16; ++i) {
        for (unsigned j = 0; j < 16; ++j) K.ginv[i][j] = C.ginv[i][j];
        K.half[i] = C.half[i];
    }
    uint64_t Qt = 1;
    for (unsigned i = 0; i < hp.L; ++i) {
        const uint64_t r = hp.limbs[i].lp.q % t;
        K.qt[i] = (uint32_t)r;
        K.qt_s[i] = shoup32_of(r, t);
        Qt = Qt * r % t;
    }
    K.Qt = (uint32_t)Qt;
    K.m = make_mod32(t);
}

// a^-1 mod m for gcd(a, m) = 1, m >= 2
static uint64_t inv_mod(uint64_t a, uint64_t m) {
    __int128 r0 = m, r1 = a % m, s0 = 0, s1 = 1;
    while (r1) {
        const __int128 q = r0 / r1, r2 = r0 - q * r1, s2 = s0 - q * s1;
        r0 = r1; r1 = r2; s0 = s1; s1 = s2;
    }
    return (uint64_t)(s0 < 0 ? s0 + m : s0);
}
// floor(w 2^64 / m), w < m
static uint64_t companion(uint64_t w, uint64_t m) { return (uint64_t)(((unsigned __int128)w << 64) / m); }

void build_compact_args(uint64_t q0, unsigned log_n, unsigned bits, uint64_t t_plain, CompactArgs &A) {
    A = CompactArgs();
    A.q = q0;
    A.r = (uint64_t)(((unsigned __int128)1 << bits) % q0);
    A.r_s = companion(A.r, q0);
    uint64_t inv = 1;   // q0^-1 mod 2^64 by Newton's iteration (q0 odd): each step doubles the correct low bits
    for (int i = 0; i < 6; ++i) inv *= 2 - q0 * inv;
    A.qinv64 = inv;
    A.t = t_plain;
    if (t_plain) {
        const uint64_t qinv_t = inv_mod(q0 % t_plain, t_plain);
        A.c = (t_plain - qinv_t) % t_plain;
        A.c_s = companion(A.c, t_plain);
        const uint64_t lambda = (uint64_t)((unsigned __int128)(((unsigned __int128)1 << bits) % t_plain) * qinv_t % t_plain);
        A.mu = inv_mod(lambda, t_plain);
        A.mu_s = companion(A.mu, t_plain);
    }
    A.bits = bits;
    A.tiles = (uint32_t)(((size_t)1 << log_n) / 64);
}

}  // namespace dpfhe
