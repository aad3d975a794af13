// host_ctx.cpp — see host_ctx.h. Product code (host), no CUDA, no dependency on oracle/.
#include "host_ctx.h"
#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace b200
{
typedef unsigned __int128 u128;

// ------------------------------------------------------------------------------------------------
// scalar number theory
// ------------------------------------------------------------------------------------------------
Modulus::Modulus(u64 value) : p(value)
{
    if (value < 2)
        throw std::invalid_argument("modulus must be >= 2");
    bits = 64 - __builtin_clzll(value);
    // floor(2^128 / p) by two-step long division (2^128 = (2^64)*(2^64))
    u128 hi = ((u128)1 << 64) / p;           // floor(2^64/p)        (< 2^64 since p >= 2)
    u128 rem = ((u128)1 << 64) - hi * p;     // 2^64 mod p
    u128 lo = (rem << 64) / p;               // floor(rem*2^64 / p)  (< 2^64)
    r1 = (u64)hi;
    r0 = (u64)lo;
}

Shoup Modulus::shoup(u64 w) const
{
    Shoup s;
    s.w = w;
    s.wq = (u64)(((u128)w << 64) / p);
    return s;
}

u64 pow_mod(u64 a, u64 e, u64 p)
{
    u64 r = 1 % p;
    a %= p;
    while (e)
    {
        if (e & 1)
            r = (u64)((u128)r * a % p);
        a = (u64)((u128)a * a % p);
        e >>= 1;
    }
    return r;
}

bool try_inv_mod(u64 a, u64 m, u64 &out)
{
    // extended Euclid on (a mod m, m) with signed 128-bit cofactors
    if (m < 2)
        return false;
    __int128 t0 = 0, t1 = 1;
    u64 r0 = m, r1 = a % m;
    if (r1 == 0)
        return false;
    while (r1)
    {
        u64 q = r0 / r1;
        u64 r2 = r0 - q * r1;
        __int128 t2 = t0 - (__int128)q * t1;
        r0 = r1;
        r1 = r2;
        t0 = t1;
        t1 = t2;
    }
    if (r0 != 1)
        return false;
    __int128 v = t0 % (__int128)m;
    if (v < 0)
        v += m;
    out = (u64)v;
    return true;
}

u64 inv_mod(u64 a, u64 m)
{
    u64 r;
    if (!try_inv_mod(a, m, r))
        throw std::logic_error("invalid rns bases (value not invertible)");
    return r;
}

bool is_prime(u64 v)
{
    if (v < 2)
        return false;
    static const u64 small[] = { 2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37 };
    for (u64 s : small)
    {
        if (v == s)
            return true;
        if (v % s == 0)
            return false;
    }
    u64 d = v - 1;
    int r = 0;
    while (!(d & 1))
    {
        d >>= 1;
        r++;
    }
    // deterministic Miller-Rabin: these 12 bases decide primality for every 64-bit integer
    for (u64 a : small)
    {
        u64 x = pow_mod(a, d, v);
        if (x == 1 || x == v - 1)
            continue;
        bool comp = true;
        for (int i = 1; i < r; i++)
        {
            x = (u64)((u128)x * x % v);
            if (x == v - 1)
            {
                comp = false;
                break;
            }
        }
        if (comp)
            return false;
    }
    return true;
}

std::vector<u64> get_primes(u64 factor, int bit_size, size_t count)
{
    // largest candidates == 1 mod factor below 2^bit_size, descending (the reference's order)
    std::vector<u64> out;
    u64 value = ((u64(1) << bit_size) - 1) / factor * factor + 1;
    u64 lower = u64(1) << (bit_size - 1);
    while (count > 0 && value > lower)
    {
        if (is_prime(value))
        {
            out.push_back(value);
            count--;
        }
        value -= factor;
    }
    if (count > 0)
        throw std::logic_error("failed to find enough qualifying primes");
    return out;
}

bool minimal_primitive_root(u64 degree, u64 p, u64 &root)
{
    if ((p - 1) % degree)
        return false;
    u64 quotient = (p - 1) / degree;
    // any generator-ish candidate a: a^quotient has order dividing `degree`; primitive iff ^(degree/2) == -1
    u64 g = 0;
    for (u64 a = 2; a < p && a < 100000; a++)
    {
        u64 c = pow_mod(a, quotient, p);
        if (pow_mod(c, degree >> 1, p) == p - 1)
        {
            g = c;
            break;
        }
    }
    if (!g)
        return false;
    // the primitive degree-th roots are exactly the odd powers of g; take the smallest
    u64 g2 = (u64)((u128)g * g % p);
    u64 cur = g, best = g;
    for (u64 i = 0; i < degree; i += 2)
    {
        if (cur < best)
            best = cur;
        cur = (u64)((u128)cur * g2 % p);
    }
    root = best;
    return true;
}

u64 reverse_bits(u64 v, int bits)
{
    u64 r = 0;
    for (int i = 0; i < bits; i++)
        r |= ((v >> i) & 1) << (bits - 1 - i);
    return r;
}

// ------------------------------------------------------------------------------------------------
// BigUInt
// ------------------------------------------------------------------------------------------------
void BigUInt::mul(u64 m)
{
    u64 carry = 0;
    for (auto &x : w)
    {
        u128 t = (u128)x * m + carry;
        x = (u64)t;
        carry = (u64)(t >> 64);
    }
    if (carry)
        w.push_back(carry);
}
void BigUInt::sub_small(u64 v)
{
    for (size_t i = 0; i < w.size() && v; i++)
    {
        u64 before = w[i];
        w[i] -= v;
        v = before < v ? 1 : 0;
    }
}
u64 BigUInt::divmod(u64 d)
{
    u64 rem = 0;
    for (size_t i = w.size(); i-- > 0;)
    {
        u128 cur = ((u128)rem << 64) | w[i];
        w[i] = (u64)(cur / d);
        rem = (u64)(cur % d);
    }
    while (w.size() > 1 && w.back() == 0)
        w.pop_back();
    return rem;
}
u64 BigUInt::mod(u64 d) const
{
    u64 rem = 0;
    for (size_t i = w.size(); i-- > 0;)
        rem = (u64)((((u128)rem << 64) | w[i]) % d);
    return rem;
}
int BigUInt::bit_length() const
{
    for (size_t i = w.size(); i-- > 0;)
        if (w[i])
            return (int)(64 * i + 64 - __builtin_clzll(w[i]));
    return 0;
}
bool BigUInt::operator<(const BigUInt &o) const
{
    size_t a = w.size(), b = o.w.size();
    while (a > 1 && w[a - 1] == 0)
        a--;
    while (b > 1 && o.w[b - 1] == 0)
        b--;
    if (a != b)
        return a < b;
    for (size_t i = a; i-- > 0;)
        if (w[i] != o.w[i])
            return w[i] < o.w[i];
    return false;
}

// ------------------------------------------------------------------------------------------------
// BLAKE2b-256 (RFC 7693, unkeyed) for parms_id = H(scheme, n, q_0.., t)  (S/encryptionparams.cpp:124-158)
// ------------------------------------------------------------------------------------------------
namespace
{
const u64 blake2b_iv[8] = { 0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                            0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL };
const unsigned char blake2b_sigma[12][16] = {
    { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 },
    { 11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4 }, { 7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8 },
    { 9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13 }, { 2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9 },
    { 12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11 }, { 13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10 },
    { 6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5 }, { 10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0 },
    { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 }
};
inline u64 rotr64(u64 x, int r) { return (x >> r) | (x << (64 - r)); }
void blake2b_compress(u64 h[8], const unsigned char block[128], u128 t, bool last)
{
    u64 m[16], v[16];
    std::memcpy(m, block, 128);
    for (int i = 0; i < 8; i++)
    {
        v[i] = h[i];
        v[i + 8] = blake2b_iv[i];
    }
    v[12] ^= (u64)t;
    v[13] ^= (u64)(t >> 64);
    if (last)
        v[14] = ~v[14];
    for (int r = 0; r < 12; r++)
    {
        const unsigned char *s = blake2b_sigma[r];
        auto G = [&](int a, int b, int c, int d, u64 x, u64 y) {
            v[a] = v[a] + v[b] + x;
            v[d] = rotr64(v[d] ^ v[a], 32);
            v[c] = v[c] + v[d];
            v[b] = rotr64(v[b] ^ v[c], 24);
            v[a] = v[a] + v[b] + y;
            v[d] = rotr64(v[d] ^ v[a], 16);
            v[c] = v[c] + v[d];
            v[b] = rotr64(v[b] ^ v[c], 63);
        };
        G(0, 4, 8, 12, m[s[0]], m[s[1]]);
        G(1, 5, 9, 13, m[s[2]], m[s[3]]);
        G(2, 6, 10, 14, m[s[4]], m[s[5]]);
        G(3, 7, 11, 15, m[s[6]], m[s[7]]);
        G(0, 5, 10, 15, m[s[8]], m[s[9]]);
        G(1, 6, 11, 12, m[s[10]], m[s[11]]);
        G(2, 7, 8, 13, m[s[12]], m[s[13]]);
        G(3, 4, 9, 14, m[s[14]], m[s[15]]);
    }
    for (int i = 0; i < 8; i++)
        h[i] ^= v[i] ^ v[i + 8];
}
void blake2b_256(const void *in, size_t len, u64 out[4])
{
    u64 h[8];
    for (int i = 0; i < 8; i++)
        h[i] = blake2b_iv[i];
    h[0] ^= 0x01010000ULL ^ 32; // digest length 32, no key, fanout = depth = 1
    const unsigned char *p = (const unsigned char *)in;
    unsigned char block[128];
    u128 t = 0;
    while (len > 128)
    {
        t += 128;
        blake2b_compress(h, p, t, false);
        p += 128;
        len -= 128;
    }
    std::memset(block, 0, 128);
    std::memcpy(block, p, len);
    t += len;
    blake2b_compress(h, block, t, true);
    for (int i = 0; i < 4; i++)
        out[i] = h[i];
}
} // namespace

void compute_parms_id(size_t n, const std::vector<u64> &moduli, u64 t, u64 out[4])
{
    std::vector<u64> data;
    data.push_back(1); // scheme_type::bfv
    data.push_back((u64)n);
    for (u64 m : moduli)
        data.push_back(m);
    data.push_back(t);
    blake2b_256(data.data(), data.size() * sizeof(u64), out);
}

// ------------------------------------------------------------------------------------------------
// tables
// ------------------------------------------------------------------------------------------------
static NttPrimeHost make_ntt_prime(u64 p, int logn, bool allow_fp = true)
{
    NttPrimeHost P;
    P.mod = Modulus(p);
    const size_t n = size_t(1) << logn;
    if (!minimal_primitive_root(2 * n, p, P.root))
        throw std::invalid_argument("modulus does not support the NTT for this degree");
    P.fwd.assign(2 * n, 0);
    P.inv.assign(2 * n, 0);
    u64 power = 1;
    std::vector<u64> pw(n);
    for (size_t i = 0; i < n; i++)
    {
        pw[reverse_bits(i, logn)] = power; // fwd[bitrev(i)] = psi^i
        power = P.mod.mul(power, P.root);
    }
    // batch inversion of the forward twiddles (inv[idx] = fwd[idx]^-1)
    std::vector<u64> prefix(n);
    u64 acc = 1;
    for (size_t i = 0; i < n; i++)
    {
        prefix[i] = acc;
        acc = P.mod.mul(acc, pw[i]);
    }
    u64 inv_acc = inv_mod(acc, p);
    std::vector<u64> ipw(n);
    for (size_t i = n; i-- > 0;)
    {
        ipw[i] = P.mod.mul(inv_acc, prefix[i]);
        inv_acc = P.mod.mul(inv_acc, pw[i]);
    }
    for (size_t i = 0; i < n; i++)
    {
        Shoup a = P.mod.shoup(pw[i]), b = P.mod.shoup(ipw[i]);
        P.fwd[2 * i] = a.w;
        P.fwd[2 * i + 1] = a.wq;
        P.inv[2 * i] = b.w;
        P.inv[2 * i + 1] = b.wq;
    }
    u64 inv_n = inv_mod((u64)n % p, p);
    P.inv_n = P.mod.shoup(inv_n);
    P.inv_n_w = P.mod.shoup(P.mod.mul(inv_n, n > 1 ? ipw[1] : 1));
    P.fp = P.mod.bits <= FP_PRIME_BITS && allow_fp;
    if (P.fp)
    {
        const double pd = (double)p;
        P.dfwd.resize(n);
        P.dinv.resize(n);
        for (size_t i = 0; i < n; i++)
        {
            P.dfwd[i] = (double)pw[i];
            P.dinv[i] = (double)ipw[i];
        }
        P.inv_n_d[0] = (double)P.inv_n.w;
        P.inv_n_d[1] = (double)P.inv_n.w / pd;
        P.inv_n_w_d[0] = (double)P.inv_n_w.w;
        P.inv_n_w_d[1] = (double)P.inv_n_w.w / pd;
    }
    return P;
}

static u64 prod_mod(const std::vector<u64> &v, u64 p, int skip = -1)
{
    u64 r = 1 % p;
    for (size_t i = 0; i < v.size(); i++)
        if ((int)i != skip)
            r = (u64)((u128)r * (v[i] % p) % p);
    return r;
}

BfvHostContext::BfvHostContext(size_t poly_modulus_degree, const std::vector<u64> &coeff_modulus, u64 plain_modulus)
{
    n = poly_modulus_degree;
    if (n < 2 || (n & (n - 1)) || n > 131072)
        throw std::invalid_argument("poly_modulus_degree is invalid");
    logn = __builtin_ctzll((u64)n);
    K = (int)coeff_modulus.size();
    if (K < 1 || K > 64)
        throw std::invalid_argument("coeff_modulus is invalid");
    t = plain_modulus;
    if (t < 2)
        throw std::invalid_argument("plain_modulus is invalid");
    t_mod = Modulus(t);
    for (int i = 0; i < K; i++)
    {
        u64 q = coeff_modulus[i];
        if (q < 2 || (64 - __builtin_clzll(q)) > 60 || !is_prime(q))
            throw std::invalid_argument("coeff_modulus is invalid");
        for (int j = 0; j < i; j++)
            if (coeff_modulus[j] == q)
                throw std::invalid_argument("coeff_modulus is invalid (not coprime)");
        primes.push_back(make_ntt_prime(q, logn));
    }
    using_keyswitching = K > 1;
    using_batching = false;
    if (is_prime(t) && (t - 1) % (2 * n) == 0)
    {
        plain_ntt = make_ntt_prime(t, logn);
        using_batching = true;
        // BatchEncoder::populate_matrix_reps_index_map (S/batchencoder.cpp:64-88): slot i of the 2 x n/2 matrix lives at
        // coefficient slot_index_map[i] of the transformed polynomial
        const size_t row = n >> 1, m = n << 1;
        slot_index_map.resize(n);
        u64 pos = 1;
        for (size_t i = 0; i < row; i++)
        {
            slot_index_map[i] = (uint32_t)reverse_bits((pos - 1) >> 1, logn);
            slot_index_map[row | i] = (uint32_t)reverse_bits((m - pos - 1) >> 1, logn);
            pos = (pos * 3) & (m - 1);
        }
    }

    // Auxiliary BEHZ base: m_sk, gamma, then B.
    // The reference takes the largest 61-bit primes == 1 mod 2n (S/util/rns.cpp:634-644).  The result of
    // bfv_multiply does not depend on WHICH auxiliary primes are used, only on their product being large enough
    // (t * n * K * Q * (1+rho)^2 < prod(B) * m_sk, the reference's own condition, rns.cpp:617-624): every
    // approximation error in the BEHZ chain (the q-overflows of the two fast base conversions) is a function of
    // the base-q residues alone, and the Shenoy-Kumaresan step is exact.  So when every user prime fits the FP64
    // NTT path we pick 47..49-bit auxiliary primes instead (as wide as the widest user prime, at least 47), so that the
    // Bsk transforms take the same fast path;
    // gamma (decryption only, never transformed) stays the reference's.
    aux0 = K;
    bool all_fp = std::getenv("B200_FORCE_AUX61") == nullptr;
    for (int i = 0; i < K; i++)
        all_fp = all_fp && primes[i].fp;
    int user_bits = 0;
    for (int i = 0; i < K; i++)
        user_bits = std::max(user_bits, primes[i].mod.bits);
    aux_bits = all_fp ? std::max(FP_AUX_BITS_MIN, user_bits) : 61;
    const int aux_centibits = aux_bits * 100 - 10; // every prime found just below 2^aux_bits carries more than this
    const std::vector<u64> ref_aux = get_primes(2 * (u64)n, 61, 2);
    // enough 47-bit primes for the largest level: bits(prod(B) * m_sk) >= 33 + bits(t) + bits(Q)
    size_t aux_count = (size_t)K + 3;
    if (all_fp)
    {
        BigUInt Qall(1);
        for (int i = 0; i < K; i++)
            Qall.mul(coeff_modulus[i]);
        aux_count = (size_t)((33 + t_mod.bits + Qall.bit_length()) * 100 / aux_centibits + 3);
    }
    std::vector<u64> aux;
    { // descending from 2^aux_bits, skipping anything the user's chain (or t) already uses
        std::vector<u64> cand = get_primes(2 * (u64)n, aux_bits, aux_count + (size_t)K + 1);
        for (u64 v : cand)
        {
            bool used = v == plain_modulus;
            for (int i = 0; i < K; i++)
                used = used || v == coeff_modulus[i];
            if (!used && aux.size() < aux_count)
                aux.push_back(v);
        }
    }
    aux[1] = ref_aux[1]; // gamma: the reference's second 61-bit prime
    for (size_t i = 0; i < aux.size(); i++)
        primes.push_back(make_ntt_prime(aux[i], logn));
    const u64 m_sk = aux[0], gamma = aux[1];
    const u64 mt = u64(1) << 32;

    // levels: [key level (K primes)] + data levels K-1 .. 1 primes (only the key level when K == 1)
    std::vector<int> sizes;
    sizes.push_back(K);
    for (int s = K - 1; s >= 1; s--)
        sizes.push_back(s);
    for (int k : sizes)
    {
        LevelHost L;
        L.k = k;
        std::vector<u64> q(coeff_modulus.begin(), coeff_modulus.begin() + k);
        for (int i = 0; i < k; i++)
            L.q_idx.push_back(i);
        compute_parms_id(n, q, t, L.parms_id);

        BigUInt Q(1);
        for (u64 v : q)
            Q.mul(v);
        L.total_bits = Q.bit_length();
        if (aux_bits == 61)
        { // the reference's rule (S/util/rns.cpp:617-624)
            L.nB = k;
            if (32 + t_mod.bits + L.total_bits >= 61 * k + 61)
                L.nB++;
        }
        else
        { // same inequality, solved for aux_bits-bit primes (each contributes > aux_bits - 0.1 bits)
            int need = 33 + t_mod.bits + L.total_bits;
            int cnt = (need * 100 + aux_centibits - 1) / aux_centibits;
            L.nB = std::max(1, cnt - 1);
        }
        L.nBsk = L.nB + 1;
        if ((size_t)L.nB + 2 > aux.size())
            throw std::logic_error("internal: auxiliary base too small");
        std::vector<u64> B(aux.begin() + 2, aux.begin() + 2 + L.nB);
        for (int b = 0; b < L.nB; b++)
            L.bsk_idx.push_back(aux0 + 2 + b);
        L.bsk_idx.push_back(aux0);
        L.gamma_idx = aux0 + 1;
        std::vector<u64> bsk = B;
        bsk.push_back(m_sk);

        // (Q/q_i)^-1 mod q_i
        std::vector<u64> inv_punc_q(k);
        for (int i = 0; i < k; i++)
            inv_punc_q[i] = inv_mod(prod_mod(q, q[i], i), q[i]);

        // ---- lift
        L.lift_c.resize(k);
        L.lift_mt.resize(k);
        for (int i = 0; i < k; i++)
        {
            Modulus qi(q[i]);
            L.lift_c[i] = qi.shoup(qi.mul(mt % q[i], inv_punc_q[i]));
            L.lift_mt[i] = prod_mod(q, mt, i);
        }
        L.neg_inv_q_mod_mt = (mt - inv_mod(prod_mod(q, mt), mt)) % mt;
        L.lift_mat.resize((size_t)L.nBsk * k);
        L.lift_qm.resize(L.nBsk);
        L.scale_tq.resize(L.nBsk);
        L.scale_mat.resize((size_t)L.nBsk * k);
        for (int j = 0; j < L.nBsk; j++)
        {
            Modulus pj(bsk[j]);
            u64 inv_mt = inv_mod(mt % pj.p, pj.p);
            u64 Qp = prod_mod(q, pj.p);
            u64 invQ = inv_mod(Qp, pj.p);
            L.lift_qm[j] = pj.mul(Qp, inv_mt);
            L.scale_tq[j] = pj.mul(t % pj.p, invQ);
            for (int i = 0; i < k; i++)
            {
                u64 punc = prod_mod(q, pj.p, i);
                L.lift_mat[(size_t)j * k + i] = pj.mul(punc, inv_mt);
                u64 v = pj.mul(punc, invQ);
                L.scale_mat[(size_t)j * k + i] = v ? pj.p - v : 0;
            }
        }
        // ---- scale / Shenoy-Kumaresan
        L.scale_c.resize(k);
        for (int i = 0; i < k; i++)
        {
            Modulus qi(q[i]);
            L.scale_c[i] = qi.shoup(qi.mul(t % q[i], inv_punc_q[i]));
        }
        L.sk_c.resize(L.nB);
        for (int b = 0; b < L.nB; b++)
            L.sk_c[b] = Modulus(B[b]).shoup(inv_mod(prod_mod(B, B[b], b), B[b]));
        L.sk_mat_q.resize((size_t)k * L.nB);
        L.sk_prod_b_q.resize(k);
        for (int i = 0; i < k; i++)
        {
            for (int b = 0; b < L.nB; b++)
                L.sk_mat_q[(size_t)i * L.nB + b] = prod_mod(B, q[i], b);
            L.sk_prod_b_q[i] = prod_mod(B, q[i]);
        }
        {
            Modulus ms(m_sk);
            L.sk_inv_b_msk = inv_mod(prod_mod(B, m_sk), m_sk);
            L.sk_mat_msk.resize(L.nB);
            for (int b = 0; b < L.nB; b++)
                L.sk_mat_msk[b] = ms.mul(prod_mod(B, m_sk, b), L.sk_inv_b_msk);
        }
        // ---- q_last^-1 mod q_i
        for (int i = 0; i + 1 < k; i++)
            L.inv_qlast.push_back(Modulus(q[i]).shoup(inv_mod(q[k - 1] % q[i], q[i])));
        // ---- plaintext constants
        {
            BigUInt D = Q;
            L.q_mod_t = D.divmod(t); // D = floor(Q/t)
            L.delta.resize(k);
            for (int i = 0; i < k; i++)
                L.delta[i] = D.mod(q[i]);
            L.plain_upper_half_threshold = (t + 1) >> 1;
            L.fast_plain_lift = true;
            for (int i = 0; i < k; i++)
                L.fast_plain_lift = L.fast_plain_lift && (q[i] > t);
            L.plain_upper_half_inc.resize(k);
            if (L.fast_plain_lift)
                for (int i = 0; i < k; i++)
                    L.plain_upper_half_inc[i] = q[i] - t;
            else
            {
                // (Q - t) mod q_i ; requires Q > t which valid BFV parameters guarantee
                for (int i = 0; i < k; i++)
                    L.plain_upper_half_inc[i] = (q[i] - t % q[i]) % q[i];
            }
        }
        // ---- decrypt (scale & round through {t, gamma})
        {
            Modulus gm(gamma);
            L.dec_c.resize(k);
            L.dec_mat_t.resize(k);
            L.dec_mat_g.resize(k);
            u64 Qt = prod_mod(q, t), Qg = prod_mod(q, gamma);
            u64 neg_inv_t = 0, neg_inv_g = 0;
            u64 tmp;
            if (try_inv_mod(Qt, t, tmp))
                neg_inv_t = (t - tmp) % t;
            else
                throw std::logic_error("invalid rns bases (t not coprime to q)");
            neg_inv_g = gamma - inv_mod(Qg, gamma);
            for (int i = 0; i < k; i++)
            {
                Modulus qi(q[i]);
                L.dec_c[i] = qi.shoup(qi.mul(qi.mul(t % q[i], gamma % q[i]), inv_punc_q[i]));
                L.dec_mat_t[i] = t_mod.mul(prod_mod(q, t, i), neg_inv_t);
                L.dec_mat_g[i] = gm.mul(prod_mod(q, gamma, i), neg_inv_g);
            }
            L.inv_gamma_mod_t = inv_mod(gamma % t, t);
        }
        levels.push_back(std::move(L));
    }
}

uint32_t BfvHostContext::galois_elt_from_step(int steps) const
{
    const uint32_t m = (uint32_t)(2 * n);
    if (steps == 0)
        return m - 1; // column swap
    const uint32_t row = (uint32_t)(n >> 1);
    bool sign = steps < 0;
    uint32_t pos = (uint32_t)(sign ? -steps : steps);
    if (pos >= row)
        throw std::invalid_argument("step count too large");
    pos = sign ? row - pos : pos;
    u64 g = 1;
    for (uint32_t i = 0; i < pos; i++)
        g = (g * 3) & (m - 1);
    return (uint32_t)g;
}

} // namespace b200
