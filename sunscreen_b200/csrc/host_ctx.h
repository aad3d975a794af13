// host_ctx.h — host-side precomputation for the BFV hot path (product code, no CUDA).
//
// Restates WHAT the reference's context precomputes — not how:
//   prime search        get_primes(2n, 61, count)                S/util/numth.cpp:278-311
//   minimal 2n-th root  try_minimal_primitive_root               S/util/numth.cpp:386-412
//   NTT tables          NTTTables::initialize                    S/util/ntt.cpp:240-299
//   BEHZ toolbox        RNSTool::initialize                      S/util/rns.cpp:590-799
//   plain lift consts   SEALContext::validate                    S/context.cpp:303-346
//   modulus chain       SEALContext::create_next_context_data    S/context.cpp:422-522
// Constants are pre-folded for our fused kernels (see bfv_body.cuh); every folded constant is an exact
// product/inverse modulo the same prime, so the kernels' results equal the reference's word for word.
#pragma once
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <vector>

namespace b200
{
typedef unsigned long long u64;

struct Shoup
{
    u64 w = 0, wq = 0; // wq = floor(w * 2^64 / p)
};

struct Modulus
{
    u64 p = 0;
    u64 r0 = 0, r1 = 0; // floor(2^128 / p) = r1*2^64 + r0
    int bits = 0;
    Modulus() {}
    explicit Modulus(u64 value);
    u64 reduce(u64 x) const { return x % p; }
    u64 mul(u64 a, u64 b) const { return (u64)(((unsigned __int128)a * b) % p); }
    Shoup shoup(u64 w) const;
};

u64 pow_mod(u64 a, u64 e, u64 p);
bool try_inv_mod(u64 a, u64 m, u64 &out); // works for non-prime m (extended Euclid)
u64 inv_mod(u64 a, u64 m);                // throws std::logic_error if not invertible
bool is_prime(u64 v);
std::vector<u64> get_primes(u64 factor, int bit_size, size_t count);
bool minimal_primitive_root(u64 degree, u64 p, u64 &root); // degree = 2n (power of two)
u64 reverse_bits(u64 v, int bits);

// Little-endian multi-precision unsigned integer (only what the context needs).
struct BigUInt
{
    std::vector<u64> w;
    explicit BigUInt(u64 v = 0) : w(1, v) {}
    void mul(u64 m);
    void sub_small(u64 v);
    u64 divmod(u64 d); // this /= d, returns remainder
    u64 mod(u64 d) const;
    int bit_length() const;
    bool operator<(const BigUInt &o) const;
};

// Per-prime NTT tables (host copy). fwd/inv hold 2n words: {w, wq} per index.
struct NttPrimeHost
{
    Modulus mod;
    u64 root = 0; // minimal primitive 2n-th root
    Shoup inv_n, inv_n_w;
    std::vector<u64> fwd, inv;
    // FP64 fast path (primes < 2^FP_PRIME_BITS): the same twiddles as exact integer-valued doubles {w, w/p}
    bool fp = false;
    std::vector<double> dfwd, dinv; // [n] twiddles as doubles (FP64 transform)
    double inv_n_d[2] = { 0, 0 }, inv_n_w_d[2] = { 0, 0 };
    unsigned renorm_inv_mask = 0;   // bit i: renormalise the inputs of inverse pass i (see ntt_fp_body.cuh)
    unsigned renorm_fwd_mask = 0;
};

// Largest prime size (bits) the FP64 NTT path accepts; also the size of the auxiliary BEHZ primes we pick
// when every user prime qualifies.
// Primes up to this many bits take the FP64 path.  Every value the FP64 kernels hold is an integer of magnitude <= 2^53
// (exactly representable); the host-side bound bookkeeping (b200_bfv.cu: build_device) places a renormalisation before
// any NTT pass whose butterflies could exceed that.  49 bits is the largest width for which a radix-16 inverse pass
// (x16 growth on the sum path) still fits after a renormalisation: 16 * 0.76 * 2^49 < 2^53.
static const int FP_PRIME_BITS = 49;
static const int FP_AUX_BITS_MIN = 47; // auxiliary BEHZ primes are at least this wide (fewer of them are needed)

// One level of the modulus chain (mirrors ContextData + RNSTool for that level).
// Index conventions: q_idx / bsk_idx / gamma_idx index into BfvHostContext::primes.
struct LevelHost
{
    int k = 0;                 // residues at this level
    std::vector<int> q_idx;    // [k]
    int nB = 0, nBsk = 0;      // |B|, |Bsk| = |B|+1 (m_sk last)
    std::vector<int> bsk_idx;  // [nBsk]  B primes then m_sk
    int gamma_idx = -1;
    u64 parms_id[4] = { 0, 0, 0, 0 };

    // --- BEHZ lift (steps 1-2 of bfv_multiply, fused): z_j = (sum_i y_i*lift_mat[j][i] + rc*lift_qm[j]) mod p_j
    std::vector<Shoup> lift_c;       // [k]      m~ * (Q/q_i)^-1 mod q_i
    std::vector<u64> lift_mat;       // [nBsk*k] (Q/q_i) * m~^-1 mod p_j
    std::vector<u64> lift_mt;        // [k]      (Q/q_i) mod m~   (low 32 bits)
    u64 neg_inv_q_mod_mt = 0;        //          -Q^-1 mod m~
    std::vector<u64> lift_qm;        // [nBsk]   Q * m~^-1 mod p_j
    // --- BEHZ scale (steps 6-8 fused)
    std::vector<Shoup> scale_c;      // [k]      t * (Q/q_i)^-1 mod q_i
    std::vector<u64> scale_tq;       // [nBsk]   t * Q^-1 mod p_j
    std::vector<u64> scale_mat;      // [nBsk*k] -(Q/q_i) * Q^-1 mod p_j
    std::vector<Shoup> sk_c;         // [nB]     (B/b)^-1 mod b
    std::vector<u64> sk_mat_q;       // [k*nB]   (B/b) mod q_i
    std::vector<u64> sk_mat_msk;     // [nB]     (B/b) * B^-1 mod m_sk
    u64 sk_inv_b_msk = 0;            //          B^-1 mod m_sk
    std::vector<u64> sk_prod_b_q;    // [k]      B mod q_i
    // --- mod-down by the last prime of THIS level (divide_and_round_q_last / key-switch uses the key level's)
    std::vector<Shoup> inv_qlast;    // [k-1]    q_last^-1 mod q_i
    // --- plaintext constants (BFV)
    std::vector<u64> delta;          // [k] floor(Q/t) mod q_i
    u64 q_mod_t = 0;                 //     Q mod t
    u64 plain_upper_half_threshold = 0;        // floor((t+1)/2)
    std::vector<u64> plain_upper_half_inc;     // [k] (Q - t) mod q_i  (== q_i - t when q_i > t)
    bool fast_plain_lift = false;              // all q_i > t
    // --- decrypt (scale and round with gamma)
    std::vector<Shoup> dec_c;        // [k] t*gamma*(Q/q_i)^-1 mod q_i
    std::vector<u64> dec_mat_t;      // [k] -(Q/q_i)*Q^-1 mod t       (pre-folded neg_inv_q_mod_t)
    std::vector<u64> dec_mat_g;      // [k] -(Q/q_i)*Q^-1 mod gamma
    u64 inv_gamma_mod_t = 0;
    int total_bits = 0;              // bit length of Q
};

struct BfvHostContext
{
    int logn = 0;
    size_t n = 0;
    u64 t = 0;
    Modulus t_mod;
    std::vector<NttPrimeHost> primes; // key primes [0,K), then aux primes: m_sk, gamma, B...
    int K = 0;                        // key-level prime count
    int aux0 = 0;                     // index of m_sk; gamma = aux0+1; B_i = aux0+2+i
    int aux_bits = 61;                // 61 = the reference's aux base; 47..49 = FP64-friendly base (same results, see DESIGN.md)
    std::vector<LevelHost> levels;    // levels[0] = key level, levels[1] = first data level, ...
    bool using_keyswitching = false;  // K > 1
    bool using_batching = false;      // t prime and t == 1 mod 2n
    NttPrimeHost plain_ntt;           // tables mod t when using_batching (for BatchEncoder)
    std::vector<uint32_t> slot_index_map; // [n] when using_batching: coefficient index of each slot (BatchEncoder)

    // Build everything. Throws std::invalid_argument for parameters the reference would reject
    // (non-power-of-two n, moduli not == 1 mod 2n, duplicates, t >= q_i is allowed, ...).
    BfvHostContext(size_t poly_modulus_degree, const std::vector<u64> &coeff_modulus, u64 plain_modulus);

    int first_level() const { return K > 1 ? 1 : 0; }
    // Galois element for a row rotation by `steps` / column swap (S/util/galois.cpp:53-95).
    uint32_t galois_elt_from_step(int steps) const;
};

void compute_parms_id(size_t n, const std::vector<u64> &moduli, u64 t, u64 out[4]);

} // namespace b200
