// sampling.h — host-side randomness for key generation / encryption (SURVEY.md §8(a) row E).
//
// Bit-parity with the reference's seeded entry points requires the SAME random stream, so sampling stays on the
// host and restates the reference's generators:
//   Blake2xbPRNG           S/randomgen.cpp:201-211, S/randomgen.h:320-395 (4096-byte buffer, blake2xb(counter; key=seed))
//   sample_poly_ternary    S/util/rlwe.cpp:23-41    (std::uniform_int_distribution<uint64_t>(0,2) over a 32-bit engine)
//   sample_poly_normal     S/util/rlwe.cpp:43-67    (ClippedNormalDistribution: std::normal_distribution, sigma 3.2, clip 19.2)
//   sample_poly_uniform    S/util/rlwe.cpp:107-135  (rejection below the largest multiple of the modulus)
// The std:: distributions are used as such (same libstdc++ as the reference build), only the engine is ours.
// The arithmetic around the samples (NTT, dyadic products, additions) runs on the GPU (b200_bfv.cu, sealc_api.cpp).
#pragma once
#include <array>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace b200
{
typedef std::array<uint64_t, 8> PrngSeed;

class Blake2xbPrng
{
public:
    explicit Blake2xbPrng(const PrngSeed &seed);
    void generate(size_t bytes, void *dst);
    uint32_t generate32()
    {
        uint32_t r;
        if (head_ + sizeof(r) <= buffer_.size())
        { // the common case inline: the distributions draw one 32-bit word at a time
            __builtin_memcpy(&r, buffer_.data() + head_, sizeof(r));
            head_ += sizeof(r);
            return r;
        }
        generate(sizeof(r), &r);
        return r;
    }
    const PrngSeed &seed() const { return seed_; }

private:
    void refill();
    PrngSeed seed_;
    uint64_t counter_ = 0;
    std::vector<unsigned char> buffer_;
    size_t head_;
};

// std-compatible engine over the PRNG (S/randomtostd.h:21-74)
struct PrngEngine
{
    typedef uint32_t result_type;
    Blake2xbPrng &g;
    explicit PrngEngine(Blake2xbPrng &p) : g(p) {}
    result_type operator()() { return g.generate32(); }
    static constexpr result_type min() { return 0; }
    static constexpr result_type max() { return 0xFFFFFFFFu; }
};

PrngSeed random_seed(); // from the operating system (std::random_device)

// out: [moduli.size()][n]
void sample_poly_ternary(Blake2xbPrng &prng, size_t n, const std::vector<uint64_t> &moduli, uint64_t *out);
void sample_poly_normal(Blake2xbPrng &prng, size_t n, const std::vector<uint64_t> &moduli, uint64_t *out);
void sample_poly_uniform(Blake2xbPrng &prng, size_t n, const std::vector<uint64_t> &moduli, uint64_t *out);

// BLAKE2b / BLAKE2Xb primitives (RFC 7693 and the BLAKE2X specification)
void blake2xb(void *out, size_t outlen, const void *in, size_t inlen, const void *key, size_t keylen);
} // namespace b200
