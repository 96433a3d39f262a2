// csprng.hpp -- the randomness of key generation and encryption (secret key, encryption masks, error
// polynomials, the uniform half of the public key, and the 32-byte seeds from which the device expands the uniform halves
// of the relinearization / Galois keys, key_expand.cuh).
//
// The reference samples from SEAL's Blake2/SHAKE CSPRNG seeded with 512 bits.  This backend uses the ChaCha20
// block function (RFC 8439) as a stream generator keyed with 256 bits from the operating system (getrandom(2),
// /dev/urandom as a fallback).  A non-zero `seed` selects a DETERMINISTIC stream derived from that 64-bit value:
// it exists for reproducible tests and fixtures only and carries at most 64 bits of security.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include "../key_expand.cuh"
#if defined(__linux__)
#include <sys/random.h>
#endif

namespace evab {

class ChaChaRng {
public:
  explicit ChaChaRng(std::uint64_t seed) {
    std::uint32_t key[8];
    if (seed == 0) {
      osEntropy(key, sizeof(key));
      deterministic_ = false;
    } else {   // test-only: SplitMix64 expansion of the seed
      std::uint64_t x = seed;
      for (int i = 0; i < 4; i++) {
        x += 0x9E3779B97F4A7C15ull;
        std::uint64_t z = x;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
        key[2 * i] = (std::uint32_t)z; key[2 * i + 1] = (std::uint32_t)(z >> 32);
      }
      deterministic_ = true;
    }
    std::memcpy(key_, key, 32);   // the block counter starts at 0, the nonce is 0 (one stream per key)
    pos_ = 16;
    std::memset(key, 0, sizeof(key));
  }
  bool deterministic() const { return deterministic_; }
  std::uint64_t operator()() {
    if (pos_ + 2 > 16) refill();
    const std::uint64_t v = (std::uint64_t)block_[pos_] | ((std::uint64_t)block_[pos_ + 1] << 32);
    pos_ += 2;
    return v;
  }
  // uniform in [0, bound) by rejection (no modulo bias)
  std::uint64_t below(std::uint64_t bound) {
    const std::uint64_t lim = ~0ull - (~0ull % bound + 1) % bound;   // largest multiple of bound, minus one
    std::uint64_t v;
    do { v = (*this)(); } while (v > lim);
    return v % bound;
  }

private:
  void refill() {
    chacha20_block(key_, counter_++, 0, block_);
    pos_ = 0;
  }
  static void osEntropy(void *buf, std::size_t n) {
#if defined(__linux__)
    std::size_t got = 0;
    while (got < n) {
      const ssize_t r = getrandom((char *)buf + got, n - got, 0);
      if (r <= 0) break;
      got += (std::size_t)r;
    }
    if (got == n) return;
#endif
    std::FILE *f = std::fopen("/dev/urandom", "rb");
    if (!f || std::fread(buf, 1, n, f) != n) { if (f) std::fclose(f); throw std::runtime_error("no entropy source (getrandom / /dev/urandom)"); }
    std::fclose(f);
  }
  std::uint32_t key_[8], block_[16];
  std::uint64_t counter_ = 0;
  int pos_;
  bool deterministic_;
};

}  // namespace evab
