// key_expand.cuh -- the uniform halves of seed-compressed key-switch keys (DESIGN §2, "Seed-compressed evaluation keys") and of
// seed-compressed input ciphertexts (the same rule with other row ids, at the end of this file).
//
// Digit J of a key-switch key [k-1][2][k][N] is (c0, c1) = (-(a s + e) + P [J] s', a), where a is uniform public randomness.  A
// compressed key keeps c0 and a 32-byte seed; its (k-1) k rows of c1 are rebuilt from the seed alone by this rule:
//   block(seed, counter, nonce)  the ChaCha20 block function of RFC 8439 (20 rounds, output = rounds(x) + x) on the state
//                                constants (words 0-3), the seed as 8 little-endian key words (4-11), a 64-bit block counter
//                                (12-13) and a 64-bit nonce (14-15)
//   candidate i of a block       w[2i] | w[2i+1] << 32, i = 0 .. 7
//   row r = J k + m              digit J, prime index m (m = k-1: the special prime), modulus q = q_m
//   primary draw                 coefficient j of row r takes candidate j mod 8 of block(seed, j / 8, r)
//   acceptance                   v < q floor((2^64-1) / q) (= q floor(2^64 / q) for every q that is not a power of two); the
//                                value is then v mod q, without modulo bias
//   fallback                     a rejected coefficient reads the candidates of block(seed, j 256 + t, 2^63 | r), t = 0 .. 255,
//                                in order and takes the first accepted one (all 2048 rejected, probability < 2^-2048: the last
//                                candidate mod q)
// Each coefficient depends on (seed, r, j) only, so a key expands in one parallel pass.  The block function is also the host
// CSPRNG's (host/csprng.hpp), and tests/emu/emu_expand.cpp (key rows) and tests/emu/emu_cipher_expand.cpp (ciphertext rows) replay
// this file on the CPU.
#pragma once
#include <stddef.h>
#include <stdint.h>

#ifndef EVAB_HD
#if defined(__CUDACC__)
#define EVAB_HD __host__ __device__ __forceinline__
#else
#define EVAB_HD inline
#endif
#endif

EVAB_HD uint32_t chacha_rotl(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }
EVAB_HD void chacha_qr(uint32_t *s, int a, int b, int c, int d) {
  s[a] += s[b]; s[d] ^= s[a]; s[d] = chacha_rotl(s[d], 16);
  s[c] += s[d]; s[b] ^= s[c]; s[b] = chacha_rotl(s[b], 12);
  s[a] += s[b]; s[d] ^= s[a]; s[d] = chacha_rotl(s[d], 8);
  s[c] += s[d]; s[b] ^= s[c]; s[b] = chacha_rotl(s[b], 7);
}
// out[16] = ChaCha20 block of (key[8], 64-bit counter, 64-bit nonce)
EVAB_HD void chacha20_block(const uint32_t *key, uint64_t counter, uint64_t nonce, uint32_t *out) {
  uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u,   // "expand 32-byte k"
                    key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                    (uint32_t)counter, (uint32_t)(counter >> 32), (uint32_t)nonce, (uint32_t)(nonce >> 32)};
  uint32_t x[16];
#pragma unroll
  for (int i = 0; i < 16; i++) x[i] = s[i];
#pragma unroll
  for (int i = 0; i < 10; i++) {
    chacha_qr(x, 0, 4, 8, 12); chacha_qr(x, 1, 5, 9, 13); chacha_qr(x, 2, 6, 10, 14); chacha_qr(x, 3, 7, 11, 15);
    chacha_qr(x, 0, 5, 10, 15); chacha_qr(x, 1, 6, 11, 12); chacha_qr(x, 2, 7, 8, 13); chacha_qr(x, 3, 4, 9, 14);
  }
#pragma unroll
  for (int i = 0; i < 16; i++) out[i] = x[i] + s[i];
}

#define KX_MAXK 64                        // primes per key (the moduli travel in the kernel arguments)
#define KX_FALLBACK_BLOCKS 256u
#define KX_FALLBACK_NONCE (1ull << 63)
// largest accepted candidate + 1 for modulus q >= 2
EVAB_HD uint64_t kx_limit(uint64_t q) { return q * (~0ull / q); }

struct ExpandArgs {
  const uint32_t *seeds;                  // [n][8] key words (32 bytes per key)
  uint64_t *keys;                         // [n][k-1][2][k][N]: only the c1 rows are written
  uint64_t q[KX_MAXK], lim[KX_MAXK];      // modulus of prime index m, kx_limit(q)
  uint32_t N, k;
};

// The reduction of an accepted candidate v < lim is a parameter of the draw: any exact v mod q gives the same value.  KxRem is the
// rule as written (v % q); the key-switch inner products of seeded keys (ops_kernels.cuh seeded_c1_draw8) pass a Barrett reducer.
struct KxRem {
  uint64_t q;
  EVAB_HD uint64_t operator()(uint64_t v) const { return v % q; }
};

// coefficient j of row r, rejected in the primary draw: the fallback search
template <class Red> EVAB_HD uint64_t kx_fallback(const uint32_t *key, const Red &red, uint64_t lim, uint64_t r, uint32_t j) {
  uint32_t w[16];
  uint64_t v = 0;
  for (uint32_t t = 0; t < KX_FALLBACK_BLOCKS; t++) {
    chacha20_block(key, (uint64_t)j * KX_FALLBACK_BLOCKS + t, KX_FALLBACK_NONCE | r, w);
    for (int i = 0; i < 8; i++) {
      v = (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32);
      if (v < lim) return red(v);
    }
  }
  return red(v);
}
EVAB_HD uint64_t kx_fallback(const uint32_t *key, uint64_t q, uint64_t lim, uint64_t r, uint32_t j) { return kx_fallback(key, KxRem{q}, lim, r, j); }

// the rule's draw, shared by key rows and ciphertext rows: coefficients 8 t .. 8 t + 7 of row r (lim = kx_limit(q), red: v mod q)
// from one primary block, a rejected candidate replaced by its fallback search
template <class Red> EVAB_HD void kx_draw8(const uint32_t *key, uint64_t r, uint32_t t, const Red &red, uint64_t lim, uint64_t *v) {
  uint32_t w[16];
  chacha20_block(key, t, r, w);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint64_t c = (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32);
    v[i] = c < lim ? red(c) : kx_fallback(key, red, lim, r, 8 * t + i);
  }
}
EVAB_HD void kx_draw8(const uint32_t *key, uint64_t r, uint32_t t, uint64_t q, uint64_t lim, uint64_t *v) { kx_draw8(key, r, t, KxRem{q}, lim, v); }

// 8 coefficients to dst (64-byte aligned: N is a multiple of 8 and rows start on 64-byte boundaries): 16-byte stores on the device
EVAB_HD void kx_store8(uint64_t *dst, const uint64_t *v) {
#if defined(__CUDA_ARCH__)
  ulonglong2 *d2 = reinterpret_cast<ulonglong2 *>(dst);
#pragma unroll
  for (int i = 0; i < 4; i++) d2[i] = make_ulonglong2(v[2 * i], v[2 * i + 1]);
#else
  for (int i = 0; i < 8; i++) dst[i] = v[i];
#endif
}

// key g, row r, coefficients 8 t .. 8 t + 7: one primary block
EVAB_HD void expand_uniform_elem(const ExpandArgs &A, uint32_t g, uint32_t r, uint32_t t) {
  uint32_t key[8];
  const uint32_t *sk = A.seeds + (size_t)g * 8;
#pragma unroll
  for (int i = 0; i < 8; i++) key[i] = sk[i];
  const uint32_t J = r / A.k, m = r % A.k;
  uint64_t v[8];
  kx_draw8(key, r, t, A.q[m], A.lim[m], v);
  kx_store8(A.keys + (size_t)g * (A.k - 1) * 2 * A.k * A.N + ((size_t)(2 * J + 1) * A.k + m) * A.N + (size_t)8 * t, v);
}

// ---- seed-compressed ciphertexts (DESIGN §2, "Seed-compressed input ciphertexts").  A fresh secret-key encryption
// (c0, c1) = (-(a s + e) + m, a) at level ell keeps c0 and a 32-byte seed; its ell rows of c1 follow the same rule with their own
// row ids:
//   row id of ciphertext row m   r = 2^62 | m (prime index m < ell, modulus q_m); key rows are r = J k + m < 2^12, so a key and
//                                a ciphertext never share a ChaCha stream, even under the same seed.  The fallback nonce is
//                                2^63 | r as for keys
//   primary draw                 coefficient j of row m takes candidate j mod 8 of block(seed, j / 8, 2^62 | m)
#define KX_CIPHER_ROW (1ull << 62)
#define CX_MAX_ENTRIES 56                 // ciphertexts per launch: the arguments stay under 4 KB of kernel parameters

struct CipherExpandEntry {
  uint32_t seed[8];                       // 32 bytes, as 8 little-endian key words
  uint64_t *c1;                           // the ell rows [ell][N] of c1 (the ciphertext [2][ell][N] starts ell N words before)
  uint32_t ell;
};
struct CipherExpandArgs {
  uint64_t q[KX_MAXK], lim[KX_MAXK];      // modulus of prime index m, kx_limit(q)
  CipherExpandEntry e[CX_MAX_ENTRIES];
  uint32_t N;
};
#if defined(__cplusplus) && __cplusplus >= 201103L
static_assert(sizeof(CipherExpandArgs) <= 4096, "the ciphertext expansion's arguments must fit the classic 4 KB parameter space");
#endif

// entry i, row m < e[i].ell, coefficients 8 t .. 8 t + 7
EVAB_HD void expand_cipher_elem(const CipherExpandArgs &A, uint32_t i, uint32_t m, uint32_t t) {
  uint32_t key[8];
#pragma unroll
  for (int w = 0; w < 8; w++) key[w] = A.e[i].seed[w];
  uint64_t v[8];
  kx_draw8(key, KX_CIPHER_ROW | m, t, A.q[m], A.lim[m], v);
  kx_store8(A.e[i].c1 + (size_t)m * A.N + (size_t)8 * t, v);
}
