// compact_kernels.cuh -- compact responses (evab_compact_ciphers and the client's evab_compact_unpack / evab_compact_finish):
// CKKS modulus switching of an output ciphertext from its RNS modulus Q to the power of two 2^b, then bit packing.
//
// For every coefficient x in [0, Q) of c0 and c1 (coefficient form), with shift sh >= b:
//   y = floor((2^(sh+1) x + Q) / (2Q)) mod 2^b
// Q is odd, so the rounding never ties.  Because 2^(sh+1) x = 2^(b+1) (2^(sh-b) x), only x' = 2^(sh-b) x mod Q matters:
//   y = floor((2^b x' + (Q-1)/2) / Q) mod 2^b
// x' is composed directly by the decoder's CRT (crt_compose) with every (Q/q_i)^-1 multiplied by 2^(sh-b) mod q_i, and the
// quotient is an exact division: one 128-by-64 division for ell = 1, a restoring bit-serial division by the multi-word Q otherwise
// (b quotient bits, the remainder kept below Q).  Packed layout: polynomial j is a little-endian bit stream of N b-bit fields at
// words [j W, (j+1) W), W = ceil(N b / 64), unused high bits of the last word zero.
//
// Bodies are __host__ __device__ so the CPU emulator (tests/emu/emu_compact.cpp) replays them.
#pragma once
#include "encode_kernels.cuh"

#define CMP_MAX_ENTRIES 256   // output values per compaction launch (pointers by value in the launch arguments)
#define CMP_THREADS 256

struct CompactArgs {
  CrtTables T;                  // of the first ell primes, ipunct[i] multiplied by 2^(sh-b) mod q_i
  u64 hhi[DEC_WORDS];           // (Q-1)/2 >> b
  u64 hlo;                      // (Q-1)/2 mod 2^b
  const PrimeDev *primes;
  const u64 *src;               // [count][2][ell][N] coefficient form
  u64 *dst[CMP_MAX_ENTRIES];    // [2][W] each
  u32 N, ell, bits, words;      // words: W
};

// the rounded value y of coefficient i of polynomial `poly` ([ell][N] coefficient form), 0 <= y < 2^b
EVAB_HD u64 compact_coeff(const CompactArgs &A, const u64 *poly, u32 i) {
  const int nw = (int)A.ell + 1;
  const u32 b = A.bits;
  u64 R[DEC_WORDS];
  crt_compose(A.T, A.primes, A.ell, poly + i, A.N, R);   // x' in [0, Q)
  const u64 mask = (1ull << b) - 1;
  if (A.ell == 1) {
    typedef unsigned __int128 u128;
    const u128 num = ((u128)R[0] << b) + (((u128)A.hhi[0] << b) | A.hlo);
    return (u64)(num / A.T.Q[0]) & mask;
  }
  // R = x' + hhi: then (R 2^b + hlo) / Q, one quotient bit per step (the top one, 2^b, vanishes mod 2^b)
  u64 carry = 0;
  for (int w = 0; w < nw; w++) { const u64 s = R[w] + A.hhi[w], c1 = s < R[w]; R[w] = s + carry; carry = c1 | (R[w] < s); }
  if (dec_cmp(R, A.T.Q, nw) >= 0) dec_sub(R, A.T.Q, nw);
  u64 y = 0;
  for (int t = (int)b - 1; t >= 0; t--) {
    for (int w = nw - 1; w > 0; w--) R[w] = (R[w] << 1) | (R[w - 1] >> 63);   // R < Q: 2 R + 1 fits in ell + 1 words
    R[0] = (R[0] << 1) | ((A.hlo >> t) & 1);
    if (dec_cmp(R, A.T.Q, nw) >= 0) { dec_sub(R, A.T.Q, nw); y |= 1ull << t; }
  }
  return y;
}

// output word w of polynomial `poly` (0: c0, 1: c1) of entry e: the thread computes every coefficient that overlaps the word
EVAB_HD void compact_word(const CompactArgs &A, u32 e, u32 poly, u32 w) {
  const u32 b = A.bits;
  const u64 *src = A.src + ((size_t)e * 2 + poly) * A.ell * A.N;
  const u64 bit0 = (u64)w * 64;
  const u64 first = bit0 / b;
  u64 last = (bit0 + 63) / b;
  if (last > A.N - 1) last = A.N - 1;
  u64 out = 0;
  for (u64 i = first; i <= last; i++) {
    const u64 y = compact_coeff(A, src, (u32)i);
    const long long off = (long long)(i * b) - (long long)bit0;   // -b < off < 64
    out |= off >= 0 ? y << off : y >> -off;
  }
  A.dst[e][(size_t)poly * A.words + w] = out;
}

// host: the constants of a compaction of ell-residue values over primes[0 .. ell) (primes, src and dst are the caller's):
// (Q/q_i)^-1 multiplied by 2^(shift-bits) mod q_i, and (Q-1)/2 split at bit `bits`
inline void compact_args(CompactArgs &A, const u64 *primes, int ell, int shift, int bits, u32 N) {
  typedef unsigned __int128 u128;
  memset(&A, 0, sizeof(A));
  crt_tables(A.T, primes, ell);
  for (int i = 0; i < ell; i++) {
    const u64 p = primes[i];
    u64 r = 1, base = 2 % p;
    for (long long e = (long long)shift - bits; e; e >>= 1) { if (e & 1) r = (u64)((u128)r * base % p); base = (u64)((u128)base * base % p); }
    A.T.ipunct[i] = (u64)((u128)A.T.ipunct[i] * r % p);
  }
  const int nw = ell + 1;
  u64 h[DEC_WORDS];                                   // (Q - 1) / 2 = halfQ - 1
  for (int w = 0; w < nw; w++) h[w] = A.T.halfQ[w];
  for (int w = 0; w < nw; w++) if (h[w]--) break;
  A.hlo = h[0] & ((1ull << bits) - 1);
  for (int w = 0; w < nw; w++) A.hhi[w] = (h[w] >> bits) | (w + 1 < nw ? h[w + 1] << (64 - bits) : 0);
  A.N = N; A.ell = (u32)ell; A.bits = (u32)bits; A.words = (u32)(((u64)N * bits + 63) / 64);
}

// ---- client side
// field i of a packed polynomial
EVAB_HD u64 compact_field(const u64 *words, u32 b, u32 i) {
  const u64 bit = (u64)i * b;
  const u32 w = (u32)(bit >> 6), off = (u32)(bit & 63);
  u64 v = words[w] >> off;
  if (off + b > 64) v |= words[w + 1] << (64 - off);
  return v & ((1ull << b) - 1);
}
// coefficient i of both polynomials of a packed value [2][W] -> residues mod primes 0 .. nres-1: out [2][nres][N]
EVAB_HD void compact_unpack_elem(const u64 *words, u32 b, u32 W, const PrimeDev *primes, u32 nres, u32 N, u64 *out, u32 i) {
  for (u32 j = 0; j < 2; j++) {
    const u64 y = compact_field(words + (size_t)j * W, b, i);
    for (u32 r = 0; r < nres; r++) out[((size_t)j * nres + r) * N + i] = barrett64(y, primes[r].p, primes[r].ratio64);
  }
}
// coefficient i of y0 + y1 s ([nres][N] coefficient form, exact: the primes' product exceeds 2 (N+1) 2^b) -> the centred value
// z in (-2^(b-1), 2^(b-1)] of it mod 2^b -> zout[i] (if not null) and residues mod primes 0 .. nout-1 (out [nout][N])
EVAB_HD void compact_finish_elem(const CrtTables &T, const PrimeDev *primes, u32 nres, u32 N, u32 b, const u64 *coef, u32 nout, u64 *out,
                                 long long *zout, u32 i) {
  const int nw = (int)nres + 1;
  u64 X[DEC_WORDS];
  crt_compose(T, primes, nres, coef + i, N, X);
  const bool neg = dec_cmp(X, T.halfQ, nw) >= 0;   // the centred lift is X - P: its low b bits are those of X[0] - P[0]
  const u64 m = (X[0] - (neg ? T.Q[0] : 0)) & ((1ull << b) - 1);
  const long long z = m > (1ull << (b - 1)) ? (long long)m - (1ll << b) : (long long)m;
  if (zout) zout[i] = z;
  const u64 mag = z < 0 ? (u64)(-z) : (u64)z;
  for (u32 r = 0; r < nout; r++) {
    const u64 v = barrett64(mag, primes[r].p, primes[r].ratio64);
    out[(size_t)r * N + i] = (z < 0 && v) ? primes[r].p - v : v;
  }
}
