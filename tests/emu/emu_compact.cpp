// emu_compact.cpp -- CPU replay of the compact-response elements (TEST INFRASTRUCTURE): the compaction word body of
// evab_compact_ciphers and the client bodies of evab_compact_unpack / evab_compact_finish, from compact_kernels.cuh, run serially
// (tests/test_compact_outputs.py).  The inputs are already in coefficient form (the device call's inverse transform is not replayed).
#include <vector>
#include "../../eva_b200/csrc/compact_kernels.cuh"

static std::vector<PrimeDev> prime_devs(const uint64_t *primes, int n) {
  typedef unsigned __int128 u128;
  std::vector<PrimeDev> P(n);
  for (int i = 0; i < n; i++) {
    memset(&P[i], 0, sizeof(PrimeDev));
    P[i].p = primes[i];
    const u128 ratio = ~(u128)0 / primes[i];
    P[i].ratio_lo = (u64)ratio; P[i].ratio_hi = (u64)(ratio >> 64);
    P[i].ratio64 = (u64)(((u128)1 << 64) / primes[i]);
  }
  return P;
}

extern "C" {
// one value: coef [2][ell][N] (coefficient form) -> dst [2][W]
int emu_compact(uint32_t N, int ell, const uint64_t *primes, int shift, int bits, const uint64_t *coef, uint64_t *dst) {
  if (ell < 1 || ell > DEC_MAX_ELL || bits < 1 || bits > 62 || shift < bits) return 1;
  std::vector<PrimeDev> P = prime_devs(primes, ell);
  CompactArgs A;
  compact_args(A, primes, ell, shift, bits, N);
  A.primes = P.data(); A.src = coef; A.dst[0] = dst;
  for (uint32_t poly = 0; poly < 2; poly++)
    for (uint32_t w = 0; w < A.words; w++) compact_word(A, 0, poly, w);
  return 0;
}
// words [2][W] -> out [2][nres][N]
int emu_compact_unpack(uint32_t N, int nres, const uint64_t *primes, int bits, const uint64_t *words, uint64_t *out) {
  if (nres < 1 || nres > DEC_MAX_ELL || bits < 1 || bits > 62) return 1;
  std::vector<PrimeDev> P = prime_devs(primes, nres);
  const uint32_t W = (uint32_t)(((uint64_t)N * bits + 63) / 64);
  for (uint32_t i = 0; i < N; i++) compact_unpack_elem(words, (u32)bits, W, P.data(), (u32)nres, N, out, i);
  return 0;
}
// coef [nres][N] (y0 + y1 s, coefficient form) -> out [nout][N], z [N]
int emu_compact_finish(uint32_t N, int nres, const uint64_t *primes, int bits, const uint64_t *coef, int nout, uint64_t *out, int64_t *z) {
  if (nres < 1 || nres > DEC_MAX_ELL || nout < 1 || nout > DEC_MAX_ELL || bits < 1 || bits > 62) return 1;
  std::vector<PrimeDev> P = prime_devs(primes, nres > nout ? nres : nout);
  CrtTables T;
  crt_tables(T, primes, nres);
  for (uint32_t i = 0; i < N; i++) compact_finish_elem(T, P.data(), (u32)nres, N, (u32)bits, coef, (u32)nout, out, (long long *)z, i);
  return 0;
}
}
