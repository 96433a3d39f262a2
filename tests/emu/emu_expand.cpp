// emu_expand.cpp -- CPU replay of evab_expand_key_uniform (TEST INFRASTRUCTURE): the element body of key_expand.cuh run serially,
// the shared ChaCha20 block function, and the host CSPRNG built on it (tests/test_compressed_keys.py).
#include "../../eva_b200/csrc/key_expand.cuh"
#include "../../eva_b200/csrc/host/csprng.hpp"

extern "C" {
void emu_chacha20_block(const uint32_t *key, uint64_t counter, uint64_t nonce, uint32_t *out) { chacha20_block(key, counter, nonce, out); }
// the first `count` outputs of the deterministic host stream of `seed` (csprng.hpp ChaChaRng)
void emu_chacha_rng(uint64_t seed, int count, uint64_t *out) {
  evab::ChaChaRng r(seed);
  for (int i = 0; i < count; i++) out[i] = r();
}
int emu_expand_key_uniform(uint32_t N, int k, int n, const uint8_t *seeds, const uint64_t *moduli, uint64_t *keys) {
  if (k < 2 || k > KX_MAXK || n < 1 || N % 8) return 1;
  ExpandArgs A{};
  A.seeds = reinterpret_cast<const uint32_t *>(seeds); A.keys = keys; A.N = N; A.k = (uint32_t)k;
  for (int m = 0; m < k; m++) { A.q[m] = moduli[m]; A.lim[m] = kx_limit(moduli[m]); }
  for (int g = 0; g < n; g++)
    for (uint32_t r = 0; r < (uint32_t)((k - 1) * k); r++)
      for (uint32_t t = 0; t < N / 8; t++) expand_uniform_elem(A, g, r, t);
  return 0;
}
}
