// emu_cipher_expand.cpp -- CPU replay of evab_expand_cipher_uniform (TEST INFRASTRUCTURE): the ciphertext-row element body of
// key_expand.cuh run serially (tests/test_seeded_inputs.py).
#include <cstring>
#include "../../eva_b200/csrc/key_expand.cuh"

extern "C" {
// entry i writes ell[i] rows [ell[i]][N] at c1[i] from seeds[i] (32 bytes), row m modulo moduli[m]
int emu_expand_cipher_uniform(uint32_t N, int n, const uint8_t *seeds, uint64_t *const *c1, const int *ell, const uint64_t *moduli) {
  if (n < 1 || N % 8) return 1;
  CipherExpandArgs A{};
  A.N = N;
  for (int i = 0; i < n; i++) {
    if (ell[i] < 1 || ell[i] > KX_MAXK - 1) return 1;
    for (int m = 0; m < ell[i]; m++) { A.q[m] = moduli[m]; A.lim[m] = kx_limit(moduli[m]); }
    std::memcpy(A.e[0].seed, seeds + (size_t)32 * i, 32);
    A.e[0].c1 = c1[i]; A.e[0].ell = (uint32_t)ell[i];
    for (uint32_t m = 0; m < (uint32_t)ell[i]; m++)
      for (uint32_t t = 0; t < N / 8; t++) expand_cipher_elem(A, 0, m, t);
  }
  return 0;
}
}
