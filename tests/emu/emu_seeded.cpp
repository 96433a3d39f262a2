// emu_seeded.cpp -- CPU replay of the key switches with seeded keys (TEST INFRASTRUCTURE): the emulator of emu_inline.cpp with a
// backend whose key-switch bodies are the SEED variants (evab_set_key_seeded on: every key operand is a seeded image, c0 rows then
// the seed, and the c1 words are drawn into SeedTileHost tiles by seeded_c1_draw8, the code the kernels run).  The inline hoist
// constants are on unless emus_set_hoist_inline(0) (the refusal of the hoisted calls).  Built as its own library
// (tests/test_seeded_slots.py); the emus_* entry points are the emub_* / emui_* ones issued through that backend.
#include "emu_inline.cpp"

static bool g_seeded_inline = true;

struct SeededBE : InlineBE {
  bool key_seeded() const { return true; }
  bool hoist_inline() const { return g_seeded_inline; }
  int inner(const IpArgs &A) {
    const long long koff = key_off();
    const u64 *keys[1] = {A.key};
    seeded_replay<true>(keys, 1, koff, A.primes, A.ell, A.k, A.N, [&](int mi, int j, SeedTileHost *t) {
      if (A.cadd) ks_inner_elem<true, true>(A, mi, j, 0, koff, t);
      else ks_inner_elem<false, true>(A, mi, j, 0, koff, t);
    });
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    const long long koff = key_off();
    seeded_replay<true>(A.key, A.n, koff, A.primes, A.ell, A.k, A.N, [&](int mi, int j, SeedTileHost *t) {
      for (int i = 0; i < A.n; i++) rot_many_elem<true, true>(A, i, mi, j, 0, koff, t);
    });
    return 0;
  }
};
#define SEEDED_BE SeededBE be{{{{{c}}}}}

extern "C" {
int emus_set_hoist_inline(int on) { g_seeded_inline = on != 0; return 0; }
size_t emus_seeded_key_words(int k, size_t N) { return seeded_key_words(k, N); }
// the c1 rows [k-1][k][N] of the seeded image `key` (k primes, moduli of c): what the seeded bodies draw, through seeded_c1_draw8
int emus_draw_c1(EmuCtx *c, const uint64_t *key, uint64_t *out) {
  const int k = c->v.k;
  const size_t N = c->v.N;
  uint32_t seed[8];
  seeded_seed(key, k, N, seed);
  for (int J = 0; J < k - 1; J++)
    for (int m = 0; m < k; m++) {
      const PrimeDev &P = c->v.primes[m];
      for (u32 t = 0; t < N / 8; t++) seeded_c1_draw8(seed, J, m, k, P, kx_limit(P.p), t, out + ((size_t)J * k + m) * N + 8 * t);
    }
  return 0;
}
// the rule's draw with an exact `%` reducer for arbitrary moduli (q[m] < 2^64, rows J k + m): the acceptance test and the fallback
// search of key_expand.cuh at high rejection rates, as the seeded draw runs them
int emus_draw_rows_rem(const uint8_t *seed32, int k, uint32_t N, const uint64_t *q, uint64_t *out) {
  uint32_t seed[8];
  std::memcpy(seed, seed32, 32);
  for (int J = 0; J < k - 1; J++)
    for (int m = 0; m < k; m++)
      for (u32 t = 0; t < N / 8; t++) kx_draw8(seed, (uint64_t)J * k + m, t, KxRem{q[m]}, kx_limit(q[m]), out + ((size_t)J * k + m) * N + 8 * t);
  return 0;
}
// barrett64 (the seeded draw's reducer) against % on n values of a ring prime of c
int emus_barrett_vs_rem(EmuCtx *c, int m, const uint64_t *v, int n, uint64_t *out) {
  const KxBarrett red{c->v.primes[m]};
  for (int i = 0; i < n; i++) out[i] = red(v[i]);
  return 0;
}
int emus_relinearize(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *key, void *work) {
  SEEDED_BE;
  return relinearize_impl(be, c->v, ell, o, a, key, (u64 *)work);
}
int emus_rotate(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, uint64_t elt, const uint64_t *key, void *work) {
  SEEDED_BE;
  return rotate_impl(be, c->v, ell, o, a, emu_perm(c, elt), key, (u64 *)work);
}
int emus_rotate_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *hoist, uint64_t elt, const uint64_t *key, void *work) {
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  SEEDED_BE;
  return rotate_prepared_impl(be, c->v, ell, o, a, hoist, emu_perm(c, elt), c->cperms[elt].data(), key, (u64 *)work);
}
int emus_rotate_modup_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key, const uint64_t *ind,
                               void *work) {
  SEEDED_BE;
  return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, emu_perm(c, elt), key, ind, (u64 *)work);
}
int emus_rotate_modup_many(EmuCtx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts, const uint64_t *const *keys,
                           const uint64_t *const *inds, void *work) {
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n && i < ROTMANY_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  SEEDED_BE;
  return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, inds, (u64 *)work);
}
int emus_rotate_wsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *inds, const uint64_t *const *wts, int ntap, const uint64_t *const *taps, const uint64_t *const *twts, void *work) {
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n && i < WS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  SEEDED_BE;
  return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, inds, wts, ntap, taps, twts, (u64 *)work);
}
int emus_lazy_rotsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *inds, const uint64_t *const *wts, void *work) {
  const u32 *perms[LRS_MAX];
  for (int i = 0; i < n && i < LRS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  SEEDED_BE;
  return lazy_rotsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, inds, wts, (u64 *)work);
}
int emus_rotate_hoist_const(EmuCtx *c, int ell, uint64_t elt, const uint64_t *key, uint64_t *out, void *tmp) {
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  SEEDED_BE;
  return hoist_const_impl(be, c->v, ell, c->cperms[elt].data(), key, out, (u64 *)tmp);
}
}
