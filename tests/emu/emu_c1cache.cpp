// emu_c1cache.cpp -- CPU replay of the key switches with cached c1 rows (TEST INFRASTRUCTURE): the emulator of emu_seeded.cpp with
// a backend that reads a region table (evab_set_key_c1_rows; the emulator runs instance 0, which reads region[0]): region[0] >= 0
// fills the seeded bodies' tiles from the c1 rows at key + region[0] * stride (SeedTileHost::c1off), region[0] < 0 draws them.  The
// seeded flag can be turned off (emuc_set_key_seeded) for the refusals.  Built as its own library (tests/test_c1_cache.py); the
// emuc_* entry points are the emus_* ones issued through that backend, and emuc_expand_seeded_c1 runs evab_expand_seeded_c1's body.
#include "emu_seeded.cpp"

static const int32_t *g_c1 = nullptr;
static bool g_c1_seeded = true;

struct C1BE : SeededBE {
  bool key_seeded() const { return g_c1_seeded; }
  bool key_bank() const { return g_tenant != nullptr; }
  bool key_c1_rows() const { return g_c1 != nullptr; }
  long long c1_off() const { return g_c1 && g_c1[0] >= 0 ? (long long)g_c1[0] * g_kstride : -1; }
  int inner(const IpArgs &A) {
    const long long koff = key_off();
    const u64 *keys[1] = {A.key};
    seeded_replay<true>(keys, 1, koff, A.primes, A.ell, A.k, A.N, [&](int mi, int j, SeedTileHost *t) {
      if (A.cadd) ks_inner_elem<true, true>(A, mi, j, 0, koff, t);
      else ks_inner_elem<false, true>(A, mi, j, 0, koff, t);
    }, c1_off());
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    const long long koff = key_off();
    seeded_replay<true>(A.key, A.n, koff, A.primes, A.ell, A.k, A.N, [&](int mi, int j, SeedTileHost *t) {
      for (int i = 0; i < A.n; i++) rot_many_elem<true, true>(A, i, mi, j, 0, koff, t);
    }, c1_off());
    return 0;
  }
};
#define C1_BE C1BE be{{{{{{c}}}}}}

extern "C" {
int emuc_set_key_c1_rows(const int32_t *region_of_instance) { g_c1 = region_of_instance; return 0; }
int emuc_set_key_seeded(int on) { g_c1_seeded = on != 0; return 0; }
// evab_expand_seeded_c1's body over every (image, row, block of 8)
int emuc_expand_seeded_c1(EmuCtx *c, int n, const uint64_t *images, uint64_t *rows) {
  const int k = c->v.k;
  const size_t N = c->v.N;
  for (int i = 0; i < n; i++)
    for (int r = 0; r < (k - 1) * k; r++)
      for (u32 t = 0; t < N / 8; t++) expand_seeded_c1_elem(images, rows, c->v.primes, k, N, i, r, t);
  return 0;
}
int emuc_relinearize(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *key, void *work) {
  C1_BE;
  return relinearize_impl(be, c->v, ell, o, a, key, (u64 *)work);
}
int emuc_rotate(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, uint64_t elt, const uint64_t *key, void *work) {
  C1_BE;
  return rotate_impl(be, c->v, ell, o, a, emu_perm(c, elt), key, (u64 *)work);
}
int emuc_rotate_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *hoist, uint64_t elt, const uint64_t *key, void *work) {
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  C1_BE;
  return rotate_prepared_impl(be, c->v, ell, o, a, hoist, emu_perm(c, elt), c->cperms[elt].data(), key, (u64 *)work);
}
int emuc_rotate_modup_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key, const uint64_t *ind,
                               void *work) {
  C1_BE;
  return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, emu_perm(c, elt), key, ind, (u64 *)work);
}
int emuc_rotate_modup_many(EmuCtx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts, const uint64_t *const *keys,
                           const uint64_t *const *inds, void *work) {
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n && i < ROTMANY_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  C1_BE;
  return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, inds, (u64 *)work);
}
int emuc_rotate_wsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *inds, const uint64_t *const *wts, int ntap, const uint64_t *const *taps, const uint64_t *const *twts, void *work) {
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n && i < WS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  C1_BE;
  return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, inds, wts, ntap, taps, twts, (u64 *)work);
}
}
