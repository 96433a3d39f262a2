// emu_bank.cpp -- CPU replay of the key-switch ops with per-instance key selection (TEST INFRASTRUCTURE): the emulator of
// emu_wsum.cpp with a backend whose key-switch bodies take the key-bank offset of the replayed instance (evab_set_key_bank;
// the emulator runs instance 0, which reads tenant[0]).  Built as its own library (tests/test_tenants.py); the emub_* entry
// points are the emu_* ones of the key-switch ops, issued through that backend.
#include "emu_wsum.cpp"

static const int32_t *g_tenant = nullptr;
static long long g_kstride = 0;

struct BankBE : WsumBE {
  long long key_off() const { return g_tenant ? (long long)g_tenant[0] * g_kstride : 0; }
  int inner(const IpArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++)
      for (int j = 0; j < A.N; j += 2) ks_inner_elem(A, mi, j, 0, key_off());
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    for (int i = 0; i < A.n; i++) for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) rot_many_elem(A, i, mi, j, 0, key_off());
    return 0;
  }
  int lazy_rotsum(const LazyRotSumArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) {
      u64 sum[LRS_OUT][4] = {}, part[LRS_OUT][4];
      for (int i = 0; i < A.n; i++) { lazy_rotsum_part(A, mi, j, i, 0, part, key_off()); for (int o = 0; o < A.nout; o++) for (int c = 0; c < 4; c++) sum[o][c] += part[o][c]; }
      for (int o = 0; o < A.nout; o++) lazy_rotsum_store(A, mi, j, o, 0, sum[o]);
    }
    return 0;
  }
};

static const u32 *emu_perm(EmuCtx *c, u64 elt) {
  if (!c->perms.count(elt)) evab_host::galois_table(c->v.N, c->v.logN, elt, c->perms[elt]);
  return c->perms[elt].data();
}

extern "C" {
int emu_set_key_bank(const int32_t *tenant_of_instance, size_t tenant_stride_words) {
  g_tenant = tenant_of_instance; g_kstride = tenant_of_instance ? (long long)tenant_stride_words : 0;
  return 0;
}
int emub_relinearize(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *key, void *work) {
  BankBE be{{{c}}};
  return relinearize_impl(be, c->v, ell, o, a, key, (u64 *)work);
}
int emub_rotate(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, uint64_t elt, const uint64_t *key, void *work) {
  BankBE be{{{c}}};
  return rotate_impl(be, c->v, ell, o, a, emu_perm(c, elt), key, (u64 *)work);
}
int emub_rotate_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *hoist, uint64_t elt, const uint64_t *key, void *work) {
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  BankBE be{{{c}}};
  return rotate_prepared_impl(be, c->v, ell, o, a, hoist, emu_perm(c, elt), c->cperms[elt].data(), key, (u64 *)work);
}
int emub_rotate_modup_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key, const uint64_t *cadd,
                               void *work) {
  BankBE be{{{c}}};
  return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, emu_perm(c, elt), key, cadd, (u64 *)work);
}
int emub_rotate_modup_many(EmuCtx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts, const uint64_t *const *keys,
                           const uint64_t *const *cadds, void *work) {
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n && i < ROTMANY_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  BankBE be{{{c}}};
  return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, cadds, (u64 *)work);
}
int emub_lazy_rotsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *cadds, const uint64_t *const *wts, void *work) {
  const u32 *perms[LRS_MAX];
  for (int i = 0; i < n && i < LRS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  BankBE be{{{c}}};
  return lazy_rotsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, (u64 *)work);
}
int emub_rotate_wsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *cadds, const uint64_t *const *wts, int ntap, const uint64_t *const *taps, const uint64_t *const *twts, void *work) {
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n && i < WS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  BankBE be{{{c}}};
  return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, ntap, taps, twts, (u64 *)work);
}
}
