// emu_inline.cpp -- CPU replay of the hoisted rotations with inline hoist constants (TEST INFRASTRUCTURE): the emulator of
// emu_bank.cpp with a backend whose key-switch bodies are the INL variants (evab_set_hoist_inline on: the cadd operands are the
// elements' indicator rows, never moved by the key-bank offset, which applies to the keys only).  Built as its own library
// (tests/test_hoist_inline.py); the emui_* entry points are the emub_* ones issued through that backend.
#include "emu_bank.cpp"

struct InlineBE : BankBE {
  bool hoist_inline() const { return true; }
  int inner(const IpArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++)
      for (int j = 0; j < A.N; j += 2) {
        if (A.cadd) ks_inner_elem<true>(A, mi, j, 0, key_off());
        else ks_inner_elem(A, mi, j, 0, key_off());
      }
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    for (int i = 0; i < A.n; i++) for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) rot_many_elem<true>(A, i, mi, j, 0, key_off());
    return 0;
  }
};

extern "C" {
size_t emu_hoist_indicators_bytes(EmuCtx *c, int n) { return hoist_indicators_elems(c->v, n) * 8; }
int emu_hoist_indicators(EmuCtx *c, int n, const uint64_t *elts, uint64_t *out) {
  std::vector<const u32 *> ctabs;
  for (int g = 0; g < n; g++) {
    if (!c->cperms.count(elts[g])) evab_host::galois_coeff_table(c->v.N, elts[g], c->cperms[elts[g]]);
    ctabs.push_back(c->cperms[elts[g]].data());
  }
  EmuBE be{c};
  return hoist_indicators_impl(be, c->v, n, ctabs.data(), out);
}
int emui_rotate_modup_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key, const uint64_t *ind,
                               void *work) {
  InlineBE be{{{{c}}}};
  return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, emu_perm(c, elt), key, ind, (u64 *)work);
}
int emui_rotate_modup_many(EmuCtx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts, const uint64_t *const *keys,
                           const uint64_t *const *inds, void *work) {
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n && i < ROTMANY_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  InlineBE be{{{{c}}}};
  return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, inds, (u64 *)work);
}
int emui_rotate_wsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *inds, const uint64_t *const *wts, int ntap, const uint64_t *const *taps, const uint64_t *const *twts, void *work) {
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n && i < WS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  InlineBE be{{{{c}}}};
  return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, inds, wts, ntap, taps, twts, (u64 *)work);
}
int emui_lazy_rotsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                     const uint64_t *const *inds, const uint64_t *const *wts, void *work) {
  const u32 *perms[LRS_MAX];
  for (int i = 0; i < n && i < LRS_MAX; i++) perms[i] = emu_perm(c, elts[i]);
  InlineBE be{{{{c}}}};
  return lazy_rotsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, inds, wts, (u64 *)work);
}
}
