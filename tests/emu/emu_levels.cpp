// emu_levels.cpp -- CPU replay of evab_rotate_hoist_const_levels (TEST INFRASTRUCTURE): the emulator of emu.cpp with a backend
// that also runs the all-levels hoist-constant body (hoist_levels_elem) serially.  Built as its own library
// (tests/test_hoist_const_levels.py).
#include "emu.cpp"

struct LevelsBE : EmuBE {
  int hoist_levels(const HoistLevelsArgs &A, int n) {
    for (int g = 0; g < n; g++) for (int m = 0; m < A.k; m++) for (int j = 0; j < A.N; j += 2) hoist_levels_elem(A, g, m, j);
    return 0;
  }
};

extern "C" {
size_t emu_hoist_const_levels_bytes(EmuCtx *c) { return hoist_levels_words(c->v.k, c->v.N) * 8; }
size_t emu_rotate_hoist_const_levels_work_bytes(EmuCtx *c, int n) { return hoist_const_levels_work_elems(c->v, n) * 8; }
int emu_rotate_hoist_const_levels(EmuCtx *c, int n, const uint64_t *elts, const uint64_t *keys, uint64_t *out, uint64_t *tmp) {
  std::vector<const u32 *> ctabs;
  for (int g = 0; g < n; g++) {
    if (!c->cperms.count(elts[g])) evab_host::galois_coeff_table(c->v.N, elts[g], c->cperms[elts[g]]);
    ctabs.push_back(c->cperms[elts[g]].data());
  }
  LevelsBE be{{c}};
  return hoist_const_levels_impl(be, c->v, n, ctabs.data(), keys, out, tmp);
}
}
