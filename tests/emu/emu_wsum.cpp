// emu_wsum.cpp -- CPU replay of evab_rotate_wsum (TEST INFRASTRUCTURE): the emulator of emu.cpp plus the two pieces the
// weighted rotation sums add, the k_rot_wsum body and the forward NTT with PRO_PLAIN + EPI_DIVROUND.  Built as its own library
// (tests/test_rotation_wsum.py); every other op is emu.cpp's.
#include "emu.cpp"

template <int LOGN, int AR> static void run_plain_divround(const NttLaunch &L, size_t jobs) {
  if constexpr (LOGN >= 12) {
    if (g_cl == 4) return run_ntt_m<LOGN, false, PRO_PLAIN, EPI_DIVROUND, 4, AR>(L, jobs);
    if (g_cl == 8) return run_ntt_m<LOGN, false, PRO_PLAIN, EPI_DIVROUND, 8, AR>(L, jobs);
    if (g_cl == 2 || LOGN == 15) return run_ntt_m<LOGN, false, PRO_PLAIN, EPI_DIVROUND, 2, AR>(L, jobs);
  }
  if constexpr (LOGN <= 14) return run_ntt_m<LOGN, false, PRO_PLAIN, EPI_DIVROUND, 1, AR>(L, jobs);
}
template <int LOGN> static void run_plain_divround(const NttLaunch &L, size_t jobs, bool fold) {
  if (fold) { g_folded++; run_plain_divround<LOGN, 1>(L, jobs); } else run_plain_divround<LOGN, 0>(L, jobs);
}

struct WsumBE : EmuBE {
  int fwd(const NttLaunch &L, size_t jobs) {
    if (L.pro != PRO_PLAIN || L.epi != EPI_DIVROUND) return EmuBE::fwd(L, jobs);
    const bool fold = c->v.arith == 0 && ntt_launch_folds(L, jobs, c->v.foldmask);
    switch (c->v.logN) {
      case 10: run_plain_divround<10>(L, jobs, fold); break;
      case 11: run_plain_divround<11>(L, jobs, fold); break;
      case 12: run_plain_divround<12>(L, jobs, fold); break;
      case 13: run_plain_divround<13>(L, jobs, fold); break;
      case 14: run_plain_divround<14>(L, jobs, fold); break;
      case 15: run_plain_divround<15>(L, jobs, fold); break;
      default: return error("unsupported N");
    }
    return 0;
  }
  int rot_wsum(const WsumArgs &A) {
    for (int c = 0; c < 2; c++) for (int r = 0; r < A.ell; r++) for (int j = 0; j < A.N; j += 2) rot_wsum_elem(A, c, r, j);
    return 0;
  }
};

extern "C" {
size_t emu_rotate_wsum_work_bytes(EmuCtx *c, int ell, int n, int nout) { return rotate_wsum_work_elems(c->v, ell, n, nout) * 8; }
int emu_rotate_wsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                    const uint64_t *const *cadds, const uint64_t *const *wts, int ntap, const uint64_t *const *taps, const uint64_t *const *twts, void *work) {
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n && i < WS_MAX; i++) {
    if (!c->perms.count(elts[i])) evab_host::galois_table(c->v.N, c->v.logN, elts[i], c->perms[elts[i]]);
    perms[i] = c->perms[elts[i]].data();
  }
  WsumBE be{{c}};
  return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, ntap, taps, twts, (u64 *)work);
}
}
