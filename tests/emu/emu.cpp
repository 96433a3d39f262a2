// emu.cpp -- CPU replay of the CUDA kernel bodies (TEST INFRASTRUCTURE).
// Compiles eva_b200/csrc/{ntt_kernels,ops_kernels}.cuh + ops_impl.hpp with g++
// and executes every CTA / thread / phase serially on host memory, so indexing,
// swizzles, strides and lazy-reduction bounds are validated against the oracle
// in a container without a GPU.  Not product code; the product path is CUDA only.
#include "../../eva_b200/csrc/host_tables.hpp"
#include "../../eva_b200/csrc/ops_impl.hpp"
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

static std::string g_err;

struct EmuCtx {
  CtxView v;
  evab_host::Tables T;
  std::vector<u64> zeros;
  std::map<u64, std::vector<u32>> perms, cperms;
};

// run phase PH of body B for every thread of every CTA of one job (the CTAs of a cluster advance in
// lockstep, phase by phase -- what the block / cluster barriers guarantee on the device), then PH+1
template <class B, int CL, int PH, int NPH> struct EmuPhases {
  static void run(NttState *st, int Tc, int nctas, const NttLaunch &L, const NttJob *J, const SmemView<CL> *sm) {
    for (int h = 0; h < nctas; h++)
      for (u32 t = 0; t < (u32)Tc; t++) B::template phase<PH>(st[(size_t)h * Tc + t], L, J[h], t, sm[h], NoHooks());
    EmuPhases<B, CL, PH + 1, NPH>::run(st, Tc, nctas, L, J, sm);
  }
};
template <class B, int CL, int NPH> struct EmuPhases<B, CL, NPH, NPH> {
  static void run(NttState *, int, int, const NttLaunch &, const NttJob *, const SmemView<CL> *) {}
};

// one residue over a cluster of CL CTAs (CL = 1: a single CTA); distributed shared memory = the
// SmemView's peer pointers
template <int LOGN, bool INV, int PRO, int EPI, int CL, int AR> static void run_ntt_m(const NttLaunch &L, size_t jobs) {
  typedef NttGeom<LOGN> G;
  constexpr int Tc = G::T / CL;                // threads per CTA
  constexpr size_t SMC = (size_t)G::N / CL;    // shared-memory words per CTA
  std::vector<u64> smc((size_t)CL * SMC);
  std::vector<NttState> stc((size_t)CL * Tc);
  for (size_t job = 0; job < jobs; job++) {
    NttJob J[CL];
    SmemView<CL> sm[CL];
    for (int h = 0; h < CL; h++) {
      J[h] = ntt_job(L, (u32)(job * CL + h), CL);
      sm[h].local = smc.data() + (size_t)h * SMC;
      for (int r = 0; r < CL; r++) sm[h].peer[r] = smc.data() + (size_t)r * SMC;
    }
    if (J[0].skip) continue;
    if (!INV && PRO == PRO_PLAIN && EPI == EPI_STORE && J[0].bcast) {
      for (int h = 0; h < CL; h++)
        for (u32 t = 0; t < (u32)Tc; t++) fwd_const_poly<LOGN>(J[h], (u32)h * Tc + t);
      continue;
    }
    if (!INV) {
      typedef FwdBody<LOGN, PRO, EPI, CL, AR> B;
      EmuPhases<B, CL, 0, B::NPH>::run(stc.data(), Tc, CL, L, J, sm);
      for (int h = 0; h < CL; h++)
        for (u32 t = 0; t < (u32)Tc; t++) B::phE(stc[(size_t)h * Tc + t], L, J[h], t);
    } else {
      typedef InvBody<LOGN, PRO, EPI, CL, AR> B;
      EmuPhases<B, CL, 0, B::NPH>::run(stc.data(), Tc, CL, L, J, sm);
    }
  }
}

static int g_cl = 1;   // emu_set_cluster: CTAs per residue for N >= 4096 (1, 2, 4)

template <int LOGN, bool INV, int CL, int AR> static void run_ntt_c(const NttLaunch &L, size_t jobs) {
  if (!INV) {
    if (L.pro == PRO_PLAIN && L.epi == EPI_STORE) return run_ntt_m<LOGN, false, PRO_PLAIN, EPI_STORE, CL, AR>(L, jobs);
    if (L.pro == PRO_MODRED && L.epi == EPI_STORE) return run_ntt_m<LOGN, false, PRO_MODRED, EPI_STORE, CL, AR>(L, jobs);
    if (L.pro == PRO_MODRED && L.epi == EPI_STORE_LAZY) return run_ntt_m<LOGN, false, PRO_MODRED, EPI_STORE_LAZY, CL, AR>(L, jobs);
    if (L.pro == PRO_MODRED && L.epi == EPI_DIVROUND) return run_ntt_m<LOGN, false, PRO_MODRED, EPI_DIVROUND, CL, AR>(L, jobs);
    if (L.pro == PRO_MODRED_SG && L.epi == EPI_STORE_LAZY) return run_ntt_m<LOGN, false, PRO_MODRED_SG, EPI_STORE_LAZY, CL, AR>(L, jobs);
  } else {
    if (L.pro == PRO_PLAIN && L.epi == EPI_STORE) return run_ntt_m<LOGN, true, PRO_PLAIN, EPI_STORE, CL, AR>(L, jobs);
    if (L.pro == PRO_PLAIN && L.epi == EPI_ADDHALF) return run_ntt_m<LOGN, true, PRO_PLAIN, EPI_ADDHALF, CL, AR>(L, jobs);
    if (L.pro == PRO_GATHER && L.epi == EPI_STORE) return run_ntt_m<LOGN, true, PRO_GATHER, EPI_STORE, CL, AR>(L, jobs);
    if (L.pro == PRO_PLAIN && L.epi == EPI_STORE_ZFLAG) return run_ntt_m<LOGN, true, PRO_PLAIN, EPI_STORE_ZFLAG, CL, AR>(L, jobs);
  }
  abort();
}
template <int LOGN, bool INV, int AR> static void run_ntt_a(const NttLaunch &L, size_t jobs) {
  if constexpr (LOGN >= 12) {
    if (g_cl == 4) return run_ntt_c<LOGN, INV, 4, AR>(L, jobs);
    if (g_cl == 8) return run_ntt_c<LOGN, INV, 8, AR>(L, jobs);
    if (g_cl == 2 || LOGN == 15) return run_ntt_c<LOGN, INV, 2, AR>(L, jobs);   // 2^15: at least 2 CTAs
  }
  if constexpr (LOGN <= 14) return run_ntt_c<LOGN, INV, 1, AR>(L, jobs);
}
static int g_folded = 0;   // launches that took the fold path (emu_fold_launches)
template <int LOGN, bool INV> static void run_ntt(const NttLaunch &L, size_t jobs, bool fold) {
  if (fold) { g_folded++; run_ntt_a<LOGN, INV, 1>(L, jobs); } else run_ntt_a<LOGN, INV, 0>(L, jobs);
}

struct EmuBE {
  const EmuCtx *c;
  int error(const char *m) { g_err = m; return 1; }
  int fwd(const NttLaunch &L, size_t jobs) {
    const bool fold = c->v.arith == 0 && ntt_launch_folds(L, jobs, c->v.foldmask);
    switch (c->v.logN) {
      case 10: run_ntt<10, false>(L, jobs, fold); break;
      case 11: run_ntt<11, false>(L, jobs, fold); break;
      case 12: run_ntt<12, false>(L, jobs, fold); break;
      case 13: run_ntt<13, false>(L, jobs, fold); break;
      case 14: run_ntt<14, false>(L, jobs, fold); break;
      case 15: run_ntt<15, false>(L, jobs, fold); break;
      default: return error("unsupported N");
    }
    return 0;
  }
  int inv(const NttLaunch &L, size_t jobs) {
    const bool fold = c->v.arith == 0 && ntt_launch_folds(L, jobs, c->v.foldmask);
    switch (c->v.logN) {
      case 10: run_ntt<10, true>(L, jobs, fold); break;
      case 11: run_ntt<11, true>(L, jobs, fold); break;
      case 12: run_ntt<12, true>(L, jobs, fold); break;
      case 13: run_ntt<13, true>(L, jobs, fold); break;
      case 14: run_ntt<14, true>(L, jobs, fold); break;
      case 15: run_ntt<15, true>(L, jobs, fold); break;
      default: return error("unsupported N");
    }
    return 0;
  }
  int dyadic(int op, const DyArgs &A) {
    if (op == DY_MULPT) {
      for (int i = 0; i < A.ell; i++)
        for (int j = 0; j < A.N; j += 4) mulpt_elem(A, i, j);
      return 0;
    }
    for (int res = 0; res < A.sout * A.ell; res++)
      for (int j = 0; j < A.N; j += 4) switch (op) {
          case DY_ADD: dyadic_elem<DY_ADD>(A, res, j); break;
          case DY_SUB: dyadic_elem<DY_SUB>(A, res, j); break;
          case DY_NEG: dyadic_elem<DY_NEG>(A, res, j); break;
          case DY_COPY: dyadic_elem<DY_COPY>(A, res, j); break;
          default: dyadic_elem<DY_MULPT>(A, res, j); break;
        }
    return 0;
  }
  int sum(const SumArgs &A) {
    for (int res = 0; res < A.sout * A.ell; res++)
      for (int j = 0; j < A.N; j += 2) sum_terms_elem(A, res, j, 0);
    return 0;
  }
  int mulct(bool sq, const MulArgs &A) {
    for (int i = 0; i < A.ell; i++)
      for (int j = 0; j < A.N; j += 2) { if (sq) mulct_elem<true>(A, i, j); else mulct_elem<false>(A, i, j); }
    return 0;
  }
  int inner(const IpArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++)
      for (int j = 0; j < A.N; j += 2) ks_inner_elem(A, mi, j);
    return 0;
  }
  int scale_c0(const u64 *c0, u64 *ext, int ell) {
    for (int mi = 0; mi < ell; mi++) for (int j = 0; j < (int)c->v.N; j++) scale_c0_elem(c0, ext, c->v.primes, ell, c->v.k, (int)c->v.N, mi, j);
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    for (int i = 0; i < A.n; i++) for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) rot_many_elem(A, i, mi, j);
    return 0;
  }
  int lazy_rotsum(const LazyRotSumArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) {
      u64 sum[LRS_OUT][4] = {}, part[LRS_OUT][4];
      for (int i = 0; i < A.n; i++) { lazy_rotsum_part(A, mi, j, i, 0, part); for (int o = 0; o < A.nout; o++) for (int c = 0; c < 4; c++) sum[o][c] += part[o][c]; }
      for (int o = 0; o < A.nout; o++) lazy_rotsum_store(A, mi, j, o, 0, sum[o]);
    }
    return 0;
  }
  int hoist_indicator(u64 *out, const u32 *ctab, int N, int rows) {
    for (int mi = 0; mi < rows; mi++) for (int j = 0; j < N; j++) hoist_indicator_elem(out, ctab, N, mi, j);
    return 0;
  }
  int hoist_const(const HoistConstArgs &A) {
    for (int mi = 0; mi <= A.ell; mi++) for (int j = 0; j < A.N; j += 2) hoist_const_elem(A, mi, j);
    return 0;
  }
  int dec_compose(const DecArgs &A) { for (u32 j = 0; j < A.N; j++) ::dec_compose(A, j); return 0; }
  int dec_fft(const DecArgs &A, u32 m) { for (u32 b = 0; b < A.N / 2; b++) dec_fft_bfly(A, m, b); return 0; }
  int dec_gather(const DecArgs &A) { for (u32 i = 0; i < A.N / 2; i++) ::dec_gather(A, i); return 0; }
  int enc_scatter(const EncBatch &B) {
    for (u32 e = 0; e < B.count; e++) for (u32 i = 0; i < B.N / 2; i++) ::enc_scatter(B, e, i);
    return 0;
  }
  int enc_fft(const EncBatch &B, u32 g, int ns) {
    for (u32 e = 0; e < B.count; e++) for (u32 t = 0; t < B.N / 8; t++) enc_fft8(B, e, t, g, ns);
    return 0;
  }
  int enc_uniform(const EncUniform &B) {
    for (u32 e = 0; e < B.count; e++)
      for (u32 i = 0; i < B.ell; i++)
        for (u32 j = 0; j < B.N; j += 2) enc_uniform_elem(B, e, i, j);
    return 0;
  }
  int enc_round(const EncBatch &B) {
    for (u32 e = 0; e < B.count; e++) for (u32 j = 0; j < B.N; j++) ::enc_round(B, e, j);
    return 0;
  }
};

extern "C" {
const char *emu_last_error() { return g_err.c_str(); }
EmuCtx *emu_ctx_create(uint64_t N, const uint64_t *primes, int k) {
  int logN = 0;
  while ((1ull << logN) < N) logN++;
  EmuCtx *c = new EmuCtx();
  const char *err = evab_host::build_tables(N, logN, primes, k, nullptr, c->T);
  if (err[0]) { g_err = err; delete c; return nullptr; }
  for (int i = 0; i < k; i++) {  // re-point the tables at the final host storage
    c->T.pd[i].tw = c->T.tw.data() + ((size_t)i * 2 + 0) * N;
    c->T.pd[i].itw = c->T.tw.data() + ((size_t)i * 2 + 1) * N;
    c->T.pd[i].ftw = c->T.tw.data() + ((size_t)(k + i) * 2 + 0) * N;
    c->T.pd[i].fitw = c->T.tw.data() + ((size_t)(k + i) * 2 + 1) * N;
  }
  c->zeros.assign(32, 0);
  c->v.N = N; c->v.logN = logN; c->v.k = k;
  c->v.primes = c->T.pd.data(); c->v.qinv = c->T.qinv.data(); c->v.halfmod = c->T.halfmod.data(); c->v.zeros = c->zeros.data();
  c->v.qinv_f = c->T.qinv_f.data(); c->v.foldmask = c->T.foldmask; c->v.arith = 0;
  for (int i = 0; i < k; i++) { c->T.fp[i].ftw = c->T.pd[i].ftw; c->T.fp[i].fitw = c->T.pd[i].fitw; }
  c->v.fold_host = c->T.fp.data();
  c->v.roots = reinterpret_cast<const cplx *>(c->T.roots.data()); c->v.slot_index = c->T.slot_index.data(); c->v.pow2 = c->T.pow2.data();
  return c;
}
void emu_ctx_destroy(EmuCtx *c) { delete c; }
int emu_ctx_set_ntt_arith(EmuCtx *c, int mode) { c->v.arith = mode; return 0; }
unsigned emu_ctx_foldmask(EmuCtx *c) { return c->v.foldmask; }
int emu_fold_launches() { return g_folded; }
#if defined(EVAB_BOUND_CHECK)
int emu_bound_checked() { return 1; }   // this library verifies every tracked bound of the fold arithmetic (ntt_core.cuh)
#else
int emu_bound_checked() { return 0; }
#endif
int emu_ntt_fwd(EmuCtx *c, uint64_t *d, size_t count, const int *pidx, int np) { EmuBE be{c}; return ntt_batch_impl(be, c->v, false, d, count, pidx, np); }
int emu_ntt_inv(EmuCtx *c, uint64_t *d, size_t count, const int *pidx, int np) { EmuBE be{c}; return ntt_batch_impl(be, c->v, true, d, count, pidx, np); }
int emu_add(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *b, int sb) { EmuBE be{c}; return dyadic_impl<DY_ADD>(be, c->v, ell, o, a, sa, b, sb, 0); }
int emu_sub(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *b, int sb) { EmuBE be{c}; return dyadic_impl<DY_SUB>(be, c->v, ell, o, a, sa, b, sb, 0); }
int emu_add_plain(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt) { EmuBE be{c}; return dyadic_impl<DY_ADD>(be, c->v, ell, o, a, sa, pt, 1, 1); }
int emu_sub_plain(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt) { EmuBE be{c}; return dyadic_impl<DY_SUB>(be, c->v, ell, o, a, sa, pt, 1, 1); }
int emu_negate(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa) { EmuBE be{c}; return dyadic_impl<DY_NEG>(be, c->v, ell, o, a, sa, (const u64 *)nullptr, 0, 0); }
int emu_mul_plain(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt) { EmuBE be{c}; return dyadic_impl<DY_MULPT>(be, c->v, ell, o, a, sa, pt, 1, 1); }
int emu_mul(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *b) { EmuBE be{c}; return mulct_impl(be, c->v, false, ell, o, a, b); }
int emu_square(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a) { EmuBE be{c}; return mulct_impl(be, c->v, true, ell, o, a, (const u64 *)nullptr); }
int emu_set_cluster(int cl) { if (cl != 1 && cl != 2 && cl != 4 && cl != 8) return 1; g_cl = cl; return 0; }
int emu_sum_terms(EmuCtx *c, int ell, uint64_t *o, int n, const uint64_t *const *cts, const int *sizes, const uint64_t *const *pts) {
  EmuBE be{c};
  return sum_terms_impl(be, c->v, ell, o, n, cts, sizes, pts);
}
int emu_sum_products(EmuCtx *c, int ell, uint64_t *o, int n, const uint64_t *const *cts, const int *sizes, const uint64_t *const *seconds, const int *kinds) {
  EmuBE be{c};
  return sum_terms_impl(be, c->v, ell, o, n, cts, sizes, seconds, kinds);
}
int emu_encode_uniform(EmuCtx *c, int count, const double *values, const double *scales, int ell, uint64_t *out) {
  EmuBE be{c};
  return encode_uniform_impl(be, c->v, count, values, scales, ell, out);
}
size_t emu_encode_work_bytes(EmuCtx *c, int count) { return encode_work_bytes(c->v, count); }
int emu_encode(EmuCtx *c, int count, const double *const *vals, const uint32_t *vec, const double *scales, int ell, uint64_t *out, void *work) {
  EmuBE be{c};
  return encode_impl(be, c->v, count, vals, vec, scales, ell, out, (cplx *)work);
}
int emu_encode_ext(EmuCtx *c, int count, const double *const *vals, const uint32_t *vec, const double *scales, int ell, int with_p, uint64_t *out, void *work) {
  EmuBE be{c};
  return encode_impl(be, c->v, count, vals, vec, scales, ell, out, (cplx *)work, with_p);
}
int emu_encode_uniform_ext(EmuCtx *c, int count, const double *values, const double *scales, int ell, int with_p, uint64_t *out) {
  EmuBE be{c};
  return encode_uniform_impl(be, c->v, count, values, scales, ell, out, with_p);
}
int emu_rotate_modup_scale_c0(EmuCtx *c, int ell, uint64_t *ext, const uint64_t *a) {
  EmuBE be{c};
  return rotate_modup_scale_c0_impl(be, c->v, ell, ext, a);
}
size_t emu_rotate_modup_many_work_bytes(EmuCtx *c, int ell, int n) { return rotate_modup_many_work_elems(c->v, ell, n) * 8; }
int emu_rotate_modup_many(EmuCtx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts, const uint64_t *const *keys,
                          const uint64_t *const *cadds, void *work) {
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n && i < ROTMANY_MAX; i++) {
    if (!c->perms.count(elts[i])) evab_host::galois_table(c->v.N, c->v.logN, elts[i], c->perms[elts[i]]);
    perms[i] = c->perms[elts[i]].data();
  }
  EmuBE be{c};
  return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, cadds, (u64 *)work);
}
size_t emu_lazy_rotsum_work_bytes(EmuCtx *c, int ell, int nout) { return lazy_rotsum_work_elems(c->v, ell, nout) * 8; }
int emu_lazy_rotsum(EmuCtx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts, const uint64_t *const *keys,
                    const uint64_t *const *cadds, const uint64_t *const *wts, void *work) {
  const u32 *perms[LRS_MAX];
  for (int i = 0; i < n && i < LRS_MAX; i++) {
    if (!c->perms.count(elts[i])) evab_host::galois_table(c->v.N, c->v.logN, elts[i], c->perms[elts[i]]);
    perms[i] = c->perms[elts[i]].data();
  }
  EmuBE be{c};
  return lazy_rotsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, (u64 *)work);
}
int emu_decode(EmuCtx *c, int ell, const uint64_t *primes, const uint64_t *pt, double scale, double *out) {
  EmuBE be{c};
  std::vector<u64> tmp(decode_tmp_elems(c->v, ell));
  std::vector<cplx> work(c->v.N);
  return decode_impl(be, c->v, ell, primes, pt, scale, out, tmp.data(), work.data());
}
size_t emu_rescale_work_bytes(EmuCtx *c, int sa) { return rescale_work_elems(c->v, sa) * 8; }
int emu_rescale(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, int sa, void *work) { EmuBE be{c}; return rescale_impl(be, c->v, ell, o, a, sa, (u64 *)work); }
size_t emu_keyswitch_work_bytes(EmuCtx *c, int ell) { return keyswitch_work_elems(c->v, ell) * 8; }
int emu_relinearize(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *key, void *work) { EmuBE be{c}; return relinearize_impl(be, c->v, ell, o, a, key, (u64 *)work); }
int emu_rotate(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, uint64_t elt, const uint64_t *key, void *work) {
  if (!c->perms.count(elt)) evab_host::galois_table(c->v.N, c->v.logN, elt, c->perms[elt]);
  EmuBE be{c};
  return rotate_impl(be, c->v, ell, o, a, c->perms[elt].data(), key, (u64 *)work);
}
// shared mod-up of a rotation group (exact): returns the zero flag through *zflag
int emu_rotate_modup_prepare(EmuCtx *c, int ell, uint64_t *that, uint64_t *ext, const uint64_t *a, uint64_t *zflag) {
  EmuBE be{c};
  return rotate_modup_prepare_impl(be, c->v, ell, that, ext, a, zflag);
}
int emu_rotate_hoist_const(EmuCtx *c, int ell, uint64_t elt, const uint64_t *key, uint64_t *out, uint64_t *tmp) {
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  EmuBE be{c};
  return hoist_const_impl(be, c->v, ell, c->cperms[elt].data(), key, out, tmp);
}
size_t emu_rotate_modup_work_bytes(EmuCtx *c, int ell) { return rotate_modup_work_elems(c->v, ell) * 8; }
int emu_rotate_modup_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key, const uint64_t *cadd, void *work) {
  if (!c->perms.count(elt)) evab_host::galois_table(c->v.N, c->v.logN, elt, c->perms[elt]);
  EmuBE be{c};
  return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, c->perms[elt].data(), key, cadd, (u64 *)work);
}
int emu_rotate_prepare(EmuCtx *c, int ell, uint64_t *hoist, const uint64_t *a) {
  EmuBE be{c};
  return rotate_prepare_impl(be, c->v, ell, hoist, a);
}
int emu_rotate_prepared(EmuCtx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *hoist, uint64_t elt, const uint64_t *key, void *work) {
  if (!c->perms.count(elt)) evab_host::galois_table(c->v.N, c->v.logN, elt, c->perms[elt]);
  if (!c->cperms.count(elt)) evab_host::galois_coeff_table(c->v.N, elt, c->cperms[elt]);
  EmuBE be{c};
  return rotate_prepared_impl(be, c->v, ell, o, a, hoist, c->perms[elt].data(), c->cperms[elt].data(), key, (u64 *)work);
}
}
