// ops_impl.hpp -- composition of the evaluator ops out of kernel launches,
// templated on a backend (CUDA launches in evab200.cu; serial replay in the
// CPU emulator used by the tests).  Each function names the SEAL call it
// replaces at the reference call site in eva/seal/seal_executor.h.
#pragma once
#include "ntt_kernels.cuh"
#include "ops_kernels.cuh"
#include "encode_kernels.cuh"
#include <cstring>

struct CtxView {
  u64 N; int logN, k;
  const PrimeDev *primes;   // [k]
  const u64x2 *qinv;        // [k][k]
  const u64 *halfmod;       // [k][k]
  const u64 *zeros;         // [k]
  const cplx *roots;        // [N]   CKKS encoder tables
  const u32 *slot_index;    // [N]
  const u64 *pow2;          // [k][ENC_POW2_ROW]
  const u64x2 *qinv_f;      // [k][k]   fold rows of qinv
  unsigned foldmask;        // bit i: prime i is fold-friendly (modarith.cuh prime_foldable)
  const FoldPrime *fold_host;   // [k] HOST array: per-prime fold constants, copied into every NttLaunch
  int arith;                // 0: fold arithmetic where every prime of a launch allows it; 1: lazy Shoup everywhere
};

// Backend concept:
//   int fwd(const NttLaunch&, size_t jobs);  int inv(const NttLaunch&, size_t jobs);
//   int dyadic(int op, const DyArgs&);       int mulct(bool square, const MulArgs&);
//   int inner(const IpArgs&);                int perm(u64*, const u64*, const u32*, int N, int rows);
//   int drop_last(u64* out, const u64* in, int ell, int polys, u64 N);
//   int enc_scatter(const EncBatch&);  int enc_fft(const EncBatch&, u32 gap, int nstages);  int enc_round(const EncBatch&);
//   int error(const char*);

inline NttLaunch base_launch(const CtxView &c) {
  NttLaunch L;
  memset(&L, 0, sizeof(L));
  L.primes = c.primes;
  for (int i = 0; i < c.k && i < NTT_MAX_PRIMES; i++) L.fp[i] = c.fold_host[i];
  L.inner = 1;
  L.aux1_polys = 1 << 30;
  return L;
}

template <class BE>
int ntt_batch_impl(BE &be, const CtxView &c, bool inverse, u64 *d, size_t count, const int *pidx, int np) {
  if (np < 1 || np > 32) return be.error("evab_ntt: nprimes must be in [1,32]");
  if (count % np) return be.error("evab_ntt: count must be a multiple of nprimes");
  NttLaunch L = base_launch(c);
  L.src = d; L.dst = d;
  L.inner = np;
  L.src_sq = L.dst_sq = (long long)np * c.N;
  L.src_sr = L.dst_sr = (long long)c.N;
  for (int i = 0; i < np; i++) {
    if (pidx[i] < 0 || pidx[i] >= c.k) return be.error("evab_ntt: prime index out of range");
    L.pmap[i] = (unsigned char)pidx[i];
  }
  return inverse ? be.inv(L, count) : be.fwd(L, count);
}

template <int OP, class BE>
int dyadic_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, int sa, const u64 *b, int sb, int plain) {
  if (ell < 1 || ell > c.k) return be.error("ell out of range");
  if (sa < 1 || sa > 3 || (b && !plain && (sb < 1 || sb > 3))) return be.error("ciphertext size must be 1..3");
  DyArgs A;
  A.out = out; A.a = a; A.b = b; A.primes = c.primes; A.ell = ell; A.N = (int)c.N;
  A.sa = sa; A.sb = sb; A.b_is_plain = plain; A.a_ell = ell;
  A.sout = (plain || !b) ? sa : (sa > sb ? sa : sb);
  return be.dyadic(OP, A);
}
// copy the first `ell_out` residues of every polynomial: ell_out == ell_in is a plain
// ciphertext copy (rotate_vector by 0), ell_out == ell_in - 1 is
// Evaluator::mod_switch_to_next (reference eva/seal/seal_executor.h:206; Appendix A.7)
template <class BE> int copy_impl(BE &be, const CtxView &c, int ell_in, int ell_out, u64 *out, const u64 *a, int sa) {
  if (ell_out < 1 || ell_out > ell_in || ell_in > c.k) return be.error("copy: bad residue counts");
  if (sa < 1 || sa > 3) return be.error("ciphertext size must be 1..3");
  DyArgs A;
  A.out = out; A.a = a; A.b = nullptr; A.primes = c.primes; A.ell = ell_out; A.N = (int)c.N;
  A.sa = sa; A.sb = 0; A.b_is_plain = 0; A.a_ell = ell_in; A.sout = sa;
  return be.dyadic(DY_COPY, A);
}

// out = sum of terms; kinds[t] (null = derive from pts: 1 when pts[t], else 0): 0 cts[t], 1 cts[t] * pts[t]
// (plaintext), 2 cts[t] (x) pts[t] (both size-2 ciphertexts, value of size 3).  sizes[t] = polynomials of
// cts[t].  Up to 64 products of < 2^120 fit the 128-bit accumulators (32 terms, two products for the
// middle component of a tensor product).
template <class BE>
int sum_terms_impl(BE &be, const CtxView &c, int ell, u64 *out, int nterms, const u64 *const *cts, const int *sizes, const u64 *const *pts,
                   const int *kinds = nullptr) {
  if (ell < 1 || ell > c.k) return be.error("ell out of range");
  if (nterms < 1 || nterms > SUM_MAX_TERMS) return be.error("evab_sum_terms: 1..32 terms");
  SumArgs A;
  memset(&A, 0, sizeof(A));
  A.out = out; A.primes = c.primes; A.n = nterms; A.ell = ell; A.N = (int)c.N; A.sout = 0;
  for (int t = 0; t < nterms; t++) {
    if (sizes[t] < 1 || sizes[t] > 3) return be.error("ciphertext size must be 1..3");
    const int kind = kinds ? kinds[t] : ((pts && pts[t]) ? 1 : 0);
    if (kind < 0 || kind > 2 || (kind && !(pts && pts[t]))) return be.error("evab_sum_terms: bad term kind");
    if (kind == 2 && sizes[t] != 2) return be.error("evab_sum_terms: ciphertext products need size-2 operands");
    A.ct[t] = cts[t]; A.pt[t] = pts ? pts[t] : nullptr; A.kind[t] = (unsigned char)kind;
    A.size[t] = (unsigned char)(kind == 2 ? 3 : sizes[t]);
    if ((int)A.size[t] > A.sout) A.sout = A.size[t];
  }
  return be.sum(A);
}

template <class BE> int mulct_impl(BE &be, const CtxView &c, bool square, int ell, u64 *out, const u64 *a, const u64 *b) {
  if (ell < 1 || ell > c.k) return be.error("ell out of range");
  MulArgs A;
  A.out = out; A.a = a; A.b = b; A.primes = c.primes; A.ell = ell; A.N = (int)c.N;
  return be.mulct(square, A);
}

// RNS divide-and-round by the last residue's prime (SEAL
// RNSTool::divide_and_round_q_last_ntt_inplace; Appendix A.6), shared by
// rescale and the key-switch mod-down.  Poly q (< npoly) of `in` has `nres`
// residues: prime indices pm[0..nres-2] followed by the divisor `last`.
//   out[q][r] = (in[q][r] - NTT((iNTT(in[q][last]) + h) mod q_last mod q_r - h mod q_r)) * q_last^-1  (+ add[q][r])
// first half: tmp[q] = iNTT(in[q][last]) + h, canonical mod q_last
template <class BE>
int divround_inv_impl(BE &be, const CtxView &c, const u64 *in, long long in_poly_stride, int npoly, int nres, int last, u64 *tmp) {
  const long long N = (long long)c.N;
  NttLaunch A = base_launch(c);
  A.src = in + (long long)(nres - 1) * N; A.dst = tmp;
  A.src_sq = in_poly_stride; A.dst_sq = N; A.inner = 1; A.prime_on_q = 1;
  for (int q = 0; q < npoly; q++) A.pmap[q] = (unsigned char)last;
  A.epi = EPI_ADDHALF;
  return be.inv(A, npoly);
}
template <class BE>
int divround_impl(BE &be, const CtxView &c, const u64 *in, long long in_poly_stride, int npoly, int nres, const unsigned char *pm,
                  int last, u64 *out, long long out_poly_stride, const u64 *add, long long add_poly_stride, u64 *tmp,
                  int add_polys = 1 << 30, const u32 *add_perm = nullptr) {
  const long long N = (long long)c.N;
  if (int rc = divround_inv_impl(be, c, in, in_poly_stride, npoly, nres, last, tmp)) return rc;
  NttLaunch B = base_launch(c);
  B.src = tmp; B.src_sq = N; B.src_sr = 0;
  B.aux0 = in; B.aux0_sq = in_poly_stride; B.aux0_sr = N;
  B.aux1 = add; B.aux1_sq = add_poly_stride; B.aux1_sr = N; B.aux1_polys = add_polys; B.aux1_perm = add_perm;
  B.dst = out; B.dst_sq = out_poly_stride; B.dst_sr = N;
  B.inner = nres - 1; B.prime_on_q = 0;
  for (int r = 0; r < nres - 1; r++) { B.pmap[r] = pm[r]; B.pmap2[r] = (unsigned char)last; }   // src holds residues mod q_last
  B.pro = PRO_MODRED; B.epi = EPI_DIVROUND;
  B.subtab = c.halfmod + (size_t)last * c.k;
  B.consts = c.qinv + (size_t)last * c.k;
  B.consts_f = c.qinv_f + (size_t)last * c.k;
  return be.fwd(B, (size_t)npoly * (nres - 1));
}

inline size_t rescale_work_elems(const CtxView &c, int sa) { return (size_t)sa * c.N; }

// Evaluator::rescale_to_next -- reference eva/seal/seal_executor.h:213
template <class BE> int rescale_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, int sa, u64 *work) {
  if (ell < 2 || ell > c.k) return be.error("rescale needs 2 <= ell <= k");
  if (sa < 1 || sa > 3) return be.error("ciphertext size must be 1..3");
  unsigned char pm[32];
  for (int i = 0; i < ell; i++) pm[i] = (unsigned char)i;
  const long long N = (long long)c.N;
  return divround_impl(be, c, a, ell * N, sa, ell, pm, ell - 1, out, (ell - 1) * N, (const u64 *)nullptr, 0, work);
}

// workspace (in u64): that[ell] + ext[ell+1][ell] + acc[2][ell+1] + tmp[2]
inline size_t ks_off_ext(const CtxView &c, int ell) { return (size_t)ell * c.N; }
inline size_t ks_off_acc(const CtxView &c, int ell) { return ks_off_ext(c, ell) + (size_t)(ell + 1) * ell * c.N; }
inline size_t ks_off_tmp(const CtxView &c, int ell) { return ks_off_acc(c, ell) + (size_t)2 * (ell + 1) * c.N; }
inline size_t keyswitch_work_elems(const CtxView &c, int ell) { return ks_off_tmp(c, ell) + (size_t)2 * c.N; }

// Evaluator::switch_key_inplace (Appendix A.5): out[c][J] = base[c][J] + ks_c[J];
// base holds `base_polys` (1 or 2) polynomials.
// Rotations: t and base are the UNrotated c1 / c0 and `nperm` is the NTT-domain permutation of the
// automorphism, through which they are read (digit iNTT, inner product, mod-down epilogue).
// Hoisted form (rotations sharing the inverse NTT of their input, exact): `that_in` = iNTT of the
// unrotated digits, read by the mod-up through `ctab`, the coefficient-domain signed gather.
// step 2 of A.5: ext[m][J] = NTT_m(that[J] mod m) for every output modulus m != q_J; `ctab` != null reads the digits through
// the signed coefficient-domain gather of an automorphism
template <class BE> int ks_modup(BE &be, const CtxView &c, int ell, const u64 *that, u64 *ext, const u32 *ctab) {
  const long long N = (long long)c.N;
  const int sp = c.k - 1;
  NttLaunch B = base_launch(c);
  B.src = that; B.src_sq = 0; B.src_sr = N;
  B.dst = ext; B.dst_sq = (long long)ell * N; B.dst_sr = N;
  B.inner = ell; B.prime_on_q = 1; B.skip_diag = 1; B.pro = ctab ? PRO_MODRED_SG : PRO_MODRED;
  B.perm = ctab;
  // the extended digits only feed the 128-bit inner product, which reduces lazily:
  // skip their canonicalisation while the accumulated sum stays below 2^128
  B.epi = (ell <= 15) ? EPI_STORE_LAZY : EPI_STORE;
  B.subtab = c.zeros;
  for (int mi = 0; mi <= ell; mi++) B.pmap[mi] = (unsigned char)(mi == ell ? sp : mi);
  for (int J = 0; J < ell; J++) B.pmap2[J] = (unsigned char)J;
  return be.fwd(B, (size_t)(ell + 1) * ell);
}
// steps 3 and 4: inner product with the key rows of the live primes and P, then the mod-down by P with rounding fused with
// the accumulation into base (c0 and c1 for relinearize, c0 only for a rotation: the switched c1 has no base)
template <class BE>
int ks_finish(BE &be, const CtxView &c, int ell, u64 *out, const u64 *t, const u64 *ext, const u64 *key, const u64 *base, int base_polys, u64 *acc, u64 *tmp,
              const u32 *nperm, const u32 *eperm, const u64 *cadd) {
  const long long N = (long long)c.N;
  const int k = c.k, sp = k - 1;
  IpArgs I;
  I.t = t; I.ext = ext; I.key = key; I.acc = acc; I.primes = c.primes; I.ell = ell; I.k = k; I.N = (int)N;
  I.tperm = nperm; I.eperm = eperm; I.cadd = cadd;
  if (int rc = be.inner(I)) return rc;
  unsigned char pm[32];
  for (int i = 0; i < ell; i++) pm[i] = (unsigned char)i;
  return divround_impl(be, c, acc, (long long)(ell + 1) * N, 2, ell + 1, pm, sp, out, (long long)ell * N, base, (long long)ell * N, tmp,
                       base_polys, nperm);
}
template <class BE>
int keyswitch_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *t, const u64 *key, const u64 *base, int base_polys, u64 *work,
                   const u64 *that_in = nullptr, const u32 *ctab = nullptr, const u32 *nperm = nullptr) {
  const long long N = (long long)c.N;
  const int k = c.k;
  if (ell < 1 || ell > k - 1) return be.error("key switching needs 1 <= ell <= k-1");
  u64 *that = work;
  u64 *ext = work + ks_off_ext(c, ell);
  u64 *acc = work + ks_off_acc(c, ell);
  u64 *tmp = work + ks_off_tmp(c, ell);
  // 1. digits to coefficient form: that[J] = iNTT_{q_J}(t[J])
  if (!that_in) {
    NttLaunch A = base_launch(c);
    A.src = t; A.dst = that; A.inner = ell; A.src_sr = A.dst_sr = N;
    if (nperm) { A.pro = PRO_GATHER; A.perm = nperm; }   // single rotation: the automorphism is the load pattern
    for (int J = 0; J < ell; J++) A.pmap[J] = (unsigned char)J;
    if (int rc = be.inv(A, ell)) return rc;
  } else if (ell > 15) {
    return be.error("hoisted key switching supports ell <= 15");
  }
  if (int rc = ks_modup(be, c, ell, that_in ? that_in : that, ext, that_in ? ctab : nullptr)) return rc;
  return ks_finish(be, c, ell, out, t, ext, key, base, base_polys, acc, tmp, nperm, nullptr, nullptr);
}

// Evaluator::relinearize (3 -> 2) -- reference eva/seal/seal_executor.h:200
template <class BE> int relinearize_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, const u64 *key, u64 *work) {
  return keyswitch_impl(be, c, ell, out, a + (size_t)2 * ell * c.N, key, a, 2, work);
}

// Evaluator::rotate_vector -> apply_galois_inplace -- seal_executor.h:181,188
template <class BE>
int rotate_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, const u32 *perm, const u64 *key, u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  // no permuted copy: c1 enters the digit iNTT through the permutation (PRO_GATHER), the inner product
  // and the mod-down epilogue read c1 / c0 through it as well
  return keyswitch_impl(be, c, ell, out, a + (size_t)ell * c.N, key, a, 1, work, nullptr, nullptr, perm);
}


// seal::CKKSEncoder::encode of vectors whose elements are all equal (scalar constants): see enc_uniform_elem
// with_p: the plaintexts get ell + 1 rows, the last one being the residue mod the key-switch prime (lazy_rotsum below)
template <class BE> int encode_uniform_impl(BE &be, const CtxView &c, int count, const double *values, const double *scales, int ell, u64 *out, int with_p = 0) {
  if (ell < 1 || ell + (with_p ? 1 : 0) > c.k) return be.error("encode: ell out of range");
  const int ell_in = ell;
  if (with_p) ell = ell + 1;
  for (int e0 = 0; e0 < count; e0 += ENC_MAX_BATCH) {
    EncUniform B;
    memset(&B, 0, sizeof(B));
    B.count = (u32)((count - e0) < ENC_MAX_BATCH ? (count - e0) : ENC_MAX_BATCH);
    for (u32 e = 0; e < B.count; e++) { B.value[e] = values[e0 + e]; B.scale[e] = scales[e0 + e]; }
    B.out = out + (size_t)e0 * ell * c.N; B.primes = c.primes; B.pow2 = c.pow2; B.N = (u32)c.N; B.ell = (u32)ell;
    B.special_row = with_p ? (u32)(c.k - 1) : 0u;
    if (int rc = be.enc_uniform(B)) return rc;
  }
  (void)ell_in;
  return 0;
}

// encoder workspace: count*N complex values followed by count u64 flags
inline size_t encode_work_bytes(const CtxView &c, int count) { return (size_t)count * c.N * sizeof(cplx) + (size_t)((count + 7) & ~7) * sizeof(u64); }
inline u64 *encode_flags(const CtxView &c, int count, cplx *work) { return reinterpret_cast<u64 *>(work + (size_t)count * c.N); }

// Rotations of one ciphertext share the inverse NTT of its c1 (the automorphism commutes with the
// transform): rotate_prepare_impl computes it once, rotate_prepared_impl is rotate_impl without the
// per-rotation inverse NTTs (the mod-up reads the shared coefficients through the signed
// coefficient-domain gather).  Results are identical to rotate_impl.
template <class BE> int rotate_prepare_impl(BE &be, const CtxView &c, int ell, u64 *hoist, const u64 *a) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  NttLaunch A = base_launch(c);
  A.src = a + (size_t)ell * c.N; A.dst = hoist; A.inner = ell; A.src_sr = A.dst_sr = (long long)c.N;
  for (int J = 0; J < ell; J++) A.pmap[J] = (unsigned char)J;
  return be.inv(A, ell);
}
template <class BE>
int rotate_prepared_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, const u64 *hoist, const u32 *nperm, const u32 *ctab, const u64 *key,
                         u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  return keyswitch_impl(be, c, ell, out, a + (size_t)ell * c.N, key, a, 1, work, hoist, ctab, nperm);
}

// ---- hoisted_modup: rotations of one ciphertext share the inverse NTT AND the mod-up of its c1 -- exactly ---------------
// SEAL rotates first and decomposes afterwards (A.5 step 1 on sigma_g(c1)): the digit of the rotated ciphertext is the signed
// coefficient permutation of the unrotated digit, d'[j] = +-that_J[pi(j)] with the canonical negation q_J - v.  Reduced to an
// output modulus m this is the ring automorphism of w = that_J mod m, EXCEPT that a negated coefficient is (q_J - v) mod m,
// i.e. sigma_g(w)[j] + (q_J mod m):
//     NTT_m(d' mod m) = perm_g( NTT_m(that_J mod m) ) + (q_J mod m) * NTT_m(I_g),      I_g = indicator of the negated positions,
// whenever no negated coefficient of that_J is zero (negate(0) = 0 has no +q_J).  The second term does not depend on the data:
//     acc_c[m] = sum_J perm_g(ext[m][J]) (.) K_g[J][c][m]  +  cadd_g[c][m],   cadd_g[c][m] = NTT_m(I_g) (.) sum_J (q_J mod m) K_g[J][c][m]
// so the ell(ell+1) - ell mod-up transforms are done ONCE per ciphertext (rotate_modup_prepare_impl) and a rotation costs an inner
// product through the permutation + 2 + 2 ell transforms (rotate_modup_prepared_impl): 10 instead of 26 at ell = 4, same bits.
// A zero coefficient in a digit (probability 2^-60 each) raises `zflag`; the caller must then redo the rotations of that
// ciphertext on the ordinary path (the executor does, transparently).
template <class BE> int rotate_modup_prepare_impl(BE &be, const CtxView &c, int ell, u64 *that, u64 *ext, const u64 *a, u64 *zflag) {
  if (ell < 1 || ell > c.k - 1 || ell > 15) return be.error("hoisted rotation needs 1 <= ell <= min(k-1, 15)");
  NttLaunch A = base_launch(c);
  A.src = a + (size_t)ell * c.N; A.dst = that; A.inner = ell; A.src_sr = A.dst_sr = (long long)c.N;
  A.epi = EPI_STORE_ZFLAG; A.zflag = zflag;
  for (int J = 0; J < ell; J++) A.pmap[J] = (unsigned char)J;
  if (int rc = be.inv(A, ell)) return rc;
  return ks_modup(be, c, ell, that, ext, nullptr);
}
// P * c0 on the (otherwise unused) diagonal of ext: required by rotate_modup_many_impl / lazy_rotsum_impl, after the prepare step
template <class BE> int rotate_modup_scale_c0_impl(BE &be, const CtxView &c, int ell, u64 *ext, const u64 *a) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  return be.scale_c0(a, ext, ell);
}
inline size_t hoist_const_elems(const CtxView &c, int ell) { return (size_t)2 * (ell + 1) * c.N; }
// cadd_g for one Galois key at one level; `tmp` holds (ell + 1) * N words
template <class BE> int hoist_const_impl(BE &be, const CtxView &c, int ell, const u32 *ctab, const u64 *key, u64 *out, u64 *tmp) {
  if (ell < 1 || ell > c.k - 1) return be.error("hoisted rotation needs 1 <= ell <= k-1");
  if (int rc = be.hoist_indicator(tmp, ctab, (int)c.N, ell + 1)) return rc;
  int pidx[32];
  for (int mi = 0; mi <= ell; mi++) pidx[mi] = mi == ell ? c.k - 1 : mi;
  if (int rc = ntt_batch_impl(be, c, false, tmp, (size_t)ell + 1, pidx, ell + 1)) return rc;
  HoistConstArgs H;
  H.ind = tmp; H.key = key; H.out = out; H.primes = c.primes; H.ell = ell; H.k = c.k; H.N = (int)c.N;
  return be.hoist_const(H);
}
inline size_t rotate_modup_work_elems(const CtxView &c, int ell) { return (size_t)2 * (ell + 1) * c.N + (size_t)2 * c.N; }   // acc + tmp
template <class BE>
int rotate_modup_prepared_impl(BE &be, const CtxView &c, int ell, u64 *out, const u64 *a, const u64 *ext, const u32 *nperm, const u64 *key, const u64 *cadd, u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  u64 *acc = work, *tmp = work + (size_t)2 * (ell + 1) * c.N;
  return ks_finish(be, c, ell, out, a + (size_t)ell * c.N, ext, key, a, 1, acc, tmp, nperm, nperm, cadd);
}

// n <= 16 rotations of one ciphertext in three launches (inner products, inverse NTT of the 2n P-rows, forward NTT + division of
// the 2n ell rows) instead of 3n: out [n][2][ell][N], same bits as n calls of rotate_modup_prepared_impl.
inline size_t rotate_modup_many_work_elems(const CtxView &c, int ell, int n) { return (size_t)n * 2 * (ell + 1) * c.N + (size_t)n * 2 * c.N; }
template <class BE>
int rotate_modup_many_impl(BE &be, const CtxView &c, int ell, int n, u64 *out, const u64 *a, const u64 *ext, const u32 *const *perms,
                           const u64 *const *keys, const u64 *const *cadds, u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate needs 1 <= ell <= k-1");
  if (n < 1 || n > ROTMANY_MAX) return be.error("rotate_modup_many: 1..16 rotations");
  const long long N = (long long)c.N;
  u64 *acc = work, *tmp = work + (size_t)n * 2 * (ell + 1) * N;
  RotManyArgs A;
  memset(&A, 0, sizeof(A));
  A.t = a + (size_t)ell * N; A.ext = ext; A.acc = acc; A.primes = c.primes; A.n = n; A.ell = ell; A.k = c.k; A.N = (int)N;
  for (int i = 0; i < n; i++) { A.perm[i] = perms[i]; A.key[i] = keys[i]; A.cadd[i] = cadds[i]; }
  if (int rc = be.rot_many(A)) return rc;
  unsigned char pm[32];
  for (int i = 0; i < ell; i++) pm[i] = (unsigned char)i;
  return divround_impl(be, c, acc, (long long)(ell + 1) * N, 2 * n, ell + 1, pm, c.k - 1, out, (long long)ell * N, (const u64 *)nullptr, 0, tmp);
}

// ---- rotate_wsum: out_o = sum_i w_oi (.) rotate(a, g_i) + sum_t w_ot (.) taps[t], every w a scalar plaintext [ell][N] (null: 0), in
// four launches: the inner products of rotate_modup_many_impl, the inverse NTT of their 2n P rows, the weighting (k_rot_wsum, see
// WsumArgs) and the forward NTT + division of the 2 nout ell weighted rows.  Same bits as rotate -> multiply_plain -> add: the
// forward NTT is linear, so it commutes with the weighting, and every rotation keeps its own rounding by P.  n(2 + 2 ell)
// transforms become 2n + 2 nout ell.  taps: size-2 ciphertexts at level ell (plain multiply_plain leaves of the sums).
// out [nout][2][ell][N]; wts[o*n+i], twts[o*ntap+t]; work: rotate_wsum_work_elems.
inline size_t rotate_wsum_work_elems(const CtxView &c, int ell, int n, int nout) {
  return rotate_modup_many_work_elems(c, ell, n) + (size_t)2 * nout * 2 * ell * c.N;
}
template <class BE>
int rotate_wsum_impl(BE &be, const CtxView &c, int ell, int nout, u64 *out, const u64 *a, const u64 *ext, int n, const u32 *const *perms,
                     const u64 *const *keys, const u64 *const *cadds, const u64 *const *wts, int ntap, const u64 *const *taps,
                     const u64 *const *twts, u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("rotate_wsum needs 1 <= ell <= k-1");
  if (n < 1 || n > WS_MAX) return be.error("rotate_wsum: 1..16 rotations");
  if (nout < 1 || nout > WS_OUT) return be.error("rotate_wsum: 1..4 output sums");
  if (ntap < 0 || ntap > WS_TAPS) return be.error("rotate_wsum: 0..16 plain taps");
  const long long N = (long long)c.N;
  u64 *acc = work, *tmp = acc + (size_t)n * 2 * (ell + 1) * N;
  u64 *A = tmp + (size_t)n * 2 * N, *D = A + (size_t)nout * 2 * ell * N;
  RotManyArgs R;
  memset(&R, 0, sizeof(R));
  R.t = a + (size_t)ell * N; R.ext = ext; R.acc = acc; R.primes = c.primes; R.n = n; R.ell = ell; R.k = c.k; R.N = (int)N;
  for (int i = 0; i < n; i++) { R.perm[i] = perms[i]; R.key[i] = keys[i]; R.cadd[i] = cadds[i]; }
  if (int rc = be.rot_many(R)) return rc;
  if (int rc = divround_inv_impl(be, c, acc, (long long)(ell + 1) * N, 2 * n, ell + 1, c.k - 1, tmp)) return rc;
  WsumArgs W;
  memset(&W, 0, sizeof(W));
  W.acc = acc; W.tmp = tmp; W.A = A; W.D = D; W.primes = c.primes; W.halfmod = c.halfmod + (size_t)(c.k - 1) * c.k;
  W.n = n; W.ntap = ntap; W.nout = nout; W.ell = ell; W.k = c.k; W.N = (int)N;
  for (int o = 0; o < nout; o++) {
    for (int i = 0; i < n; i++) W.wt[o][i] = wts[(size_t)o * n + i];
    for (int t = 0; t < ntap; t++) W.twt[o][t] = twts[(size_t)o * ntap + t];
  }
  for (int t = 0; t < ntap; t++) W.tap[t] = taps[t];
  if (int rc = be.rot_wsum(W)) return rc;
  NttLaunch B = base_launch(c);
  B.src = D; B.src_sq = ell * N; B.src_sr = N;
  B.aux0 = A; B.aux0_sq = ell * N; B.aux0_sr = N;
  B.dst = out; B.dst_sq = ell * N; B.dst_sr = N;
  B.inner = ell; B.prime_on_q = 0;
  for (int r = 0; r < ell; r++) { B.pmap[r] = (unsigned char)r; B.pmap2[r] = (unsigned char)(c.k - 1); }
  B.pro = PRO_PLAIN; B.epi = EPI_DIVROUND;
  B.consts = c.qinv + (size_t)(c.k - 1) * c.k;
  B.consts_f = c.qinv_f + (size_t)(c.k - 1) * c.k;
  return be.fwd(B, (size_t)nout * 2 * ell);
}

// seal::CKKSEncoder::encode (vector overload) for a batch of vectors -- reference
// eva/seal/seal_executor.h:242.  d_values/vec/scale are host arrays of `count` entries.
template <class BE>
int encode_impl(BE &be, const CtxView &c, int count, const double *const *d_values, const u32 *vec, const double *scale, int ell,
                u64 *out, cplx *work, int with_p = 0) {
  if (ell < 1 || ell + (with_p ? 1 : 0) > c.k) return be.error("encode: ell out of range");
  if (with_p) ell = ell + 1;
  const u32 slots = (u32)(c.N / 2);
  for (int e0 = 0; e0 < count; e0 += ENC_MAX_BATCH) {
    EncBatch B;
    memset(&B, 0, sizeof(B));
    B.count = (u32)((count - e0) < ENC_MAX_BATCH ? (count - e0) : ENC_MAX_BATCH);
    for (u32 e = 0; e < B.count; e++) {
      if (vec[e0 + e] == 0 || slots % vec[e0 + e]) return be.error("Vector size must exactly divide the slot count");
      B.vals[e] = d_values[e0 + e]; B.vec[e] = vec[e0 + e]; B.scale[e] = scale[e0 + e];
    }
    B.work = work + (size_t)e0 * c.N; B.out = out + (size_t)e0 * ell * c.N;
    B.flags = encode_flags(c, count, work) + e0;
    B.roots = c.roots; B.slot_index = c.slot_index; B.primes = c.primes; B.pow2 = c.pow2;
    B.N = (u32)c.N; B.ell = (u32)ell;
    B.special_row = with_p ? (u32)(c.k - 1) : 0u;
    if (int rc = be.enc_scatter(B)) return rc;
    int done = 0;
    for (u32 g = 1; done < c.logN;) {
      const int ns = (c.logN - done) >= 3 ? 3 : (c.logN - done);
      if (int rc = be.enc_fft(B, g, ns)) return rc;   // N/8 threads, 8 elements each
      done += ns; g <<= ns;
    }
    if (int rc = be.enc_round(B)) return rc;
  }
  // forward NTT of every residue, batched: job (q = vector, r = residue)
  NttLaunch L = base_launch(c);
  L.src = out; L.dst = out; L.inner = ell;
  L.src_sq = L.dst_sq = (long long)ell * c.N; L.src_sr = L.dst_sr = (long long)c.N;
  for (int i = 0; i < ell; i++) L.pmap[i] = (unsigned char)((with_p && i + 1 == ell) ? c.k - 1 : i);
  // scalar constants (the common case in EVA programs) encode to constant polynomials
  L.cflags = encode_flags(c, count, work);
  return be.fwd(L, (size_t)count * ell);
}

// ---- lazy_rotsum (opt-in, approximate: SURVEY 8f-4): out [2][ell][N] = sum_i w_i (.) rotate(x, g_i) with ONE mod-down for the sum.
// ext: the shared extended digits of x (rotate_modup_prepare_impl); perms / keys / cadds as for rotate_modup_prepared_impl;
// out [nout][2][ell][N]; wts[o*n+i]: plaintext [ell+1][N] whose last row is the residue mod P (encode_*_impl with_p), null when rotation i
// is not part of sum o.  work: lazy_rotsum_work_elems.
inline size_t lazy_rotsum_work_elems(const CtxView &c, int ell, int nout) { return (size_t)nout * 2 * (ell + 1) * c.N + (size_t)nout * 2 * c.N; }
template <class BE>
int lazy_rotsum_impl(BE &be, const CtxView &c, int ell, int nout, u64 *out, const u64 *a, const u64 *ext, int n, const u32 *const *perms,
                     const u64 *const *keys, const u64 *const *cadds, const u64 *const *wts, u64 *work) {
  if (ell < 1 || ell > c.k - 1) return be.error("lazy_rotsum needs 1 <= ell <= k-1");
  if (n < 1 || n > LRS_MAX) return be.error("lazy_rotsum: 1..16 rotations");
  if (nout < 1 || nout > LRS_OUT) return be.error("lazy_rotsum: 1..4 output sums");
  const long long N = (long long)c.N;
  u64 *acc = work, *tmp = work + (size_t)nout * 2 * (ell + 1) * N;
  LazyRotSumArgs A;
  memset(&A, 0, sizeof(A));
  A.t = a + (size_t)ell * N; A.ext = ext; A.acc = acc; A.primes = c.primes; A.n = n; A.nout = nout; A.ell = ell; A.k = c.k; A.N = (int)N;
  for (int i = 0; i < n; i++) { A.perm[i] = perms[i]; A.key[i] = keys[i]; A.cadd[i] = cadds[i]; }
  for (int o = 0; o < nout; o++) for (int i = 0; i < n; i++) A.wt[o][i] = wts[(size_t)o * n + i];
  if (int rc = be.lazy_rotsum(A)) return rc;
  unsigned char pm[32];
  for (int i = 0; i < ell; i++) pm[i] = (unsigned char)i;
  return divround_impl(be, c, acc, (long long)(ell + 1) * N, 2 * nout, ell + 1, pm, c.k - 1, out, (long long)ell * N, (const u64 *)nullptr, 0, tmp);
}

// seal::CKKSEncoder::decode of a plaintext [ell][N] (NTT form) -> N/2 slot values (reference eva/seal/seal.cpp:132-146).
// d_tmp: ell*N words (the coefficient form), d_work: N complex values, d_out: N/2 doubles.  CRT constants come from the host.
inline size_t decode_tmp_elems(const CtxView &c, int ell) { return (size_t)ell * c.N; }
template <class BE>
int decode_impl(BE &be, const CtxView &c, int ell, const u64 *primes_host, const u64 *pt, double scale, double *out, u64 *tmp, cplx *work) {
  if (ell < 1 || ell > c.k || ell > DEC_MAX_ELL) return be.error("decode: ell out of range (1..8)");
  typedef unsigned __int128 u128;
  const int nw = ell + 1;
  DecArgs A;
  memset(&A, 0, sizeof(A));
  auto big_mul = [&](u64 *x, u64 m) { u64 carry = 0; for (int w = 0; w < nw; w++) { const u128 t = (u128)x[w] * m + carry; x[w] = (u64)t; carry = (u64)(t >> 64); } };
  auto big_mod = [&](const u64 *x, u64 m) { u128 r = 0; for (int w = nw - 1; w >= 0; w--) r = ((r << 64) | x[w]) % m; return (u64)r; };
  A.Q[0] = 1;
  for (int i = 0; i < ell; i++) big_mul(A.Q, primes_host[i]);
  for (int i = 0; i < ell; i++) {
    A.punct[i][0] = 1;
    for (int j = 0; j < ell; j++) if (j != i) big_mul(A.punct[i], primes_host[j]);
    // inverse by Fermat: q_i prime
    const u64 p = primes_host[i];
    u64 base = big_mod(A.punct[i], p), e = p - 2, r = 1;
    while (e) { if (e & 1) r = (u64)((u128)r * base % p); base = (u64)((u128)base * base % p); e >>= 1; }
    A.ipunct[i] = r;
  }
  for (int w = 0; w < nw; w++) A.halfQ[w] = A.Q[w];
  { u64 carry = 1; for (int w = 0; w < nw && carry; w++) { A.halfQ[w] += carry; carry = A.halfQ[w] == 0; } }
  for (int w = 0; w < nw; w++) A.halfQ[w] = (A.halfQ[w] >> 1) | (w + 1 < nw ? A.halfQ[w + 1] << 63 : 0);
  // coefficient form
  if (int rc = copy_impl(be, c, ell, ell, tmp, pt, 1)) return rc;
  int pidx[32];
  for (int i = 0; i < ell; i++) pidx[i] = i;
  if (int rc = ntt_batch_impl(be, c, true, tmp, (size_t)ell, pidx, ell)) return rc;
  A.coef = tmp; A.work = work; A.out = out; A.roots = c.roots; A.slot_index = c.slot_index; A.primes = c.primes;
  A.inv_scale = 1.0 / scale; A.N = (u32)c.N; A.ell = (u32)ell;
  if (int rc = be.dec_compose(A)) return rc;
  for (u32 m = 1; m < A.N; m <<= 1)
    if (int rc = be.dec_fft(A, m)) return rc;
  return be.dec_gather(A);
}
