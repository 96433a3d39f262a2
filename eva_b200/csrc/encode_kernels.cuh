// encode_kernels.cuh -- CKKS encoder on the device (SURVEY.md 8a row E, Appendix A.9):
// seal::CKKSEncoder::encode as called at reference eva/seal/seal_executor.h:242 /
// seal.cpp:68,80.  values (vec_size doubles, replicated over N/2 slots) ->
// inverse canonical-embedding FFT in FP64 -> round(x * scale / N) -> residues
// mod each prime; the forward NTT of the residues is done by the NTT kernel.
//
// FP64 arithmetic is written with explicit round-to-nearest operations (no FMA
// contraction) in the same order as the host encoders, so device, host and
// oracle encodings agree bit for bit; twiddles come from the host (libm).
// Bodies are __host__ __device__ so the tests replay them on the CPU.
#pragma once
#include "modarith.cuh"
#include <math.h>
#include <string.h>

struct __align__(16) cplx { double re, im; };

#if defined(__CUDA_ARCH__)
#define D_ADD(a, b) __dadd_rn(a, b)
#define D_SUB(a, b) __dsub_rn(a, b)
#define D_MUL(a, b) __dmul_rn(a, b)
#else
#define D_ADD(a, b) ((a) + (b))
#define D_SUB(a, b) ((a) - (b))
#define D_MUL(a, b) ((a) * (b))
#endif

#define ENC_MAX_BATCH 32
struct EncBatch {
  const double *vals[ENC_MAX_BATCH];  // device: vec_size values each
  u32 vec[ENC_MAX_BATCH];
  double scale[ENC_MAX_BATCH];
  cplx *work;                         // [count][N]
  u64 *flags;                         // [count]: 1 when vector e encodes to a non-constant polynomial
  u64 *out;                           // [count][ell][N] coefficient-form residues
  const cplx *roots;                  // [N] zeta^bitrev(i)
  const u32 *slot_index;              // [N]
  const PrimeDev *primes;
  const u64 *pow2;                    // [k][ENC_POW2_ROW]: 2^i mod p
  u32 N, ell, count;
  u32 special_row;                    // != 0: the LAST of the ell rows is the residue mod prime `special_row` (the key-switch
                                      // prime P: plaintexts that multiply un-modded-down key-switch accumulators, lazy_rotsum)
};
EVAB_HD u32 enc_prime_of_row(u32 i, u32 ell, u32 special_row) { return (special_row && i + 1 == ell) ? special_row : i; }

// scatter: slot i (and its conjugate slot) <- values[i mod vec]
// off / voff: per-instance element offsets (u64 words / doubles) of a batched launch
EVAB_HD void enc_scatter(const EncBatch &B, u32 e, u32 i, long long off = 0, long long voff = 0) {
  const u32 slots = B.N >> 1;
  const double v = (B.vals[e] + voff)[i % B.vec[e]];
  cplx *w = B.work + off / 2 + (size_t)e * B.N;
  cplx c; c.re = v; c.im = 0.0;
  if (i == 0) (B.flags + off)[e] = 0;   // set again by enc_round when a coefficient j > 0 is non-zero
  w[B.slot_index[i]] = c;
  w[B.slot_index[slots + i]] = c;
}

// one Gentleman-Sande butterfly with the conjugate twiddle of roots[idx]
EVAB_HD void enc_bfly(cplx &x, cplx &y, const cplx r) {
  const double wr = r.re, wi = -r.im;
  const double ur = x.re, ui = x.im, vr = y.re, vi = y.im;
  x.re = D_ADD(ur, vr); x.im = D_ADD(ui, vi);
  const double dr = D_SUB(ur, vr), di = D_SUB(ui, vi);
  y.re = D_SUB(D_MUL(dr, wr), D_MUL(di, wi));
  y.im = D_ADD(D_MUL(dr, wi), D_MUL(di, wr));
}
// NS consecutive inverse-FFT stages (gaps g, 2g, .. 2^(NS-1) g) on one closed set of
// 2^NS elements spaced g apart; set u of N / 2^NS
template <int NS> EVAB_HD void enc_fft_set(const EncBatch &B, u32 e, u32 u, u32 g, long long off) {
  constexpr int M = 1 << NS;
  cplx *w = B.work + off / 2 + (size_t)e * B.N;
  const u32 low = u % g, high = u / g;
  const u32 base = high * (M * g) + low;
  cplx x[M];
#pragma unroll
  for (int j = 0; j < M; j++) x[j] = w[base + j * g];
#pragma unroll
  for (int st = 0; st < NS; st++) {
    const int d = 1 << st;                 // pair distance in units of g
    const u32 gap = g << st;
    const u32 m = B.N / (2 * gap);
#pragma unroll
    for (int j = 0; j < M; j++)
      if (!(j & d)) enc_bfly(x[j], x[j + d], B.roots[m + (base + j * g) / (2 * gap)]);
  }
#pragma unroll
  for (int j = 0; j < M; j++) w[base + j * g] = x[j];
}
// thread t of N/8 handles 8 elements = 8 / 2^nstages closed sets
EVAB_HD void enc_fft8(const EncBatch &B, u32 e, u32 t, u32 g, int nstages, long long off = 0) {
  if (nstages == 3) enc_fft_set<3>(B, e, t, g, off);
  else if (nstages == 2) { enc_fft_set<2>(B, e, 2 * t, g, off); enc_fft_set<2>(B, e, 2 * t + 1, g, off); }
  else { for (u32 s = 0; s < 4; s++) enc_fft_set<1>(B, e, 4 * t + s, g, off); }
}

// rounded coefficient c (an integer-valued double of any finite magnitude) -> residue mod prime i
// (sign-aware; exact beyond 2^64 through mantissa * 2^shift, 1 <= shift <= 960 < ENC_POW2_ROW)
EVAB_HD u64 enc_residue(double c, const PrimeDev &P, const u64 *pow2_row) {
  const bool neg = signbit(c);
  const double mag = fabs(c);
  u64 mant; int sh = 0;
  if (mag < 18446744073709551616.0) mant = (u64)mag;
  else { int ex; const double fr = frexp(mag, &ex); mant = (u64)ldexp(fr, 64); sh = ex - 64; }
  u64 v = barrett64(mant, P.p, P.ratio64);
  // the mask is the identity for every finite c; it only keeps a non-finite input's read inside the row
  if (sh) v = mulmod(v, pow2_row[sh & (ENC_POW2_ROW - 1)], P.p, P.ratio_lo, P.ratio_hi);
  return (neg && v) ? P.p - v : v;
}
// coefficient j: round(re * scale / N) -> residue mod every prime
EVAB_HD void enc_round(const EncBatch &B, u32 e, u32 j, long long off = 0) {
  const double fix = B.scale[e] / (double)B.N;
  const double c = round(D_MUL((B.work + off / 2)[(size_t)e * B.N + j].re, fix));
  if (j > 0 && c != 0.0) (B.flags + off)[e] = 1;
  for (u32 i = 0; i < B.ell; i++) {
    const u32 pi = enc_prime_of_row(i, B.ell, B.special_row);
    (B.out + off)[((size_t)e * B.ell + i) * B.N + j] = enc_residue(c, B.primes[pi], B.pow2 + (size_t)pi * ENC_POW2_ROW);
  }
}

// ---- uniform vectors (every scalar constant of an EVA program, constant_value.h:64-71): all N
// inputs of the inverse FFT are equal, so every butterfly difference is exactly zero and every sum
// an exact doubling: the FFT output is value * N at index 0 and zero elsewhere, the plaintext is the
// constant polynomial round((value * N) * (scale / N)) and its NTT is that constant at every point.
// enc_uniform writes exactly what scatter -> FFT -> enc_round -> NTT produce, in one pass.
struct EncUniform {
  double value[ENC_MAX_BATCH], scale[ENC_MAX_BATCH];
  u64 *out;                 // [count][ell][N]
  const PrimeDev *primes;
  const u64 *pow2;
  u32 N, ell, count;
  u32 special_row;          // see EncBatch
};
// coefficients j, j+1 of residue row (e, i)
EVAB_HD void enc_uniform_elem(const EncUniform &B, u32 e, u32 i, u32 j, long long off = 0) {
  const double re = D_MUL(B.value[e], (double)B.N);            // log2(N) exact doublings of the FFT
  const double c = round(D_MUL(re, B.scale[e] / (double)B.N));
  const u32 pi = enc_prime_of_row(i, B.ell, B.special_row);
  const u64 r = enc_residue(c, B.primes[pi], B.pow2 + (size_t)pi * ENC_POW2_ROW);
  u64x2 v; v.x = r; v.y = r;
  *reinterpret_cast<u64x2 *>(B.out + off + ((size_t)e * B.ell + i) * B.N + j) = v;
}

// ---- decoder on the device (SURVEY 8f-1): seal::CKKSEncoder::decode as called at reference eva/seal/seal.cpp:132-146.
// coefficient residues (after the inverse NTT) -> CRT composition to a centred multi-word integer -> double / scale ->
// forward canonical-embedding FFT (Cooley-Tukey, natural in, bit-reversed out) -> the N/2 slot values.  Same operation
// order, explicit round-to-nearest, as the host decoder and the oracle (ora_decode): identical doubles.
#define DEC_MAX_ELL 8
#define DEC_WORDS (DEC_MAX_ELL + 1)
// CRT constants of the first ell primes (multi-word, little-endian u64 words; ell + 1 words are used)
struct CrtTables {
  u64 Q[DEC_WORDS], halfQ[DEC_WORDS];        // Q = q_0 ... q_{ell-1}, (Q + 1) / 2
  u64 punct[DEC_MAX_ELL][DEC_WORDS];         // Q / q_i
  u64 ipunct[DEC_MAX_ELL];                   // (Q / q_i)^-1 mod q_i
};
struct DecArgs {
  const u64 *coef;              // [ell][N] coefficient-form residues
  cplx *work;                   // [N]
  double *out;                  // [N/2] slot values
  const cplx *roots;            // [N] zeta^bitrev(i)
  const u32 *slot_index;        // [N]
  const PrimeDev *primes;
  CrtTables T;
  double inv_scale;
  u32 N, ell;
};
EVAB_HD int dec_cmp(const u64 *a, const u64 *b, int nw) {
  for (int i = nw - 1; i >= 0; i--) { if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1; }
  return 0;
}
EVAB_HD void dec_sub(u64 *a, const u64 *b, int nw) {   // a -= b
  u64 borrow = 0;
  for (int i = 0; i < nw; i++) { const u64 t = a[i] - b[i], t2 = t - borrow; borrow = (a[i] < b[i]) | (t < borrow); a[i] = t2; }
}
// X (ell + 1 words) = the CRT composition in [0, Q) of the residues coef[i * stride], i < ell
EVAB_HD void crt_compose(const CrtTables &T, const PrimeDev *primes, u32 ell, const u64 *coef, size_t stride, u64 *X) {
  const int nw = (int)ell + 1;
  for (int w = 0; w < nw; w++) X[w] = 0;
  for (u32 i = 0; i < ell; i++) {
    const PrimeDev P = primes[i];
    const u64 v = mulmod(coef[(size_t)i * stride], T.ipunct[i], P.p, P.ratio_lo, P.ratio_hi);
    u64 carry = 0;                                        // X += punct[i] * v
    for (int w = 0; w < nw; w++) {
      const u64 lo = T.punct[i][w] * v, hi = mulhi64(T.punct[i][w], v);
      const u64 s = X[w] + lo, c1 = s < lo;
      const u64 s2 = s + carry, c2 = s2 < carry;
      X[w] = s2; carry = hi + c1 + c2;
    }
  }
  while (dec_cmp(X, T.Q, nw) >= 0) dec_sub(X, T.Q, nw);
}
// coefficient j -> work[j] = (centred CRT value / scale, 0)
EVAB_HD void dec_compose(const DecArgs &A, u32 j) {
  const int nw = (int)A.ell + 1;
  u64 X[DEC_WORDS];
  crt_compose(A.T, A.primes, A.ell, A.coef + j, A.N, X);
  const bool neg = dec_cmp(X, A.T.halfQ, nw) >= 0;
  if (neg) { u64 T[DEC_WORDS]; for (int w = 0; w < nw; w++) T[w] = A.T.Q[w]; dec_sub(T, X, nw); for (int w = 0; w < nw; w++) X[w] = T[w]; }
  double acc = 0.0, f = A.inv_scale;
  for (int w = 0; w < nw; w++) { if (X[w]) acc = D_ADD(acc, D_MUL((double)X[w], f)); f = D_MUL(f, 18446744073709551616.0); }
  cplx c; c.re = neg ? -acc : acc; c.im = 0.0;
  A.work[j] = c;
}
// stage with m groups (m = 1, 2, 4, ...; t = N / (2m)): butterfly b of N/2
EVAB_HD void dec_fft_bfly(const DecArgs &A, u32 m, u32 b) {
  const u32 t = A.N / (2 * m), i = b / t, j = 2 * i * t + b % t;
  const cplx r = A.roots[m + i];
  cplx *w = A.work;
  const double vr = D_SUB(D_MUL(w[j + t].re, r.re), D_MUL(w[j + t].im, r.im));
  const double vi = D_ADD(D_MUL(w[j + t].re, r.im), D_MUL(w[j + t].im, r.re));
  const double ur = w[j].re, ui = w[j].im;
  w[j].re = D_ADD(ur, vr); w[j].im = D_ADD(ui, vi);
  w[j + t].re = D_SUB(ur, vr); w[j + t].im = D_SUB(ui, vi);
}
EVAB_HD void dec_gather(const DecArgs &A, u32 i) { A.out[i] = A.work[A.slot_index[i]].re; }

// host: the CRT constants of primes[0 .. ell), 1 <= ell <= DEC_MAX_ELL
inline void crt_tables(CrtTables &T, const u64 *primes, int ell) {
  typedef unsigned __int128 u128;
  const int nw = ell + 1;
  memset(&T, 0, sizeof(T));
  auto big_mul = [&](u64 *x, u64 m) { u64 carry = 0; for (int w = 0; w < nw; w++) { const u128 t = (u128)x[w] * m + carry; x[w] = (u64)t; carry = (u64)(t >> 64); } };
  auto big_mod = [&](const u64 *x, u64 m) { u128 r = 0; for (int w = nw - 1; w >= 0; w--) r = ((r << 64) | x[w]) % m; return (u64)r; };
  T.Q[0] = 1;
  for (int i = 0; i < ell; i++) big_mul(T.Q, primes[i]);
  for (int i = 0; i < ell; i++) {
    T.punct[i][0] = 1;
    for (int j = 0; j < ell; j++) if (j != i) big_mul(T.punct[i], primes[j]);
    // inverse by Fermat: q_i prime
    const u64 p = primes[i];
    u64 base = big_mod(T.punct[i], p), e = p - 2, r = 1;
    while (e) { if (e & 1) r = (u64)((u128)r * base % p); base = (u64)((u128)base * base % p); e >>= 1; }
    T.ipunct[i] = r;
  }
  for (int w = 0; w < nw; w++) T.halfQ[w] = T.Q[w];
  { u64 carry = 1; for (int w = 0; w < nw && carry; w++) { T.halfQ[w] += carry; carry = T.halfQ[w] == 0; } }
  for (int w = 0; w < nw; w++) T.halfQ[w] = (T.halfQ[w] >> 1) | (w + 1 < nw ? T.halfQ[w + 1] << 63 : 0);
}
