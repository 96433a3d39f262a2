// host_tables.hpp -- host-side number theory for building the per-prime NTT
// tables and RNS constants (SEAL 3.6 conventions, SURVEY.md Appendix A.1-A.3,
// A.6).  Product code (used by evab200.cu); also compiled into the CPU kernel
// emulator used by the tests.
#pragma once
#include "modarith.cuh"
#include <cmath>
#include <vector>

namespace evab_host {
typedef unsigned __int128 u128;
inline u64 mulmod(u64 a, u64 b, u64 p) { return (u64)(((u128)a * b) % p); }
inline u64 powmod(u64 a, u64 e, u64 p) {
  u64 r = 1 % p; a %= p;
  while (e) { if (e & 1) r = mulmod(r, a, p); a = mulmod(a, a, p); e >>= 1; }
  return r;
}
inline u64 shoup(u64 w, u64 p) { return (u64)(((u128)w << 64) / p); }
inline u64 row32(u64 w, u64 p) { return (u64)(((u128)w << 32) % p); }   // companion row of the two-row fold product
inline u32 bitrev(u32 x, int bits) { u32 r = 0; for (int i = 0; i < bits; i++) { r = (r << 1) | (x & 1); x >>= 1; } return r; }
// numerically smallest primitive 2N-th root of unity mod p (0 if none)
inline u64 min_root(u64 N, u64 p) {
  if ((p - 1) % (2 * N)) return 0;
  u64 e = (p - 1) / (2 * N), root = 0;
  for (u64 g = 2; g < p && !root; g++) {
    u64 r = powmod(g, e, p);
    if (powmod(r, N, p) == p - 1) root = r;
  }
  if (!root) return 0;
  u64 sq = mulmod(root, root, p), cur = root, best = root;
  for (u64 i = 0; i < N; i++) { if (cur < best) best = cur; cur = mulmod(cur, sq, p); }
  return best;
}

struct cplxh { double re, im; };
// e^(2 pi i index / degree) from the first octant + symmetries (SEAL ComplexRoots::get_root)
inline void unit_root(u64 index, u64 degree, double &re, double &im) {
  const double PI = 3.1415926535897932384626433832795028842;
  index &= degree - 1;
  double a, b;
  if (index <= degree / 8) { const double ang = 2.0 * PI * (double)index / (double)degree; re = cos(ang); im = sin(ang); }
  else if (index <= degree / 4) { unit_root(degree / 4 - index, degree, a, b); re = b; im = a; }
  else if (index <= degree / 2) { unit_root(degree / 2 - index, degree, a, b); re = -a; im = b; }
  else if (index <= 3 * degree / 4) { unit_root(index - degree / 2, degree, a, b); re = -a; im = -b; }
  else { unit_root(degree - index, degree, a, b); re = a; im = -b; }
}
struct Tables {
  std::vector<cplxh> roots;        // [N] zeta^bitrev(i), zeta = e^(2 pi i / 2N)   (CKKS encoder)
  std::vector<u32> slot_index;     // [N] matrix_reps_index_map
  std::vector<u64> pow2;           // [k][ENC_POW2_ROW] 2^i mod p
  std::vector<u64x2> tw;       // [k][2][N]  forward / inverse {w, shoup(w)} in bit-reversed power order,
                               // followed by [k][2][N] {w, w * 2^32 mod p} (fold rows; zero for primes that are not fold-friendly)
  std::vector<PrimeDev> pd;    // tw / itw pointers are filled relative to `tw_base`
  std::vector<u64x2> qinv;     // [last][i]  {q_last^-1 mod q_i, shoup}
  std::vector<u64x2> qinv_f;   // [last][i]  {q_last^-1 mod q_i, * 2^32 mod q_i}   (fold row)
  unsigned foldmask = 0;       // bit i: primes[i] is fold-friendly
  std::vector<FoldPrime> fp;   // [k] fold constants (kernel-parameter copy)
  std::vector<u64> halfmod;    // [last][i]  floor(q_last/2) mod q_i
};

// returns empty string on success
inline const char *build_tables(u64 N, int logN, const u64 *primes, int k, const u64x2 *tw_base, Tables &T) {
  T.tw.assign((size_t)k * 4 * N, u64x2{0, 0});
  T.foldmask = 0;
  T.pd.resize(k);
  T.fp.assign(k, FoldPrime{});
  for (int i = 0; i < k; i++) {
    u64 p = primes[i];
    if (p < 3 || (p >> 60)) return "primes must be odd and < 2^60";
    u64 psi = min_root(N, p);
    if (!psi) return "prime is not congruent to 1 mod 2N";
    u64 ipsi = powmod(psi, p - 2, p), pw = 1, ipw = 1;
    u64x2 *f = &T.tw[((size_t)i * 2 + 0) * N], *b = &T.tw[((size_t)i * 2 + 1) * N];
    u64x2 *ff = &T.tw[((size_t)(k + i) * 2 + 0) * N], *fb = &T.tw[((size_t)(k + i) * 2 + 1) * N];
    const bool fold = prime_foldable(p);
    if (fold) T.foldmask |= 1u << i;
    for (u64 j = 0; j < N; j++) {
      u32 r = bitrev((u32)j, logN);
      f[r].x = pw; f[r].y = shoup(pw, p);
      b[r].x = ipw; b[r].y = shoup(ipw, p);
      if (fold) { ff[r].x = pw; ff[r].y = row32(pw, p); fb[r].x = ipw; fb[r].y = row32(ipw, p); }
      pw = mulmod(pw, psi, p); ipw = mulmod(ipw, ipsi, p);
    }
    PrimeDev &P = T.pd[i];
    P.p = p;
    u128 ratio = ~(u128)0 / p;
    P.ratio_lo = (u64)ratio; P.ratio_hi = (u64)(ratio >> 64);
    P.ratio64 = (u64)(((u128)1 << 64) / p);
    P.ninv = powmod(N % p, p - 2, p); P.ninv_s = shoup(P.ninv, p);
    P.itw1n = mulmod(b[1].x, P.ninv, p); P.itw1n_s = shoup(P.itw1n, p);
    P.tw = tw_base + ((size_t)i * 2 + 0) * N;
    P.itw = tw_base + ((size_t)i * 2 + 1) * N;
    P.ftw = tw_base + ((size_t)(k + i) * 2 + 0) * N;
    P.fitw = tw_base + ((size_t)(k + i) * 2 + 1) * N;
    P.ninv_v = row32(P.ninv, p); P.itw1n_v = row32(P.itw1n, p);
    P.foldable = fold ? 1u : 0u; P.eps = fold ? fold_eps(p) : 0u;
    FoldPrime &F = T.fp[i];
    F.p = p; F.p3 = 3 * p; F.p8 = 8 * p; F.eps = P.eps; F.foldable = P.foldable;
    F.ftw = P.ftw; F.fitw = P.fitw; F.ninv = P.ninv; F.ninv_v = P.ninv_v; F.itw1n = P.itw1n; F.itw1n_v = P.itw1n_v;
  }
  T.roots.resize(N); T.slot_index.resize(N);
  for (u64 i = 0; i < N; i++) unit_root(bitrev((u32)i, logN), 2 * N, T.roots[i].re, T.roots[i].im);
  { const u64 m = 2 * N, slots = N / 2; u64 pos = 1;
    for (u64 i = 0; i < slots; i++) {
      T.slot_index[i] = bitrev((u32)((pos - 1) >> 1), logN);
      T.slot_index[slots | i] = bitrev((u32)((m - pos - 1) >> 1), logN);
      pos = (pos * 3) & (m - 1);
    } }
  T.pow2.assign((size_t)k * ENC_POW2_ROW, 0);
  for (int i = 0; i < k; i++) {
    u64 v = 1 % primes[i];
    for (int e = 0; e < ENC_POW2_ROW; e++) { T.pow2[(size_t)i * ENC_POW2_ROW + e] = v; v = mulmod(v, 2, primes[i]); }
  }
  T.qinv.assign((size_t)k * k, u64x2{0, 0});
  T.qinv_f.assign((size_t)k * k, u64x2{0, 0});
  T.halfmod.assign((size_t)k * k, 0);
  for (int last = 0; last < k; last++)
    for (int i = 0; i < k; i++) {
      if (i == last) continue;
      u64 p = primes[i], ql = primes[last];
      u64 inv = powmod(ql % p, p - 2, p);
      T.qinv[(size_t)last * k + i] = u64x2{inv, shoup(inv, p)};
      T.qinv_f[(size_t)last * k + i] = u64x2{inv, row32(inv, p)};
      T.halfmod[(size_t)last * k + i] = (ql >> 1) % p;
    }
  return "";
}

inline u64 galois_elt_from_step(u64 N, int steps) {
  const u64 m = 2 * N;
  if (steps == 0) return m - 1;
  u64 pos = steps < 0 ? (u64)(-(long long)steps) : (u64)steps;
  if (pos >= N / 2) return 0;
  u64 s = steps < 0 ? N / 2 - pos : pos, g = 1;
  for (u64 i = 0; i < s; i++) g = (g * 3) & (m - 1);
  return g;
}
inline void galois_table(u64 N, int logN, u64 elt, std::vector<u32> &tab) {
  tab.resize(N);
  for (u64 i = 0; i < N; i++) {
    u64 r = bitrev((u32)i, logN);
    u64 raw = ((elt * (2 * r + 1)) >> 1) & (N - 1);
    tab[i] = bitrev((u32)raw, logN);
  }
}
// coefficient-domain form of the same automorphism a(X) -> a(X^elt): output coefficient j is
// +-a_i with i = j * elt^-1 mod N; entry = (i << 1) | negate.  inverse_ntt(galois_table(x)) ==
// this signed gather applied to inverse_ntt(x) (with canonical negation p - v, 0 -> 0).
inline void galois_coeff_table(u64 N, u64 elt, std::vector<u32> &tab) {
  tab.assign(N, 0);
  const u64 m = 2 * N;
  for (u64 i = 0; i < N; i++) {
    const u64 pos = (i * elt) & (m - 1);
    if (pos < N) tab[pos] = (u32)(i << 1);
    else tab[pos - N] = (u32)((i << 1) | 1u);
  }
}
}  // namespace evab_host
