// ops_kernels.cuh -- element-wise (dyadic) ciphertext kernels, fused sums of
// products and the key-switch inner product, as __host__ __device__ bodies
// (two coefficients per call, 128-bit accesses) shared by the CUDA kernels and
// the CPU emulator.  Semantics: SURVEY.md Appendix A.4 / A.5 / A.8.
#pragma once
#include "ntt_core.cuh"
#include "key_expand.cuh"

enum { DY_ADD = 0, DY_SUB = 1, DY_NEG = 2, DY_MULPT = 3, DY_COPY = 4 };

struct DyArgs {
  u64 *out; const u64 *a; const u64 *b;
  const PrimeDev *primes;
  int ell, N;
  int sa, sb, sout;  // polys in a / b / out
  int b_is_plain;    // b = plaintext [ell][N]: add/sub touch poly 0 only, mulpt every poly
  int a_ell;         // residues per polynomial of `a` (>= ell; DY_COPY with a_ell = ell+1 drops the last residue)
};

EVAB_HD u64x2 ld2(const u64 *p) { return *reinterpret_cast<const u64x2 *>(p); }
EVAB_HD void st2(u64 *p, u64x2 v) { *reinterpret_cast<u64x2 *>(p) = v; }
// 4 contiguous coefficients = two 128-bit global accesses (128 bits is the widest global access on sm_90)
EVAB_HD void load4g(u64 (&a)[4], const u64 *p) {
#if defined(__CUDA_ARCH__)
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(a[0]), "=l"(a[1]) : "l"(p));
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(a[2]), "=l"(a[3]) : "l"(p + 2));
#else
  for (int k = 0; k < 4; k++) a[k] = p[k];
#endif
}
EVAB_HD void store4g(u64 *p, const u64 (&a)[4]) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a[0]), "l"(a[1]) : "memory");
  asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(p + 2), "l"(a[2]), "l"(a[3]) : "memory");
#else
  for (int k = 0; k < 4; k++) p[k] = a[k];
#endif
}

// coefficients j .. j+3 of output residue `res` (= s*ell + i): four coefficients per operand and lane, i.e. a
// full 32-byte sector per lane in two 128-bit accesses
// boff: batch instance offset (words) applied to every ciphertext / plaintext pointer
template <int OP> EVAB_HD void dyadic_elem(const DyArgs &A, int res, int j, long long boff = 0) {
  const int s = res / A.ell, i = res % A.ell;
  const PrimeDev P = A.primes[i];
  const u64 p = P.p;
  const size_t off = (size_t)res * A.N;
  const size_t aoff = ((size_t)s * A.a_ell + i) * A.N;
  const bool has_a = s < A.sa;
  const bool has_b = A.b_is_plain ? (OP == DY_MULPT || s == 0) : (s < A.sb);
  const size_t poff = A.b_is_plain ? (size_t)i * A.N : off;
  u64 va[4] = {0, 0, 0, 0}, vb[4] = {0, 0, 0, 0}, r[4];
  if (has_a) load4g(va, A.a + boff + aoff + j);
  if (OP != DY_NEG && OP != DY_COPY && has_b) load4g(vb, A.b + boff + poff + j);
#pragma unroll
  for (int e = 0; e < 4; e++) {
    if (OP == DY_ADD) r[e] = addmod(va[e], vb[e], p);
    else if (OP == DY_SUB) r[e] = submod(va[e], vb[e], p);
    else if (OP == DY_NEG) r[e] = negmod(va[e], p);
    else if (OP == DY_COPY) r[e] = va[e];
    else r[e] = mulmod_p(va[e], vb[e], P);
  }
  store4g(A.out + boff + off + j, r);
}

// Evaluator::multiply_plain: coefficients j .. j+3 of residue i of EVERY polynomial of the ciphertext -- the plaintext
// is loaded once per thread instead of once per polynomial (algorithmic traffic (2s + 1) ell R, SURVEY 8d)
EVAB_HD void mulpt_elem(const DyArgs &A, int i, int j, long long boff = 0) {
  const PrimeDev P = A.primes[i];
  u64 w[4];
  load4g(w, A.b + boff + (size_t)i * A.N + j);
  for (int s = 0; s < A.sa; s++) {
    u64 v[4];
    load4g(v, A.a + boff + ((size_t)s * A.a_ell + i) * A.N + j);
#pragma unroll
    for (int e = 0; e < 4; e++) v[e] = mulmod_p(v[e], w[e], P);
    store4g(A.out + boff + ((size_t)s * A.ell + i) * A.N + j, v);
  }
}

// fused sum of terms; term t is  ct[t]                      (kind 0: Evaluator::add operand),
//                               ct[t] * pt[t]              (kind 1: Evaluator::multiply_plain result), or
//                               ct[t] (x) ct2[t], 2x2 -> 3 (kind 2: Evaluator::multiply / square result)
// i.e. a chain of multiply_plain / multiply / add calls (reference seal_executor.h:124,162-168)
// evaluated in one pass.  Products are accumulated in 128 bits and reduced once; the canonical
// result equals the sequence of canonical products and sums (exact modular arithmetic).
#define SUM_MAX_TERMS 32
struct SumArgs {
  u64 *out;
  const u64 *ct[SUM_MAX_TERMS];
  const u64 *pt[SUM_MAX_TERMS];          // kind 1: plaintext [ell][N]; kind 2: second ciphertext [2][ell][N]
  unsigned char size[SUM_MAX_TERMS];    // polynomials of the term's value (kind 2: 3)
  unsigned char kind[SUM_MAX_TERMS];
  const PrimeDev *primes;
  int n, ell, N, sout;
};
// coefficients j, j+1 of output residue `res` (= s*ell + i); off = batch instance offset (words)
EVAB_HD void sum_terms_elem(const SumArgs &A, int res, int j, long long off) {
  const int s = res / A.ell, i = res % A.ell;
  const PrimeDev P = A.primes[i];
  const size_t poly = (size_t)A.ell * A.N;
  const size_t roff = (size_t)i * A.N + j;          // residue i of polynomial 0
  u64 lx = 0, hx = 0, ly = 0, hy = 0;
  for (int t = 0; t < A.n; t++) {
    if (s >= (int)A.size[t]) continue;
    const u64 *a = A.ct[t] + off + roff;
    if (A.kind[t] == 2) {
      const u64 *b = A.pt[t] + off + roff;
      // tensor product component s: (a0 b0, a0 b1 + a1 b0, a1 b1)
      const u64x2 a_lo = ld2(a + (s == 2 ? poly : 0)), b_hi = ld2(b + (s == 0 ? 0 : poly));
      mac128(lx, hx, a_lo.x, b_hi.x); mac128(ly, hy, a_lo.y, b_hi.y);
      if (s == 1) {
        const u64x2 a1 = ld2(a + poly), b0 = ld2(b);
        mac128(lx, hx, a1.x, b0.x); mac128(ly, hy, a1.y, b0.y);
      }
    } else {
      const u64x2 v = ld2(a + (size_t)s * poly);
      if (A.kind[t] == 1) {
        const u64x2 w = ld2(A.pt[t] + off + roff);
        mac128(lx, hx, v.x, w.x); mac128(ly, hy, v.y, w.y);
      } else {
        lx += v.x; hx += (lx < v.x);
        ly += v.y; hy += (ly < v.y);
      }
    }
  }
  u64x2 r;
  r.x = reduce128(lx, hx, P);
  r.y = reduce128(ly, hy, P);
  st2(A.out + off + (size_t)res * A.N + j, r);
}

struct MulArgs { u64 *out; const u64 *a; const u64 *b; const PrimeDev *primes; int ell, N; };

// 2x2 -> 3 tensor product (Evaluator::multiply) or square, residue i, coeffs j,j+1
template <bool SQUARE> EVAB_HD void mulct_elem(const MulArgs &A, int i, int j, long long boff = 0) {
  const PrimeDev P = A.primes[i];
  const u64 p = P.p;
  const size_t poly = (size_t)A.ell * A.N, off = (size_t)i * A.N + j;
  const u64 *pa = A.a + boff, *pb = SQUARE ? nullptr : A.b + boff;
  u64 *po = A.out + boff;
  const u64x2 a0 = ld2(pa + off), a1 = ld2(pa + poly + off);
  u64x2 d0, d1, d2;
  if (SQUARE) {
    d0.x = mulmod_p(a0.x, a0.x, P); d0.y = mulmod_p(a0.y, a0.y, P);
    u64 x0 = mulmod_p(a0.x, a1.x, P), x1 = mulmod_p(a0.y, a1.y, P);
    d1.x = addmod(x0, x0, p); d1.y = addmod(x1, x1, p);
    d2.x = mulmod_p(a1.x, a1.x, P); d2.y = mulmod_p(a1.y, a1.y, P);
  } else {
    const u64x2 b0 = ld2(pb + off), b1 = ld2(pb + poly + off);
    d0.x = mulmod_p(a0.x, b0.x, P); d0.y = mulmod_p(a0.y, b0.y, P);
    // a0*b1 + a1*b0 accumulated in 128 bits, then one reduction: same canonical value
    u64 lo = 0, hi = 0;
    mac128(lo, hi, a0.x, b1.x); mac128(lo, hi, a1.x, b0.x); d1.x = reduce128(lo, hi, P);
    lo = hi = 0;
    mac128(lo, hi, a0.y, b1.y); mac128(lo, hi, a1.y, b0.y); d1.y = reduce128(lo, hi, P);
    d2.x = mulmod_p(a1.x, b1.x, P); d2.y = mulmod_p(a1.y, b1.y, P);
  }
  st2(po + off, d0); st2(po + poly + off, d1); st2(po + 2 * poly + off, d2);
}

// key-switch inner product over digits (Appendix A.5 step 2):
// acc[c][m][j] = sum_J opnd(m,J)[j] * key[J][c][row(m)][j] mod m, with
// opnd(m,J) = t[J] when row(m)==J (the digit's own modulus) else ext[m][J].
struct IpArgs {
  const u64 *t, *ext, *key; u64 *acc; const PrimeDev *primes;
  const u32 *tperm;   // optional: t is read through this NTT-domain permutation (rotation without a permuted copy)
  const u32 *eperm;   // optional: the extended digits are read through the same permutation (they were computed once, unrotated,
                      // for all rotations of the ciphertext: hoisted_modup), and `cadd` [2][ell+1][N] is added to the result
  const u64 *cadd;
  int ell, k, N;
};
// ---- inline hoist constants (INL = true; evab_set_hoist_inline): the `cadd` operand of a hoisted rotation is read as the element's
// indicator rows ind [k][N] = NTT_m(I_g) for every prime m (row(m): m for a q row, k - 1 for P) instead of cadd_g, and the constant
// is formed from the key words the inner product loads anyway:
//   cadd_g[c][m] = reduce128(S_c) (.) ind[row(m)],   S_c = sum_{J < ell} (q_J mod m) key[J][c][row(m)]     (128 bits)
// -- hoist_levels_elem's arithmetic (the canonical reduction of the same 128-bit sum, the same mulmod_p), so the same word.  The
// J = row term is zero (q_m mod q_m) and skipped.  The indicator rows do not depend on the tenant: the key-bank offset is never
// applied to them.  q_J mod m by Barrett (barrett64 is exact for any 64-bit input); a sum has at most k - 2 <= 22 products below
// 2^120 (both factors below m < 2^60): below 2^125.
EVAB_HD u64 q_mod(const PrimeDev *primes, int J, const PrimeDev &P) { return barrett64(primes[J].p, P.p, P.ratio64); }
// cadd_g[c][m] for both polynomials at coefficients j, j+1 from the sums S_0 = (s0x, s0y), S_1 = (s1x, s1y)
EVAB_HD void inline_const(const u64 *ind, int row, size_t N, int j, const PrimeDev &P, u64 l0x, u64 h0x, u64 l0y, u64 h0y, u64 l1x, u64 h1x,
                          u64 l1y, u64 h1y, u64x2 &c0, u64x2 &c1) {
  const u64x2 ni = ld2(ind + (size_t)row * N + j);
  c0.x = mulmod_p(reduce128(l0x, h0x, P), ni.x, P); c0.y = mulmod_p(reduce128(l0y, h0y, P), ni.y, P);
  c1.x = mulmod_p(reduce128(l1x, h1x, P), ni.x, P); c1.y = mulmod_p(reduce128(l1y, h1y, P), ni.y, P);
}

// ---- seeded key images (SEED = true; evab_set_key_seeded): the key operand of a key switch points at an image
//   [k-1][k][N] c0 rows, then the key's 32-byte seed padded to 64 bytes      (seeded_key_words)
// and its c1 rows -- the uniform half a, rows J k + m of the rule of key_expand.cuh -- are drawn where the expanded key's words are
// loaded.  The key-bank offset moves the image, seed included.  A thread owns 2 coefficients and a ChaCha block yields 8, so the
// draw is split from the inner product: a block (or the CPU replay) first draws the c1 words of its coefficient tile for every
// J < ell of its row (seeded_c1_draw8 per ChaCha block, SeedTileDev / SeedTileHost), then the unchanged body reads them from that
// tile (tile->c1).  The accepted candidates are reduced by barrett64 (exact for any 64-bit input), the rule's value.
struct KxBarrett {
  PrimeDev P;
  EVAB_HD u64 operator()(u64 v) const { return barrett64(v, P.p, P.ratio64); }
};
EVAB_HD size_t seeded_key_words(int k, size_t N) { return (size_t)(k - 1) * k * N + 8; }
// the c0 row (J, row) of a seeded image
EVAB_HD const u64 *seeded_c0(const u64 *key, int J, int row, int k, size_t N) { return key + ((size_t)J * k + row) * N; }
// coefficients 8 t .. 8 t + 7 of the c1 row (J, row) of the seeded image `key` (modulus P, lim = kx_limit(P.p)) -> dst
EVAB_HD void seeded_c1_draw8(const uint32_t *seed, int J, int row, int k, const PrimeDev &P, u64 lim, u32 t, u64 *dst) {
  u64 v[8];
  kx_draw8(seed, (u64)J * k + row, t, KxBarrett{P}, lim, v);
  // In a shared-memory tile, neighbouring lanes' blocks start 64 bytes apart, so each of these four 16-byte stores meets 4-way bank
  // conflicts.  A lane-rotated store order that avoids them (selects on the lane) was measured slower by 1-3 % on every resident
  // workload (DESIGN §4): the draw's ~1000 ALU instructions per block dominate, the selects cost more than the conflicts
  kx_store8(dst, v);
}
EVAB_HD void seeded_seed(const u64 *key, int k, size_t N, uint32_t (&seed)[8]) {
  const uint32_t *s = reinterpret_cast<const uint32_t *>(key + (size_t)(k - 1) * k * N);
#pragma unroll
  for (int i = 0; i < 8; i++) seed[i] = s[i];
}
// evab_expand_seeded_c1: coefficients 8 t .. 8 t + 7 of c1 row r = J k + m of seeded image i (images seeded_key_words apart) into
// the c1-region geometry -- the row sits where the image's c0 row (J, m) sits, at rows + i seeded_key_words + r N
EVAB_HD void expand_seeded_c1_elem(const u64 *images, u64 *rows, const PrimeDev *primes, int k, size_t N, int i, int r, u32 t) {
  const size_t sw = seeded_key_words(k, N);
  uint32_t seed[8];
  seeded_seed(images + (size_t)i * sw, k, N, seed);
  const PrimeDev &P = primes[r % k];
  seeded_c1_draw8(seed, r / k, r % k, k, P, kx_limit(P.p), t, rows + (size_t)i * sw + (size_t)r * N + 8 * (size_t)t);
}
// expanded keys: no tile (never dereferenced)
struct SeedTileNone {
  EVAB_HD void begin(int, int, const u64 *, int, int, int, int, const PrimeDev &) {}
  EVAB_HD u64x2 c1(int, int) const { return u64x2{0, 0}; }
};
// the key words k0 = key[J][0][row], k1 = key[J][1][row] at coefficients j, j+1 of an expanded key, or of a seeded image and its tile
template <bool SEED, class Tile> EVAB_HD void key_words(const u64 *key, const Tile *tile, int J, int row, int k, size_t N, int j, u64x2 &k0, u64x2 &k1) {
  if (SEED) {
    k0 = ld2(seeded_c0(key, J, row, k, N) + j);
    k1 = tile->c1(J, j);
  } else {
    k0 = ld2(key + (((size_t)J * 2 + 0) * k + row) * N + j);
    k1 = ld2(key + (((size_t)J * 2 + 1) * k + row) * N + j);
  }
}
#if defined(__CUDACC__)
// the tile of one thread block in shared memory: [ell][2 blockDim.x] words, coefficients j0 .. j0 + 2 blockDim.x - 1 of the block's
// row, j0 = j - 2 threadIdx.x.  begin(i, j, ...) is called by every thread of the block with the same key and row (the kernels' tile
// loops are uniform, N a multiple of the tile): a barrier (the previous tile's readers), ell / 4 ChaCha blocks per thread (rounded
// up), a barrier.
// Cached c1 rows (evab_set_key_c1_rows): when the block's instance has a c1 region (`cached`, uniform over the block), its rows
// [k-1][k][N] sit at the image + c1d words, c0's geometry; each thread then copies its own 2 words of every J < ell into the tile
// -- read once from memory, nothing drawn, and no barrier, since no other thread reads them
struct SeedTileDev {
  u64 *s;
  bool cached = false;
  long long c1d = 0;
  EVAB_HD void begin(int, int j, const u64 *key, int ell, int row, int k, int N, const PrimeDev &P) {
#if defined(__CUDA_ARCH__)
    if (cached) {
      const u64 *rows = key + c1d;
      for (int J = 0; J < ell; J++) st2(s + (size_t)J * 2 * blockDim.x + 2 * threadIdx.x, ld2(seeded_c0(rows, J, row, k, N) + j));
      return;
    }
    const int T = 2 * blockDim.x, per = T / 8;
    const u32 t0 = (u32)(j - 2 * (int)threadIdx.x) / 8;
    uint32_t seed[8];
    seeded_seed(key, k, N, seed);
    const u64 lim = kx_limit(P.p);
    __syncthreads();
    for (int b = threadIdx.x; b < ell * per; b += blockDim.x) seeded_c1_draw8(seed, b / per, row, k, P, lim, t0 + b % per, s + (size_t)(b / per) * T + (b % per) * 8);
    __syncthreads();
#endif
  }
  EVAB_HD u64x2 c1(int J, int) const {
#if defined(__CUDA_ARCH__)
    return ld2(s + (size_t)J * 2 * blockDim.x + 2 * threadIdx.x);
#else
    return u64x2{0, 0};
#endif
  }
};
#endif

// off: batch instance offset (words) of t / ext / acc; koff: key offset (words) of the instance's tenant in a key bank
// (evab_set_key_bank), applied to key and (INL = false) cadd; 0 when all instances share the key.  SEED: key is a seeded image, its
// c1 words come from `tile` (seeded_c1_draw8)
template <bool INL = false, bool SEED = false, class Tile = SeedTileNone>
EVAB_HD void ks_inner_elem(const IpArgs &A, int mi, int j, long long off = 0, long long koff = 0, Tile *tile = nullptr) {
  const int row = (mi == A.ell) ? A.k - 1 : mi;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  if (SEED) tile->begin(0, j, A.key + koff, A.ell, row, A.k, A.N, P);
  u64 l0x = 0, h0x = 0, l0y = 0, h0y = 0, l1x = 0, h1x = 0, l1y = 0, h1y = 0;
  u64 s0x = 0, t0x = 0, s0y = 0, t0y = 0, s1x = 0, t1x = 0, s1y = 0, t1y = 0;   // INL: S_0, S_1
  for (int J = 0; J < A.ell; J++) {
    u64x2 v;
    if (row == J) {
      const u64 *tp = A.t + off + (size_t)J * N;
      if (A.tperm) { v.x = EVAB_LDG(tp + EVAB_LDG(A.tperm + j)); v.y = EVAB_LDG(tp + EVAB_LDG(A.tperm + j + 1)); }
      else v = ld2(tp + j);
    } else {
      const u64 *ep = A.ext + off + ((size_t)mi * A.ell + J) * N;
      if (A.eperm) { v.x = EVAB_LDG(ep + EVAB_LDG(A.eperm + j)); v.y = EVAB_LDG(ep + EVAB_LDG(A.eperm + j + 1)); }
      else v = ld2(ep + j);
    }
    u64x2 k0, k1;
    key_words<SEED>(A.key + koff, tile, J, row, A.k, N, j, k0, k1);
    mac128(l0x, h0x, v.x, k0.x); mac128(l0y, h0y, v.y, k0.y);
    mac128(l1x, h1x, v.x, k1.x); mac128(l1y, h1y, v.y, k1.y);
    if (INL && J != row) {
      const u64 qj = q_mod(A.primes, J, P);
      mac128(s0x, t0x, qj, k0.x); mac128(s0y, t0y, qj, k0.y);
      mac128(s1x, t1x, qj, k1.x); mac128(s1y, t1y, qj, k1.y);
    }
  }
  u64x2 r0, r1;
  // ext operands may be lazily reduced (< 16p, see EPI_STORE_LAZY): wide reduction
  r0.x = reduce128(l0x, h0x, P); r0.y = reduce128(l0y, h0y, P);
  r1.x = reduce128(l1x, h1x, P); r1.y = reduce128(l1y, h1y, P);
  if (A.cadd) {
    u64x2 c0, c1;
    if (INL) inline_const(A.cadd, row, N, j, P, s0x, t0x, s0y, t0y, s1x, t1x, s1y, t1y, c0, c1);
    else { c0 = ld2(A.cadd + koff + ((size_t)0 * (A.ell + 1) + mi) * N + j); c1 = ld2(A.cadd + koff + ((size_t)1 * (A.ell + 1) + mi) * N + j); }
    r0.x = addmod(r0.x, c0.x, P.p); r0.y = addmod(r0.y, c0.y, P.p);
    r1.x = addmod(r1.x, c1.x, P.p); r1.y = addmod(r1.y, c1.y, P.p);
  }
  st2(A.acc + off + ((size_t)0 * (A.ell + 1) + mi) * N + j, r0);
  st2(A.acc + off + ((size_t)1 * (A.ell + 1) + mi) * N + j, r1);
}

// The shared extended digits ext[m][J] have no entry for m == q_J (the digit itself is used): rotate_modup_prepare_impl stores
// P * c0 mod q_m there, for the batched rotation kernels below.
EVAB_HD void scale_c0_elem(const u64 *c0, u64 *ext, const PrimeDev *primes, int ell, int k, int N, int mi, int j, long long off = 0) {
  const PrimeDev P = primes[mi];
  const u64 pm = primes[k - 1].p % P.p;
  ext[off + ((size_t)mi * ell + mi) * N + j] = mulmod_p(c0[off + (size_t)mi * N + j], pm, P);
}
// ---- all rotations of one ciphertext in one launch (exact; ops_impl.hpp rotate_modup_many_impl): rotation i's inner product through
// its permutation + cadd_i, and P * perm_i(c0) added to polynomial 0 -- the division by P that follows returns exactly
// perm_i(c0) + the key-switched part, the same residues as adding the permuted c0 afterwards ((x + P c - corr) P^-1 = (x - corr) P^-1 + c).
#define ROTMANY_MAX 16
struct RotManyArgs {
  const u64 *t, *ext;             // source c1 [ell][N], shared extended digits [ell+1][ell][N] (diagonal: P * c0, see scale_c0_elem)
  const u32 *perm[ROTMANY_MAX];
  const u64 *key[ROTMANY_MAX], *cadd[ROTMANY_MAX];
  u64 *acc;                       // [n][2][ell+1][N]
  const PrimeDev *primes;
  int n, ell, k, N;
};
// koff: key offset of the instance's tenant (ks_inner_elem), applied to key[i] and (INL = false) cadd[i]; INL: cadd[i] is the
// element's indicator rows (ks_inner_elem); SEED: key[i] is a seeded image (ks_inner_elem)
template <bool INL = false, bool SEED = false, class Tile = SeedTileNone>
EVAB_HD void rot_many_elem(const RotManyArgs &A, int i, int mi, int j, long long off = 0, long long koff = 0, Tile *tile = nullptr) {
  const int row = (mi == A.ell) ? A.k - 1 : mi;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  if (SEED) tile->begin(i, j, A.key[i] + koff, A.ell, row, A.k, A.N, P);
  const u32 pj0 = EVAB_LDG(A.perm[i] + j), pj1 = EVAB_LDG(A.perm[i] + j + 1);
  u64 l0x = 0, h0x = 0, l0y = 0, h0y = 0, l1x = 0, h1x = 0, l1y = 0, h1y = 0;
  u64 s0x = 0, t0x = 0, s0y = 0, t0y = 0, s1x = 0, t1x = 0, s1y = 0, t1y = 0;   // INL: S_0, S_1
  for (int J = 0; J < A.ell; J++) {
    const u64 *src = (row == J) ? A.t + off + (size_t)J * N : A.ext + off + ((size_t)mi * A.ell + J) * N;
    const u64 vx = EVAB_LDG(src + pj0), vy = EVAB_LDG(src + pj1);
    u64x2 k0, k1;
    key_words<SEED>(A.key[i] + koff, tile, J, row, A.k, N, j, k0, k1);
    mac128(l0x, h0x, vx, k0.x); mac128(l0y, h0y, vy, k0.y);
    mac128(l1x, h1x, vx, k1.x); mac128(l1y, h1y, vy, k1.y);
    if (INL && J != row) {
      const u64 qj = q_mod(A.primes, J, P);
      mac128(s0x, t0x, qj, k0.x); mac128(s0y, t0y, qj, k0.y);
      mac128(s1x, t1x, qj, k1.x); mac128(s1y, t1y, qj, k1.y);
    }
  }
  u64x2 c0, c1;
  if (INL) inline_const(A.cadd[i], row, N, j, P, s0x, t0x, s0y, t0y, s1x, t1x, s1y, t1y, c0, c1);
  else { c0 = ld2(A.cadd[i] + koff + ((size_t)0 * (A.ell + 1) + mi) * N + j); c1 = ld2(A.cadd[i] + koff + ((size_t)1 * (A.ell + 1) + mi) * N + j); }
  u64x2 r0, r1;
  r0.x = addmod(reduce128(l0x, h0x, P), c0.x, P.p); r0.y = addmod(reduce128(l0y, h0y, P), c0.y, P.p);
  r1.x = addmod(reduce128(l1x, h1x, P), c1.x, P.p); r1.y = addmod(reduce128(l1y, h1y, P), c1.y, P.p);
  if (mi < A.ell) {   // + perm_i(P * c0), which rotate_modup_prepare_impl left on the diagonal of ext
    const u64 *c0p = A.ext + off + ((size_t)mi * A.ell + mi) * N;
    r0.x = addmod(r0.x, EVAB_LDG(c0p + pj0), P.p);
    r0.y = addmod(r0.y, EVAB_LDG(c0p + pj1), P.p);
  }
  st2(A.acc + off + (((size_t)i * 2 + 0) * (A.ell + 1) + mi) * N + j, r0);
  st2(A.acc + off + (((size_t)i * 2 + 1) * (A.ell + 1) + mi) * N + j, r1);
}

// ---- shared mod-up of a rotation group (exact): per Galois key and level, the constant
//   cadd[c][m] = NTT_m(I_g) (.) sum_{J < ell} (q_J mod m) * key[J][c][row(m)]          (mod m)
// where I_g is the indicator polynomial of the coefficients the automorphism negates (ops_impl.hpp: hoisted_modup).
struct HoistConstArgs {
  const u64 *ind;     // [ell+1][N]  NTT_m(I_g), row order q_0 .. q_{ell-1}, P
  const u64 *key;     // [k-1][2][k][N]
  u64 *out;           // [2][ell+1][N]
  const PrimeDev *primes;
  int ell, k, N;
};
EVAB_HD void hoist_const_elem(const HoistConstArgs &A, int mi, int j) {
  const int row = (mi == A.ell) ? A.k - 1 : mi;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  const u64x2 ni = ld2(A.ind + (size_t)mi * N + j);
  for (int c = 0; c < 2; c++) {
    u64 lx = 0, hx = 0, ly = 0, hy = 0;
    for (int J = 0; J < A.ell; J++) {
      const u64 qj = A.primes[J].p % P.p;
      const u64x2 kv = ld2(A.key + (((size_t)J * 2 + c) * A.k + row) * N + j);
      mac128(lx, hx, qj, kv.x); mac128(ly, hy, qj, kv.y);
    }
    u64x2 r;
    r.x = mulmod_p(reduce128(lx, hx, P), ni.x, P);
    r.y = mulmod_p(reduce128(ly, hy, P), ni.y, P);
    st2(A.out + ((size_t)c * (A.ell + 1) + mi) * N + j, r);
  }
}
// I_g as residues: row mi, coefficient j = sign bit of the coefficient-domain gather table
EVAB_HD void hoist_indicator_elem(u64 *out, const u32 *ctab, int N, int mi, int j) { out[(size_t)mi * N + j] = EVAB_LDG(ctab + j) & 1u; }

// ---- the same constants for every level ell = 1 .. k-1 of n Galois keys in one pass.  The level-ell constant of prime m is
// NTT_m(I_g) (.) (sum_{J < ell} (q_J mod m) key[J][c][m]) mod m, so all levels share one prefix sum over J: a thread keeps the
// 128-bit running sum of its two coefficients (at most k - 1 <= 23 products below 2^120 each: below 2^125) and, each time J
// reaches ell - 1, reduces it once and writes level ell's row -- only the rows that exist at that level (m < ell, or m = P).
// Every key row is read once.  Reductions are canonical for any 128-bit input, so each row equals hoist_const_elem's.
struct HoistLevelsArgs {
  const u64 *ind;     // [n][k][N]  NTT_m(I_g) for every prime m = 0 .. k-1
  const u64 *key;     // [n][k-1][2][k][N]
  u64 *out;           // [n][ell = 1 .. k-1][2][ell+1][N]
  const PrimeDev *primes;
  int k, N;
};
// words of the constants of one key: sum_{ell=1}^{k-1} 2 (ell + 1) N
EVAB_HD size_t hoist_levels_words(int k, size_t N) { return (size_t)((k + 1) * k - 2) * N; }
EVAB_HD void hoist_levels_elem(const HoistLevelsArgs &A, int g, int m, int j) {
  const int k = A.k;
  const size_t N = A.N;
  const PrimeDev P = A.primes[m];
  const u64x2 ni = ld2(A.ind + ((size_t)g * k + m) * N + j);
  const u64 *key = A.key + (size_t)g * (k - 1) * 2 * k * N + (size_t)m * N + j;
  u64 *out = A.out + (size_t)g * hoist_levels_words(k, N) + j;
  u64 l0x = 0, h0x = 0, l0y = 0, h0y = 0, l1x = 0, h1x = 0, l1y = 0, h1y = 0;
  for (int J = 0; J < k - 1; J++) {
    const u64 qj = A.primes[J].p % P.p;
    const u64x2 k0 = ld2(key + ((size_t)J * 2 + 0) * k * N), k1 = ld2(key + ((size_t)J * 2 + 1) * k * N);
    mac128(l0x, h0x, qj, k0.x); mac128(l0y, h0y, qj, k0.y);
    mac128(l1x, h1x, qj, k1.x); mac128(l1y, h1y, qj, k1.y);
    const int ell = J + 1;   // the sum now covers J < ell
    if (m < ell || m == k - 1) {
      const int mi = m == k - 1 ? ell : m;
      u64x2 r0, r1;
      r0.x = mulmod_p(reduce128(l0x, h0x, P), ni.x, P); r0.y = mulmod_p(reduce128(l0y, h0y, P), ni.y, P);
      r1.x = mulmod_p(reduce128(l1x, h1x, P), ni.x, P); r1.y = mulmod_p(reduce128(l1y, h1y, P), ni.y, P);
      st2(out + (size_t)mi * N, r0);
      st2(out + ((size_t)ell + 1 + mi) * N, r1);
    }
    out += (size_t)2 * (ell + 1) * N;
  }
}

// ---- rotate_wsum (exact): sums of rotations of one ciphertext weighted by scalar plaintexts (ops_impl.hpp rotate_wsum_impl).
// A scalar weight is a constant polynomial: in the NTT domain one number w_r per residue, read at pt[r * N].  With acc_i the
// key-switch accumulator of rotation i and tmp_i = iNTT_P(acc_i's P row) + floor(P/2), every output word is
//   A[o][c][r] = sum_i w_oir acc_i[c][r] + sum_t (P mod q_r) w_otr x_t[c][r]     (folded plain taps: divided by P they give w x_t)
//   D[o][c][r] = sum_i w_oir ((tmp_i[c] mod q_r) - floor(P/2) mod q_r)
// and the forward NTT of D with the division epilogue (A - NTT(D)) P^-1 gives sum_i w_oi rotate(x, g_i) + sum_t w_ot x_t, the
// rounding of every rotation being its own.  A is formed inside the key-switch inner product (rot_wsum_ip_elem): the q rows of
// acc_i are weighted where they are computed and never stored; only the P rows are, for the inverse NTT that tmp_i comes from.
// D follows that transform (rot_wsum_elem).  Products are accumulated in 128 bits and reduced once per output word: tmp_i < P
// enters unreduced, and -floor(P/2) as + (q_r - floor(P/2) mod q_r), the same residue as pro_load's MODRED; every product is
// below 2^121 (primes < 2^60), so the WS_MAX + WS_TAPS products of one output word fit.
#define WS_MAX 16
#define WS_TAPS 16
#define WS_OUT 4
struct WsumIpArgs {
  const u64 *t, *c0, *ext;         // source c1 / c0 [ell][N], shared extended digits [ell+1][ell][N] (the diagonal is not read)
  const u32 *perm[WS_MAX];
  const u64 *key[WS_MAX], *cadd[WS_MAX];
  const u64 *wt[WS_OUT][WS_MAX];   // scalar plaintexts [ell][N] (batch instance offset applies); null: weight 0
  const u64 *tap[WS_TAPS];         // size-2 ciphertexts [2][ell][N] at the output's level (batch instance offset applies)
  const u64 *twt[WS_OUT][WS_TAPS]; // their scalar weights; null: weight 0
  u64 *prow;                       // [n][2][N]        the P rows of the accumulators
  u64 *A;                          // [nout][2][ell][N]
  const PrimeDev *primes;
  int n, ntap, nout, ell, k, N;
};
// coefficients j, j+1 of row mi (q_0 .. q_{ell-1}, P) of both polynomials, every rotation and every output (nout == NOUT).  acc_i is
// rot_many_elem's canonical value: the inner product through perm_i + cadd_i, and on a q row + perm_i(P c0) = (P mod q_m) c0[perm_i(j)],
// read from c0 directly.  A P row is stored; a q row is weighted into A, which then takes the taps.
// koff: key offset of the instance's tenant (ks_inner_elem), applied to key[i] and (INL = false) cadd[i]; INL: cadd[i] is the
// element's indicator rows (ks_inner_elem); SEED: key[i] is a seeded image, and every rotation begins its own tile (ks_inner_elem)
template <int NOUT, bool INL = false, bool SEED = false, class Tile = SeedTileNone>
EVAB_HD void rot_wsum_ip_elem(const WsumIpArgs &A, int mi, int j, long long off = 0, long long koff = 0, Tile *tile = nullptr) {
  const bool qrow = mi < A.ell;
  const int row = qrow ? mi : A.k - 1;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  const u64 pm = qrow ? barrett64(A.primes[A.k - 1].p, P.p, P.ratio64) : 0;   // P mod q_m
  const u64 *c0p = A.c0 + off + (size_t)mi * N;
  u64 al[NOUT][2][2], ah[NOUT][2][2];   // [output][polynomial][coefficient]
#pragma unroll
  for (int o = 0; o < NOUT; o++)
#pragma unroll
    for (int c = 0; c < 2; c++) al[o][c][0] = al[o][c][1] = ah[o][c][0] = ah[o][c][1] = 0;
  u32 pj0 = EVAB_LDG(A.perm[0] + j), pj1 = EVAB_LDG(A.perm[0] + j + 1);
  for (int i = 0; i < A.n; i++) {
    const u32 p0 = pj0, p1 = pj1;
    if (i + 1 < A.n) { pj0 = EVAB_LDG(A.perm[i + 1] + j); pj1 = EVAB_LDG(A.perm[i + 1] + j + 1); }   // the next gather's addresses
    u64 l0x = 0, h0x = 0, l0y = 0, h0y = 0, l1x = 0, h1x = 0, l1y = 0, h1y = 0;
    u64 s0x = 0, t0x = 0, s0y = 0, t0y = 0, s1x = 0, t1x = 0, s1y = 0, t1y = 0;   // INL: S_0, S_1
    if (SEED) tile->begin(i, j, A.key[i] + koff, A.ell, row, A.k, A.N, P);
    for (int J = 0; J < A.ell; J++) {
      const u64 *src = (row == J) ? A.t + off + (size_t)J * N : A.ext + off + ((size_t)mi * A.ell + J) * N;
      const u64 vx = EVAB_LDG(src + p0), vy = EVAB_LDG(src + p1);
      u64x2 k0, k1;
      key_words<SEED>(A.key[i] + koff, tile, J, row, A.k, N, j, k0, k1);
      mac128(l0x, h0x, vx, k0.x); mac128(l0y, h0y, vy, k0.y);
      mac128(l1x, h1x, vx, k1.x); mac128(l1y, h1y, vy, k1.y);
      if (INL && J != row) {
        const u64 qj = q_mod(A.primes, J, P);
        mac128(s0x, t0x, qj, k0.x); mac128(s0y, t0y, qj, k0.y);
        mac128(s1x, t1x, qj, k1.x); mac128(s1y, t1y, qj, k1.y);
      }
    }
    u64x2 c0, c1;
    if (INL) inline_const(A.cadd[i], row, N, j, P, s0x, t0x, s0y, t0y, s1x, t1x, s1y, t1y, c0, c1);
    else { c0 = ld2(A.cadd[i] + koff + ((size_t)0 * (A.ell + 1) + mi) * N + j); c1 = ld2(A.cadd[i] + koff + ((size_t)1 * (A.ell + 1) + mi) * N + j); }
    u64x2 r0, r1;
    r0.x = addmod(reduce128(l0x, h0x, P), c0.x, P.p); r0.y = addmod(reduce128(l0y, h0y, P), c0.y, P.p);
    r1.x = addmod(reduce128(l1x, h1x, P), c1.x, P.p); r1.y = addmod(reduce128(l1y, h1y, P), c1.y, P.p);
    if (!qrow) {
      st2(A.prow + off + ((size_t)i * 2 + 0) * N + j, r0);
      st2(A.prow + off + ((size_t)i * 2 + 1) * N + j, r1);
      continue;
    }
    r0.x = addmod(r0.x, mulmod_p(EVAB_LDG(c0p + p0), pm, P), P.p);
    r0.y = addmod(r0.y, mulmod_p(EVAB_LDG(c0p + p1), pm, P), P.p);
#pragma unroll
    for (int o = 0; o < NOUT; o++) {
      if (!A.wt[o][i]) continue;
      const u64 w = EVAB_LDG(A.wt[o][i] + off + (size_t)mi * N);
      mac128(al[o][0][0], ah[o][0][0], r0.x, w); mac128(al[o][0][1], ah[o][0][1], r0.y, w);
      mac128(al[o][1][0], ah[o][1][0], r1.x, w); mac128(al[o][1][1], ah[o][1][1], r1.y, w);
    }
  }
  if (!qrow) return;
  for (int t = 0; t < A.ntap; t++) {
    const u64x2 x0 = ld2(A.tap[t] + off + (size_t)mi * N + j), x1 = ld2(A.tap[t] + off + ((size_t)A.ell + mi) * N + j);
#pragma unroll
    for (int o = 0; o < NOUT; o++) {
      if (!A.twt[o][t]) continue;
      const u64 w = mulmod_p(pm, EVAB_LDG(A.twt[o][t] + off + (size_t)mi * N), P);
      mac128(al[o][0][0], ah[o][0][0], x0.x, w); mac128(al[o][0][1], ah[o][0][1], x0.y, w);
      mac128(al[o][1][0], ah[o][1][0], x1.x, w); mac128(al[o][1][1], ah[o][1][1], x1.y, w);
    }
  }
#pragma unroll
  for (int o = 0; o < NOUT; o++)
#pragma unroll
    for (int c = 0; c < 2; c++) {
      u64x2 v;
      v.x = reduce128(al[o][c][0], ah[o][c][0], P); v.y = reduce128(al[o][c][1], ah[o][c][1], P);
      st2(A.A + off + (((size_t)o * 2 + c) * A.ell + mi) * N + j, v);
    }
}

struct WsumArgs {
  const u64 *tmp;                  // [n][2][N]        (inverse NTT of the P rows, + floor(P/2))
  const u64 *wt[WS_OUT][WS_MAX];   // scalar plaintexts [ell][N] (batch instance offset applies); null: weight 0
  u64 *D;                          // [nout][2][ell][N]
  const PrimeDev *primes;
  const u64 *halfmod;              // [k]: floor(P/2) mod q_r
  int n, nout, ell, k, N;
};
// D: coefficients j, j+1 of residue r of polynomial c of every output
EVAB_HD void rot_wsum_elem(const WsumArgs &A, int c, int r, int j, long long off = 0) {
  const PrimeDev P = A.primes[r];
  const size_t N = A.N;
  const u64 nh = P.p - A.halfmod[r];
  u64 dl[WS_OUT][2], dh[WS_OUT][2];
#pragma unroll
  for (int o = 0; o < WS_OUT; o++) dl[o][0] = dl[o][1] = dh[o][0] = dh[o][1] = 0;
  for (int i = 0; i < A.n; i++) {
    u64x2 t = ld2(A.tmp + off + ((size_t)i * 2 + c) * N + j);
    t.x += nh; t.y += nh;
#pragma unroll
    for (int o = 0; o < WS_OUT; o++) {
      if (o >= A.nout || !A.wt[o][i]) continue;
      const u64 w = EVAB_LDG(A.wt[o][i] + off + (size_t)r * N);
      mac128(dl[o][0], dh[o][0], t.x, w); mac128(dl[o][1], dh[o][1], t.y, w);
    }
  }
#pragma unroll
  for (int o = 0; o < WS_OUT; o++) {
    if (o >= A.nout) break;
    u64x2 v;
    v.x = reduce128(dl[o][0], dh[o][0], P); v.y = reduce128(dl[o][1], dh[o][1], P);
    st2(A.D + off + (((size_t)o * 2 + c) * A.ell + r) * N + j, v);
  }
}

// ---- lazy_rotsum (OPT-IN, NOT bit-exact: SURVEY 8f-4) ------------------------------------------------------------------
// sum_i w_i (.) rotate(x, g_i) for several rotations of ONE ciphertext with plaintext weights, with a single mod-down for the
// whole sum: T[c][m] = sum_i w_i[m] (.) acc_i[c][m] over the extended basis (q_0 .. q_{ell-1}, P), acc_i the key-switch
// accumulator of rotation i (shared extended digits through the permutation + cadd, as in ks_inner_elem).  The reference
// rounds every rotation's accumulator down by P and multiplies afterwards; rounding the weighted sum once differs from that in
// the last bits (and carries less rounding noise) -- results are graded by the reference's MSE criterion only.
#define LRS_MAX 16
#define LRS_OUT 4
struct LazyRotSumArgs {
  const u64 *t, *ext;             // source c1 [ell][N], shared extended digits [ell+1][ell][N] (diagonal: P * c0, see scale_c0_elem)
  const u32 *perm[LRS_MAX];
  const u64 *key[LRS_MAX], *cadd[LRS_MAX];
  const u64 *wt[LRS_OUT][LRS_MAX]; // plaintext weights [ell+1][N], last row mod P (batch instance offset applies); null: rotation not in that sum
  u64 *acc;                       // [nout][2][ell+1][N]; poly 0 already carries P * sum_i w_i (.) perm_i(c0) (which the division by P gives back)
  const PrimeDev *primes;
  int n, nout, ell, k, N;
};
// One rotation's share at elements (j, j+1) of row mi, for every output sum it takes part in.  The key-switch inner product of
// the rotation is computed once and weighted per output; every value is reduced below p, so that up to LRS_MAX of them add up
// inside 64 bits.  part[o] = { w.(ip0+cadd0) + P.w.perm(c0), w.(ip1+cadd1) } for x and y.
// koff: key offset of the instance's tenant (ks_inner_elem), applied to key[i] and cadd[i]
EVAB_HD void lazy_rotsum_part(const LazyRotSumArgs &A, int mi, int j, int i, long long off, u64 part[LRS_OUT][4], long long koff = 0) {
  const int row = (mi == A.ell) ? A.k - 1 : mi;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  const u32 pj0 = EVAB_LDG(A.perm[i] + j), pj1 = EVAB_LDG(A.perm[i] + j + 1);
  u64 l0x = 0, h0x = 0, l0y = 0, h0y = 0, l1x = 0, h1x = 0, l1y = 0, h1y = 0;
#pragma unroll 4
  for (int J = 0; J < A.ell; J++) {
    const u64 *src = (row == J) ? A.t + off + (size_t)J * N : A.ext + off + ((size_t)mi * A.ell + J) * N;
    const u64 vx = EVAB_LDG(src + pj0), vy = EVAB_LDG(src + pj1);
    const u64x2 k0 = ld2(A.key[i] + koff + (((size_t)J * 2 + 0) * A.k + row) * N + j);
    const u64x2 k1 = ld2(A.key[i] + koff + (((size_t)J * 2 + 1) * A.k + row) * N + j);
    mac128(l0x, h0x, vx, k0.x); mac128(l0y, h0y, vy, k0.y);
    mac128(l1x, h1x, vx, k1.x); mac128(l1y, h1y, vy, k1.y);
  }
  const u64x2 c0 = ld2(A.cadd[i] + koff + ((size_t)0 * (A.ell + 1) + mi) * N + j), c1 = ld2(A.cadd[i] + koff + ((size_t)1 * (A.ell + 1) + mi) * N + j);
  u64 a0x = addmod(reduce128(l0x, h0x, P), c0.x, P.p), a0y = addmod(reduce128(l0y, h0y, P), c0.y, P.p);
  const u64 a1x = addmod(reduce128(l1x, h1x, P), c1.x, P.p), a1y = addmod(reduce128(l1y, h1y, P), c1.y, P.p);
  if (mi < A.ell) {   // + perm(P * c0) (the diagonal of ext): comes back as perm(c0) from the division by P
    const u64 *c0p = A.ext + off + ((size_t)mi * A.ell + mi) * N;
    a0x = addmod(a0x, EVAB_LDG(c0p + pj0), P.p);
    a0y = addmod(a0y, EVAB_LDG(c0p + pj1), P.p);
  }
#pragma unroll
  for (int o = 0; o < LRS_OUT; o++) {
    if (o >= A.nout || !A.wt[o][i]) { part[o][0] = part[o][1] = part[o][2] = part[o][3] = 0; continue; }
    const u64x2 w = ld2(A.wt[o][i] + off + (size_t)mi * N + j);
    part[o][0] = mulmod_p(a0x, w.x, P); part[o][1] = mulmod_p(a0y, w.y, P);
    part[o][2] = mulmod_p(a1x, w.x, P); part[o][3] = mulmod_p(a1y, w.y, P);
  }
}
// sum[4]: the parts of all rotations of output o added up as plain integers (< LRS_MAX * p < 2^64)
EVAB_HD void lazy_rotsum_store(const LazyRotSumArgs &A, int mi, int j, int o, long long off, const u64 sum[4]) {
  const int row = (mi == A.ell) ? A.k - 1 : mi;
  const PrimeDev P = A.primes[row];
  const size_t N = A.N;
  u64x2 r0, r1;
  r0.x = reduce128(sum[0], 0, P); r0.y = reduce128(sum[1], 0, P);
  r1.x = reduce128(sum[2], 0, P); r1.y = reduce128(sum[3], 0, P);
  st2(A.acc + off + (((size_t)o * 2 + 0) * (A.ell + 1) + mi) * N + j, r0);
  st2(A.acc + off + (((size_t)o * 2 + 1) * (A.ell + 1) + mi) * N + j, r1);
}
