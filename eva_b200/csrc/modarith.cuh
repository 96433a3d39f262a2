// modarith.cuh -- 64-bit modular arithmetic for RNS residues (primes < 2^60).
//
// All routines are __host__ __device__ so that the kernel phases built on top
// of them can be replayed on the CPU by tests/emu (index/bounds validation in
// a container without a GPU).  On the device everything lowers to 32-bit
// IMAD/IMAD.WIDE + IADD3 chains: the GPU has no native 64x64 multiplier.
#pragma once
#include <stdint.h>

typedef uint64_t u64;
typedef uint32_t u32;

#if defined(__CUDACC__)
#define EVAB_HD __host__ __device__ __forceinline__
#else
#define EVAB_HD inline
#endif

#if !defined(__CUDACC__) && !defined(__align__)
#define __align__(n) __attribute__((aligned(n)))
#endif
struct __align__(16) u64x2 { u64 x, y; };

EVAB_HD u64 mulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

// Per-prime constants resident in device memory (one entry per key-level prime)
struct PrimeDev {
  u64 p;
  u64 ratio_lo, ratio_hi;  // floor(2^128 / p)   (Barrett, 128-bit inputs)
  u64 ratio64;             // floor(2^64 / p)    (Barrett, 64-bit inputs)
  u64 ninv, ninv_s;        // N^-1 mod p and its Shoup companion
  u64 itw1n, itw1n_s;      // itw[1] * N^-1 mod p (+Shoup): twiddle of the last inverse stage with the scaling folded in
  const u64x2 *tw;         // forward twiddles  {psi^bitrev(i), shoup}   [N]
  const u64x2 *itw;        // inverse twiddles  {psi^-bitrev(i), shoup}  [N]
  // fold-friendly primes (prime_foldable): the same tables with the companion row {w, w * 2^32 mod p}
  const u64x2 *ftw, *fitw;
  u64 ninv_v, itw1n_v;     // companion rows of ninv / itw1n
  u32 eps;                 // 2^61 mod p
  u32 foldable;
};

// per-prime constants of the fold arithmetic, carried in the kernel parameters (constant bank -> uniform registers)
struct FoldPrime {
  u64 p, p3, p8;             // p, 3p, 8p
  u32 eps, foldable;         // 2^61 mod p
  const u64x2 *ftw, *fitw;   // {w, w * 2^32 mod p} forward / inverse, bit-reversed power order
  u64 ninv, ninv_v, itw1n, itw1n_v;
};
constexpr int NTT_MAX_PRIMES = 24;
// entries per prime of the encoder's table 2^i mod p (host_tables.hpp, encode_kernels.cuh enc_residue): a finite double
// c >= 2^64 is mant * 2^sh with sh = exponent - 64 <= 1024 - 64 = 960, so every shift has its row entry
constexpr int ENC_POW2_ROW = 1024;

// x >= c ? x - c : x
EVAB_HD u64 csub(u64 x, u64 c) {
#if defined(__CUDA_ARCH__)
  // x - c with the borrow selecting the result: ptxas keeps the borrow in the carry-out predicate of IADD3.X and selects on it
  // (IADD3, IADD3.X, SEL, SEL) instead of comparing first (two ISETP more)
  u32 lo, hi, b;
  asm("sub.cc.u32 %0, %3, %5;\n\tsubc.cc.u32 %1, %4, %6;\n\tsubc.u32 %2, 0, 0;"
      : "=r"(lo), "=r"(hi), "=r"(b) : "r"((u32)x), "r"((u32)(x >> 32)), "r"((u32)c), "r"((u32)(c >> 32)));
  return b ? x : (((u64)hi << 32) | lo);
#else
  return x >= c ? x - c : x;
#endif
}

// Shoup multiplication by a constant w (ws = floor(w*2^64/p)); any u64 y.
// Result is congruent to w*y mod p and lies in [0, 2p).
EVAB_HD u64 shoup_lazy(u64 y, u64 w, u64 ws, u64 p) {
  u64 q = mulhi64(ws, y);
  return w * y - q * p;
}
EVAB_HD u64 shoup_mul(u64 y, u64 w, u64 ws, u64 p) { return csub(shoup_lazy(y, w, ws, p), p); }
// same with the caller supplying np = 2^64 - p: w*y + q*np (mod 2^64) saves the
// negation of q in the multiply-accumulate chain
EVAB_HD u64 shoup_lazy_n(u64 y, u64 w, u64 ws, u64 np) {
  u64 q = mulhi64(ws, y);
  return w * y + q * np;
}

// ---- hand-scheduled lazy Shoup product for the NTT butterflies --------------------------------
// The GPU has no 64x64 multiplier; IMAD.WIDE.U32 / IMAD.HI.U32 occupy the fma pipe and that pipe
// bounds the transforms.  The quotient estimate therefore uses THREE partial products:
// q~ = a1*b1 + hi32(a1*b0) + hi32(a0*b1) drops a0*b0 and the low halves of the cross terms, so
// q - 2 <= q~ <= q = floor(ws*y / 2^64), and  w*y - q~*p  is congruent to w*y and lies in [0, 4p)
// for ANY u64 y (primes < 2^60 leave room for 16p).  shoup_mad4 returns  c + w*y + q~*np  (mod 2^64,
// np = 2^64 - p) with the addend c riding in the multiply-add chain: 3 wide + 2 high + 4 low
// multiplies and one 64-bit add.  Host and device evaluate the same integers.
EVAB_HD u64 shoup_mad4(u64 y, u64 w, u64 ws, u64 np, u64 c) {
  const u32 y0 = (u32)y, y1 = (u32)(y >> 32), w0 = (u32)w, w1 = (u32)(w >> 32);
  const u32 s0 = (u32)ws, s1 = (u32)(ws >> 32), n0 = (u32)np, n1 = (u32)(np >> 32);
#if defined(__CUDA_ARCH__)
  u32 c0, c1; u64 q, m;
  asm("mul.hi.u32 %0, %1, %2;" : "=r"(c0) : "r"(s1), "r"(y0));
  asm("mul.hi.u32 %0, %1, %2;" : "=r"(c1) : "r"(s0), "r"(y1));
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(q) : "r"(s1), "r"(y1), "l"((u64)c0));
  q += c1;
  const u32 q0 = (u32)q, q1 = (u32)(q >> 32);
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(m) : "r"(w0), "r"(y0), "l"(c));
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(m) : "r"(q0), "r"(n0), "l"(m));
  u32 h = (u32)(m >> 32);
  asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(h) : "r"(w0), "r"(y1));
  asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(h) : "r"(w1), "r"(y0));
  asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(h) : "r"(q0), "r"(n1));
  asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(h) : "r"(q1), "r"(n0));
  return ((u64)h << 32) | (u32)m;
#else
  const u64 q = (u64)s1 * y1 + (((u64)s1 * y0) >> 32) + (((u64)s0 * y1) >> 32);
  return c + w * y + q * np;
#endif
}

// ---- "two-row fold" multiplication for SEAL's 60-bit NTT primes -------------------------------
// CoeffModulus::Create scans downwards from 2^60 in steps of 2N, so every 60-bit prime of an EVA
// program has the form p = 2^60 - delta with delta < 2^25 ("fold-friendly": prime_foldable()).  For
// those, 2^61 = 2p + eps with eps = 2*delta < 2^26, and a product by a known constant w needs no
// quotient at all: with the companion row v = w * 2^32 mod p stored beside w,
//     S = y0*w + y1*v          (y = y1*2^32 + y0, ANY u64;  S == y*w mod p,  S < 2^33 p < 2^93)
//     r = (S mod 2^61) + (S >> 61) * eps                      (r == y*w mod p,  r < 2^61 + 2^58 < 2.2501 p)
// which is 4 + 1 IMAD.WIDE.U32 and no 32-bit low multiplies -- against 6 wide + 4 low for the lazy
// Shoup product (the fma pipe bounds the transforms).  The inputs of a
// product are unconstrained, so butterflies only ever have to keep their *sums* below 2^64.
// Bounds are tracked at compile time in units of p/16 (B16: value < B16 * p / 16; 16p < 2^64).
constexpr int FB_CANON = 16;    // [0, p)
constexpr int FB_MUL = 37;      // fold_mul result   (< 2.2501 p)
constexpr int FB_FOLD = 33;     // fold61 result     (< 2^61 + 7 * 2^26 < 2.0001 p)
constexpr int FB_MAX = 256;     // 16 p < 2^64
EVAB_HD bool prime_foldable(u64 p) { return p < (1ull << 60) && p > (1ull << 60) - (1ull << 25); }
EVAB_HD u32 fold_eps(u64 p) { return (u32)(((1ull << 60) - p) << 1); }   // 2^61 mod p

EVAB_HD u64 madw32(u32 a, u32 b, u64 c) {
#if defined(__CUDA_ARCH__)
  u64 d; asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c)); return d;
#else
  return (u64)a * b + c;
#endif
}
// a * b + (ch:cl), the addend given as its two 32-bit halves, as a carry-chained mad.lo.cc / madc.hi pair.  Written as
// mad.wide.u32 with an addend that is not itself a wide product, ptxas emits IMAD.WIDE + IADD3 + IMAD.X; from this form it
// emits one IMAD.WIDE with the halves as a register-pair addend (fold_mul, fold61, fold_canon: 8-11 % fewer instructions
// in the N = 16384 transforms, tools/ntt_sass_report.py).
EVAB_HD u64 madc32(u32 a, u32 b, u32 cl, u32 ch) {
#if defined(__CUDA_ARCH__)
  u32 rl, rh; u64 r;
  asm("mad.lo.cc.u32 %0, %2, %3, %4;\n\tmadc.hi.u32 %1, %2, %3, %5;" : "=r"(rl), "=r"(rh) : "r"(a), "r"(b), "r"(cl), "r"(ch));
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(rl), "r"(rh));
  return r;
#else
  return (u64)a * b + (((u64)ch << 32) | cl);
#endif
}
// any u64 -> congruent value < 2^61 + 7*eps
EVAB_HD u64 fold61(u64 x, u32 eps) { return madc32((u32)(x >> 61), eps, (u32)x, (u32)(x >> 32) & 0x1fffffffu); }
// x < 16p -> canonical [0,p): x = h*2^60 + l == l + h*delta, which is < p + 2^29; one conditional subtraction
EVAB_HD u64 fold_canon(u64 x, u32 eps, u64 p) {
  return csub(madc32((u32)(x >> 60), eps >> 1, (u32)x, (u32)(x >> 32) & 0x0fffffffu), p);
}
EVAB_HD u64 fold_mul(u64 y, u64 w, u64 v, u32 eps) {
  const u32 y0 = (u32)y, y1 = (u32)(y >> 32);
#if defined(__CUDA_ARCH__)
  // One asm statement per multiply: ptxas then keeps the accumulating forms (IMAD.WIDE with a 64-bit addend,
  // IMAD.WIDE with carry-out) instead of splitting them into multiply + add pairs.
  u64 B, A;
  asm("mul.wide.u32 %0, %1, %2;" : "=l"(B) : "r"(y0), "r"((u32)(w >> 32)));
  asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(B) : "r"(y1), "r"((u32)(v >> 32)));
  asm("mul.wide.u32 %0, %1, %2;" : "=l"(A) : "r"(y0), "r"((u32)w));
  const u64 A2 = madw32(y1, (u32)v, 0);
  u32 s0, s1, s2, H;
  asm("{\n\t.reg .u32 t;\n\t"
      "add.cc.u32 %0, %3, %5;\n\taddc.cc.u32 t, %4, %6;\n\taddc.u32 %2, %8, 0;\n\t"
      "add.cc.u32 %1, t, %7;\n\taddc.u32 %2, %2, 0;\n\t}"
      : "=r"(s0), "=r"(s1), "=r"(s2)
      : "r"((u32)A), "r"((u32)(A >> 32)), "r"((u32)A2), "r"((u32)(A2 >> 32)), "r"((u32)B), "r"((u32)(B >> 32)));
  asm("shf.l.wrap.b32 %0, %1, %2, 3;" : "=r"(H) : "r"(s1), "r"(s2));
  return madc32(H, eps, s0, s1 & 0x1fffffffu);   // (S mod 2^61) + (S >> 61) * eps
#else
  const unsigned __int128 S = (unsigned __int128)y0 * w + (unsigned __int128)y1 * v;
  return (u64)(S & ((1ull << 61) - 1)) + (u64)(S >> 61) * eps;
#endif
}

// canonical add / sub / neg for operands already in [0,p)
EVAB_HD u64 addmod(u64 a, u64 b, u64 p) { return csub(a + b, p); }
EVAB_HD u64 submod(u64 a, u64 b, u64 p) { return a >= b ? a - b : a + p - b; }
EVAB_HD u64 negmod(u64 a, u64 p) { return a ? p - a : 0; }

// Barrett reduction of a 64-bit value to [0,p)
EVAB_HD u64 barrett64(u64 x, u64 p, u64 ratio64) {
  u64 q = mulhi64(x, ratio64);
  return csub(x - q * p, p);
}

// Barrett reduction of a 128-bit value (hi:lo) to [0,p); valid for
// hi:lo < 2^128 and p < 2^61 (one conditional subtraction suffices).
EVAB_HD u64 barrett128(u64 lo, u64 hi, u64 p, u64 rlo, u64 rhi) {
  u64 carry = mulhi64(lo, rlo);
  u64 t0 = lo * rhi, t1 = mulhi64(lo, rhi);
  u64 tmp1 = t0 + carry;
  u64 tmp3 = t1 + (tmp1 < carry);
  u64 u0 = hi * rlo, u1 = mulhi64(hi, rlo);
  u64 tmp1b = tmp1 + u0;
  carry = u1 + (tmp1b < tmp1);
  u64 q = hi * rhi + tmp3 + carry;
  return csub(lo - q * p, p);
}

// same for any 128-bit input (e.g. sums of products of lazily reduced operands): the
// quotient estimate is short by at most 3, two conditional subtractions finish
EVAB_HD u64 barrett128_wide(u64 lo, u64 hi, u64 p, u64 rlo, u64 rhi) {
  u64 carry = mulhi64(lo, rlo);
  u64 t0 = lo * rhi, t1 = mulhi64(lo, rhi);
  u64 tmp1 = t0 + carry;
  u64 tmp3 = t1 + (tmp1 < carry);
  u64 u0 = hi * rlo, u1 = mulhi64(hi, rlo);
  u64 tmp1b = tmp1 + u0;
  carry = u1 + (tmp1b < tmp1);
  u64 q = hi * rhi + tmp3 + carry;
  return csub(csub(lo - q * p, 2 * p), p);
}

// canonical product of two values in [0,p)
EVAB_HD u64 mulmod(u64 a, u64 b, u64 p, u64 rlo, u64 rhi) {
  return barrett128(a * b, mulhi64(a, b), p, rlo, rhi);
}

// 128-bit accumulate acc += a*b
EVAB_HD void mac128(u64 &lo, u64 &hi, u64 a, u64 b) {
  u64 pl = a * b, ph = mulhi64(a, b);
  lo += pl;
  hi += ph + (lo < pl);
}

// any 128-bit value (hi:lo) -> canonical [0,p) for a fold-friendly prime: 2^64 == 8 eps (mod p), so
//   y  = lo + hi * 8eps            (94 bits: three wide multiplies' worth of work instead of a 128-bit Barrett
//   y' = y_lo64 + y_hi30 * 8eps     quotient -- 5 IMAD.WIDE against ~20 multiply instructions)
//   r  = (y' mod 2^61) + (y' >> 61) * eps,   then fold_canon.
EVAB_HD u64 fold_reduce128(u64 lo, u64 hi, u32 eps, u64 p) {
  const u32 e64 = eps << 3;
  const u64 m0 = madw32((u32)hi, e64, 0), m1 = madw32((u32)(hi >> 32), e64, 0);   // hi * 8eps = m0 + m1 * 2^32
  const u64 s = lo + m0;
  const u64 t = s + (m1 << 32);
  const u64 yh = (m1 >> 32) + (u64)(s < lo) + (u64)(t < s);                       // < 2^30
  const u64 v = t + madw32((u32)yh, e64, 0);
  const u32 c2 = (u32)(v < t);
  const u64 r = madw32((u32)(v >> 61) + 8u * c2, eps, v & ((1ull << 61) - 1));  // < 2^61 + 2^30
  return fold_canon(r, eps, p);
}
// reductions used by the element-wise kernels: fold arithmetic when the prime allows it, Barrett otherwise
EVAB_HD u64 reduce128(u64 lo, u64 hi, const PrimeDev &P) {
  return P.foldable ? fold_reduce128(lo, hi, P.eps, P.p) : barrett128_wide(lo, hi, P.p, P.ratio_lo, P.ratio_hi);
}
EVAB_HD u64 mulmod_p(u64 a, u64 b, const PrimeDev &P) { return reduce128(a * b, mulhi64(a, b), P); }

