// ntt_core.cuh -- register-resident negacyclic NTT / iNTT over one RNS residue.
//
// T = N/16 threads transform one residue polynomial (N = 2^n, 10 <= n <= 15), as one
// CTA or spread over a thread-block cluster of 2/4/8 CTAs (see SmemView below; n = 15
// needs a cluster: 2048 threads).  Every thread keeps E = 16 coefficients in registers
// for the whole transform (64 registers/thread: the register file of one SM holds one
// N = 16384 residue) -- the residue never lives in shared memory, which is only the
// exchange medium between P = ceil(n/4) register passes:
//
//   pass j < P-1   stages 4j..4j+3   thread owns idx = (H << (lb+4)) | (k << lb) | L,
//                                    lb = n - 4(j+1), tid = (H << lb) | L        (strided)
//   pass P-1       last r stages     thread owns idx = (tid << 4) | k            (contiguous)
//
// Forward = Cooley-Tukey (natural in, bit-reversed out), inverse =
// Gentleman-Sande; semantics match seal::util::ntt_negacyclic_harvey /
// inverse_ntt_negacyclic_harvey as called below reference
// eva/seal/seal_executor.h:162-213,242 (SURVEY.md Appendix A.3): out[i] =
// a(psi^(2*bitrev(i)+1)), canonical in [0,p).
//
// Butterflies are lazy: primes are < 2^60, so a u64 holds values up to 16p.
// shoup_lazy_n() accepts any u64 and returns [0,2p) (shoup_mad4, used by the inverse: [0,4p)); only the "X" input of a
// butterfly ever needs a conditional subtraction, and the unrolled code tracks
// a compile-time bound (in units of p) to place those subtractions sparsely.
//
// All phases are __host__ __device__: tests replay them on the CPU (threads
// serialised, shared memory as a plain array) to validate indexing, swizzles
// and bounds without a GPU.
#pragma once
#include "modarith.cuh"

#if defined(__CUDA_ARCH__)
#define EVAB_LDG(p) __ldg(p)
#else
#define EVAB_LDG(p) (*(p))
#endif

EVAB_HD u64x2 ldg_tw(const u64x2 *p) {
#if defined(__CUDA_ARCH__)
  ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(p));
  u64x2 r; r.x = v.x; r.y = v.y; return r;
#else
  return *p;
#endif
}

constexpr int NTT_EL = 4;            // log2(coefficients per thread)
constexpr int NTT_E = 1 << NTT_EL;   // coefficients per thread

template <int LOGN> struct NttGeom {
  static_assert(LOGN >= 10 && LOGN <= 15, "register NTT core supports 2^10..2^15 (2^15 only across a cluster: 2048 threads)");
  static constexpr int N = 1 << LOGN;
  static constexpr int T = N / NTT_E;                          // threads per residue
  static constexpr int P = (LOGN + NTT_EL - 1) / NTT_EL;       // register passes
  static constexpr int R = LOGN - NTT_EL * (P - 1);            // stages of the last pass (1..4)
  static constexpr int NPH = 2 * (P - 1);                      // barrier-separated phases before the epilogue
#if defined(__CUDACC__)
  __host__ __device__
#endif
  static constexpr int lowbits(int j) { return LOGN - NTT_EL * (j + 1); }
};

// ---------------------------------------------------------------------------
// thread <-> coefficient index maps
// ---------------------------------------------------------------------------
template <int LOGN, int J> EVAB_HD u32 idx_s(u32 tid, u32 k) {  // strided pass J < P-1
  constexpr int lb = NttGeom<LOGN>::lowbits(J);
  const u32 H = tid >> lb, L = tid & ((1u << lb) - 1u);
  return (H << (lb + NTT_EL)) | (k << lb) | L;
}
EVAB_HD u32 idx_c(u32 tid, u32 k) { return (tid << NTT_EL) | k; }  // contiguous last pass

// ---------------------------------------------------------------------------
// shared-memory exchange layouts (element = 8 bytes, 32 banks x 4 bytes)
// ---------------------------------------------------------------------------
// exchange INTO strided pass JR (from pass JR-1, or back in the inverse): linear,
// with the reader's low H bits XORed into the index bits just above its L field
// when L carries fewer than 4 bits, so a half-warp of 64-bit readers covers 16
// distinct bank pairs.  The XOR source bits are part of the writer's per-
// instruction constant k, so the writer stays conflict-free as well.
template <int LOGN, int JR> EVAB_HD u32 swz_s(u32 idx) {
  constexpr int lowR = NttGeom<LOGN>::lowbits(JR);
  if (lowR >= 4) return idx;
  constexpr u32 mask = (16u >> lowR) - 1u;
  return idx ^ (((idx >> (lowR + NTT_EL)) & mask) << lowR);
}
// exchange between pass P-2 and the contiguous last pass: 128-byte rows (one per
// last-pass thread), 16-byte chunks XOR-swizzled by the row so that the 128-bit
// row accesses of 8 consecutive threads and the 64-bit strided accesses of a
// pass-(P-2) half-warp both touch every bank once.
template <int LOGN> EVAB_HD u32 swz_rowf(u32 row) {
  constexpr int R = NttGeom<LOGN>::R;
  u32 f = row & 7u;
  if (R < 4) f ^= ((row >> 3) & 1u) << (R - 1);
  return f;
}
template <int LOGN> EVAB_HD u32 swz_c(u32 idx) {
  const u32 row = idx >> NTT_EL, e = idx & 15u;
  return (row << NTT_EL) | ((((e >> 1) ^ swz_rowf<LOGN>(row)) << 1) | (e & 1u));
}

// Every exchange layout above is GF(2)-linear in the bits of (thread, k) -- shifts, masks and XORs of
// disjoint fields -- so addr(v, k) = addr(v, 0) ^ addr(0, k): one thread-dependent base and a compile-time
// constant per register, i.e. ONE logic instruction per access (none when the two parts share no bit and
// the constant becomes the immediate offset of the access) instead of re-deriving the swizzle per element.
// A::at(v, k) = element index inside the CTA's slice; A::disjoint = the k part never overlaps the thread part.
EVAB_HD u64 *xelem(u64 *sm, u32 byte_off) { return reinterpret_cast<u64 *>(reinterpret_cast<char *>(sm) + byte_off); }
EVAB_HD const u64 *xelem(const u64 *sm, u32 byte_off) { return reinterpret_cast<const u64 *>(reinterpret_cast<const char *>(sm) + byte_off); }
template <class A> EVAB_HD void lin_write(const u64 (&x)[NTT_E], u64 *sm, u32 v) {
  const u32 b0 = A::at(v, 0) << 3;
#pragma unroll
  for (int k = 0; k < NTT_E; k++) {
    const u32 ck = A::at(0, (u32)k) << 3;
    *xelem(sm, A::disjoint ? b0 + ck : b0 ^ ck) = x[k];
  }
}
template <class A> EVAB_HD void lin_read(u64 (&x)[NTT_E], const u64 *sm, u32 v) {
  const u32 b0 = A::at(v, 0) << 3;
#pragma unroll
  for (int k = 0; k < NTT_E; k++) {
    const u32 ck = A::at(0, (u32)k) << 3;
    x[k] = *xelem(sm, A::disjoint ? b0 + ck : b0 ^ ck);
  }
}
// strided pass J <-> layout of strided pass JR; MASK = slice mask of a cluster-distributed residue (or ~0)
template <int LOGN, int J, int JR, u32 MASK> struct AddrS {
  static constexpr bool disjoint = NttGeom<LOGN>::lowbits(JR) >= 4;   // no swizzle: the k field stays where it is
  static EVAB_HD u32 at(u32 v, u32 k) { return swz_s<LOGN, JR>(idx_s<LOGN, J>(v, k)) & MASK; }
};
// strided pass J <-> rows of the contiguous last pass
template <int LOGN, int J, u32 MASK> struct AddrSC {
  static constexpr bool disjoint = false;
  static EVAB_HD u32 at(u32 v, u32 k) { return swz_c<LOGN>(idx_s<LOGN, J>(v, k)) & MASK; }
};
template <int LOGN, int J, int JR> EVAB_HD void xchg_write_s(const u64 (&x)[NTT_E], u64 *sm, u32 tid) { lin_write<AddrS<LOGN, J, JR, ~0u>>(x, sm, tid); }
template <int LOGN, int J, int JR> EVAB_HD void xchg_read_s(u64 (&x)[NTT_E], const u64 *sm, u32 tid) { lin_read<AddrS<LOGN, J, JR, ~0u>>(x, sm, tid); }
// strided pass J = P-2 side of the contiguous exchange
template <int LOGN, int J> EVAB_HD void xchg_write_sc(const u64 (&x)[NTT_E], u64 *sm, u32 tid) { lin_write<AddrSC<LOGN, J, ~0u>>(x, sm, tid); }
template <int LOGN, int J> EVAB_HD void xchg_read_sc(u64 (&x)[NTT_E], const u64 *sm, u32 tid) { lin_read<AddrSC<LOGN, J, ~0u>>(x, sm, tid); }
// contiguous side: the 16-byte chunk c of row `row` sits at chunk c ^ f(row): base ^ (c << 4) in bytes
template <u32 MASK> EVAB_HD u32 row_base_bytes(u32 v, u32 f) { return ((((v << NTT_EL) & MASK) | (f << 1)) << 3); }
template <int LOGN> EVAB_HD void xchg_read_c(u64 (&x)[NTT_E], const u64 *sm, u32 tid) {
  const u32 b0 = row_base_bytes<~0u>(tid, swz_rowf<LOGN>(tid));
#pragma unroll
  for (int c = 0; c < NTT_E / 2; c++) {
    const u64x2 v = *reinterpret_cast<const u64x2 *>(xelem(sm, b0 ^ ((u32)c << 4)));
    x[2 * c] = v.x; x[2 * c + 1] = v.y;
  }
}
template <int LOGN> EVAB_HD void xchg_write_c(const u64 (&x)[NTT_E], u64 *sm, u32 tid) {
  const u32 b0 = row_base_bytes<~0u>(tid, swz_rowf<LOGN>(tid));
#pragma unroll
  for (int c = 0; c < NTT_E / 2; c++) {
    u64x2 v; v.x = x[2 * c]; v.y = x[2 * c + 1];
    *reinterpret_cast<u64x2 *>(xelem(sm, b0 ^ ((u32)c << 4))) = v;
  }
}

// ---------------------------------------------------------------------------
// One residue spread over a cluster of CL CTAs (CL = 2 or 4, LOGN >= 12): CTA `rank` runs the
// virtual threads v = rank*Tc + tid, Tc = T/CL, and keeps the slice [rank*N/CL, (rank+1)*N/CL) of the
// exchange index space in its own shared memory (N/CL * 8 bytes), so several smaller CTAs share an SM
// and overlap each other's load / exchange / store phases.  After pass 0 (forward) the transform
// splits into 16 independent sub-transforms of N/16 points, CL-aligned: only the exchange between
// pass 0 and pass 1 crosses CTAs.  It is written straight into the consumer's shared memory
// (distributed shared memory stores) and followed by a cluster barrier; every other exchange is
// CTA-local with indices taken modulo N/CL.
// ---------------------------------------------------------------------------
template <int CL> struct SmemView {
  u64 *local;        // this CTA's slice
  u64 *peer[CL];     // generic pointers to every rank's slice (peer[rank] == local)
  // store into rank r's slice (host replay: a plain store; the device view in evab200.cu issues an asynchronous
  // distributed-shared-memory store that signals the receiver's mbarrier)
  EVAB_HD void put(int r, u32 idx, u64 v) const { peer[r][idx] = v; }
};
template <int LOGN, int CL> struct ClGeom {
  static_assert(CL == 1 || CL == 2 || CL == 4 || CL == 8, "cluster size 1, 2, 4 or 8");
  static_assert(CL == 1 || LOGN >= 12, "cluster-distributed transform needs N >= 4096");
  static constexpr int LGC = CL == 1 ? 0 : (CL == 2 ? 1 : (CL == 4 ? 2 : 3));
  static constexpr int Tc = NttGeom<LOGN>::T / CL;
  static constexpr int LGT = LOGN - NTT_EL - LGC;   // log2(Tc)
  static constexpr u32 NC = (u32)NttGeom<LOGN>::N / CL;
  static constexpr u32 mask = NC - 1u;
};
// local (masked) variants of the exchanges above; v = virtual thread id
template <int LOGN, int J, int JR, int CL> EVAB_HD void xchg_write_sl(const u64 (&x)[NTT_E], u64 *sm, u32 v) { lin_write<AddrS<LOGN, J, JR, ClGeom<LOGN, CL>::mask>>(x, sm, v); }
template <int LOGN, int J, int JR, int CL> EVAB_HD void xchg_read_sl(u64 (&x)[NTT_E], const u64 *sm, u32 v) { lin_read<AddrS<LOGN, J, JR, ClGeom<LOGN, CL>::mask>>(x, sm, v); }
template <int LOGN, int J, int CL> EVAB_HD void xchg_write_scl(const u64 (&x)[NTT_E], u64 *sm, u32 v) { lin_write<AddrSC<LOGN, J, ClGeom<LOGN, CL>::mask>>(x, sm, v); }
template <int LOGN, int J, int CL> EVAB_HD void xchg_read_scl(u64 (&x)[NTT_E], const u64 *sm, u32 v) { lin_read<AddrSC<LOGN, J, ClGeom<LOGN, CL>::mask>>(x, sm, v); }
template <int LOGN, int CL> EVAB_HD void xchg_read_cl(u64 (&x)[NTT_E], const u64 *sm, u32 v) {
  const u32 b0 = row_base_bytes<ClGeom<LOGN, CL>::mask>(v, swz_rowf<LOGN>(v));
#pragma unroll
  for (int c = 0; c < NTT_E / 2; c++) {
    const u64x2 t = *reinterpret_cast<const u64x2 *>(xelem(sm, b0 ^ ((u32)c << 4)));
    x[2 * c] = t.x; x[2 * c + 1] = t.y;
  }
}
template <int LOGN, int CL> EVAB_HD void xchg_write_cl(const u64 (&x)[NTT_E], u64 *sm, u32 v) {
  const u32 b0 = row_base_bytes<ClGeom<LOGN, CL>::mask>(v, swz_rowf<LOGN>(v));
#pragma unroll
  for (int c = 0; c < NTT_E / 2; c++) {
    u64x2 t; t.x = x[2 * c]; t.y = x[2 * c + 1];
    *reinterpret_cast<u64x2 *>(xelem(sm, b0 ^ ((u32)c << 4))) = t;
  }
}
// forward, pass 0 -> pass 1: element k of virtual thread v has natural index (k << (n-4)) | v; its
// reader is a pass-1 thread of rank k >> (4 - LGC) (compile-time per k)
template <int LOGN, int CL, class SMV> EVAB_HD void xchg_write_dist_fwd(const u64 (&x)[NTT_E], const SMV &sm, u32 v) {
  typedef ClGeom<LOGN, CL> C;
#pragma unroll
  for (int k = 0; k < NTT_E; k++) sm.put(k >> (NTT_EL - C::LGC), idx_s<LOGN, 0>(v, (u32)k) & C::mask, x[k]);
}
// inverse, pass 1 -> pass 0: the reader of natural index i is the pass-0 virtual thread
// v0 = i mod T, element k0 = i / T; it is stored in v0's CTA at (k0 << log2 Tc) | (v0 mod Tc).
// For a pass-1 writer (v, k1): k0 = v >> (n-8), v0 = (k1 << (n-8)) | (v mod 2^(n-8)), rank = k1 >> (4-LGC).
template <int LOGN, int CL, class SMV> EVAB_HD void xchg_write_dist_inv(const u64 (&x)[NTT_E], const SMV &sm, u32 v) {
  typedef ClGeom<LOGN, CL> C;
  constexpr int lb = NttGeom<LOGN>::lowbits(1);
  const u32 k0 = v >> lb, L = v & ((1u << lb) - 1u);
#pragma unroll
  for (int k = 0; k < NTT_E; k++) {
    const u32 v0 = ((u32)k << lb) | L;
    sm.put(k >> (NTT_EL - C::LGC), (k0 << C::LGT) | (v0 & (u32)(C::Tc - 1)), x[k]);
  }
}
template <int LOGN, int CL> EVAB_HD void xchg_read_dist_inv(u64 (&x)[NTT_E], const u64 *sm, u32 tid) {
#pragma unroll
  for (int k = 0; k < NTT_E; k++) x[k] = sm[((u32)k << ClGeom<LOGN, CL>::LGT) | tid];
}

// ---------------------------------------------------------------------------
// forward (Cooley-Tukey) register passes.  `b` is the compile-time tracked
// upper bound of every live value in units of p (values < b*p <= 16p < 2^64).
// `root` is the twiddle root prefix (twiddle index = (root << s) + group): 1 for a full transform.
// ---------------------------------------------------------------------------
// one forward stage over the registers: pair distance D (in k), E/2/D groups of
// twiddles starting at table index tw0 (consecutive).
template <int D> EVAB_HD void fwd_stage(u64 (&x)[NTT_E], const u64x2 *tw, u32 tw0, u64 p, int &b) {
  // exact Shoup quotient here: t < 2p, the bound grows by 2p per stage and two conditional
  // subtractions cover 14 stages (with the 3-product quotient of shoup_mad4 it grows by 4p per stage
  // and the extra subtractions cancel the cheaper multiply: measured equal at N=16384, -4 % at 4096)
  const u64 two_p = 2 * p, eight_p = 8 * p, np = 0 - p;
  const bool fix = b > 14;
  if (fix) b = 8;
#pragma unroll
  for (int g = 0; g < NTT_E / 2 / D; g++) {
    const u64x2 w = ldg_tw(tw + tw0 + g);
#pragma unroll
    for (int j = 0; j < D; j++) {
      const int k = g * 2 * D + j;
      u64 xx = x[k];
      if (fix) xx = csub(xx, eight_p);
      const u64 t = shoup_lazy_n(x[k + D], w.x, w.y, np);
      x[k] = xx + t;
      x[k + D] = xx - t + two_p;
    }
  }
  b += 2;
}
// strided pass J: stages 4J..4J+3, twiddle group prefix H = tid >> lowbits(J)
template <int LOGN, int J> EVAB_HD void fwd_pass_s(u64 (&x)[NTT_E], const u64x2 *tw, u32 root, u64 p, u32 tid, int &b) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(J);
  constexpr int s0 = NTT_EL * J;
  fwd_stage<8>(x, tw, (root << (s0 + 0)) + (H << 0), p, b);
  fwd_stage<4>(x, tw, (root << (s0 + 1)) + (H << 1), p, b);
  fwd_stage<2>(x, tw, (root << (s0 + 2)) + (H << 2), p, b);
  fwd_stage<1>(x, tw, (root << (s0 + 3)) + (H << 3), p, b);
}
// last pass: thread owns 16 contiguous coefficients; the R remaining stages pair at
// distance 2^(R-1) .. 1; stage with distance D uses group index (tid<<4|k) >> (log2 D + 1)
template <int LOGN> EVAB_HD void fwd_pass_c(u64 (&x)[NTT_E], const u64x2 *tw, u32 root, u64 p, u32 tid, int &b) {
  constexpr int R = NttGeom<LOGN>::R;
  if (R >= 4) fwd_stage<8>(x, tw, (root << (LOGN - 4)) + (tid << 0), p, b);
  if (R >= 3) fwd_stage<4>(x, tw, (root << (LOGN - 3)) + (tid << 1), p, b);
  if (R >= 2) fwd_stage<2>(x, tw, (root << (LOGN - 2)) + (tid << 2), p, b);
  if (R >= 1) fwd_stage<1>(x, tw, (root << (LOGN - 1)) + (tid << 3), p, b);
}
// reduce every register from < b*p to canonical [0,p)
EVAB_HD void canon(u64 (&x)[NTT_E], u64 p, int b) {
#pragma unroll
  for (int k = 0; k < NTT_E; k++) {
    u64 v = x[k];
    if (b > 8) v = csub(v, 8 * p);
    if (b > 4) v = csub(v, 4 * p);
    if (b > 2) v = csub(v, 2 * p);
    if (b > 1) v = csub(v, p);
    x[k] = v;
  }
}

// ---------------------------------------------------------------------------
// inverse (Gentleman-Sande) register passes.  Values stay < 8p on stage entry.
// ---------------------------------------------------------------------------
template <int D> EVAB_HD void inv_stage(u64 (&x)[NTT_E], const u64x2 *tw, u32 tw0, u64 p, int &b) {
  // entry bound b <= 8; sums are reduced by 8p only once they could reach 16p; the product is < 4p
  const u64 eight_p = 8 * p, np = 0 - p;
  const u64 bias = (u64)b * p;
  const bool fix = b > 4;
#pragma unroll
  for (int g = 0; g < NTT_E / 2 / D; g++) {
    const u64x2 w = ldg_tw(tw + tw0 + g);
#pragma unroll
    for (int j = 0; j < D; j++) {
      const int k = g * 2 * D + j;
      const u64 X = x[k], Y = x[k + D];
      u64 s = X + Y;
      if (fix) s = csub(s, eight_p);
      x[k] = s;
      x[k + D] = shoup_mad4(X - Y + bias, w.x, w.y, np, 0);
    }
  }
  b = fix ? 8 : 2 * b;
  if (b < 4) b = 4;
}
template <int LOGN> EVAB_HD void inv_pass_c(u64 (&x)[NTT_E], const u64x2 *tw, u32 root, u64 p, u32 tid, int &b) {
  constexpr int R = NttGeom<LOGN>::R;
  if (R >= 1) inv_stage<1>(x, tw, (root << (LOGN - 1)) + (tid << 3), p, b);
  if (R >= 2) inv_stage<2>(x, tw, (root << (LOGN - 2)) + (tid << 2), p, b);
  if (R >= 3) inv_stage<4>(x, tw, (root << (LOGN - 3)) + (tid << 1), p, b);
  if (R >= 4) inv_stage<8>(x, tw, (root << (LOGN - 4)) + (tid << 0), p, b);
}
template <int LOGN, int J> EVAB_HD void inv_pass_s(u64 (&x)[NTT_E], const u64x2 *tw, u32 root, u64 p, u32 tid, int &b) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(J);
  constexpr int s0 = NTT_EL * J;
  inv_stage<1>(x, tw, (root << (s0 + 3)) + (H << 3), p, b);
  inv_stage<2>(x, tw, (root << (s0 + 2)) + (H << 2), p, b);
  inv_stage<4>(x, tw, (root << (s0 + 1)) + (H << 1), p, b);
  inv_stage<8>(x, tw, (root << (s0 + 0)) + (H << 0), p, b);
}
// strided pass 0 of the inverse with the N^-1 scaling folded into its last stage (the only stage whose
// twiddle is the same for every thread, itw[1]): X' = (X + Y) * N^-1, Y' = (X - Y) * (itw[1] * N^-1),
// both canonical.  16 multiplies per thread instead of 8 + 16, and no bound fix-ups in that stage.
template <int LOGN> EVAB_HD void inv_pass0_scaled(u64 (&x)[NTT_E], const u64x2 *tw, u64 p, u32 tid, int &b, u64 ninv, u64 ninv_s, u64 w1n, u64 w1n_s) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(0);   // 0: every thread of pass 0 shares the root twiddles
  inv_stage<1>(x, tw, (1u << 3) + (H << 3), p, b);
  inv_stage<2>(x, tw, (1u << 2) + (H << 2), p, b);
  inv_stage<4>(x, tw, (1u << 1) + (H << 1), p, b);
  const u64 bias = (u64)b * p;                      // b <= 8: X + Y < 16p and X - Y + bias < 16p fit a u64
#pragma unroll
  for (int k = 0; k < NTT_E / 2; k++) {
    const u64 X = x[k], Y = x[k + NTT_E / 2];
    x[k] = csub(shoup_lazy(X + Y, ninv, ninv_s, p), p);
    x[k + NTT_E / 2] = csub(shoup_lazy(X - Y + bias, w1n, w1n_s, p), p);
  }
  b = 1;
}
// multiply by a Shoup constant (e.g. N^-1) and canonicalise
EVAB_HD void scale_canon(u64 (&x)[NTT_E], u64 c, u64 cs, u64 p) {
#pragma unroll
  for (int k = 0; k < NTT_E; k++) x[k] = csub(shoup_lazy(x[k], c, cs, p), p);
}

// ---------------------------------------------------------------------------
// The same passes in "two-row fold" arithmetic (modarith.cuh: fold_mul) for fold-friendly primes
// p = 2^60 - delta: 5 wide multiplies per butterfly instead of 6 wide + 4 low.  The multiplicand of a
// product may be ANY u64, so only sums need room; every register carries its own compile-time bound
// bb[k] in units of p/16 (the loops are fully unrolled, the bounds fold to constants) and a value is
// folded (3 instructions) only when the next sum could reach 16p.
// ---------------------------------------------------------------------------
struct FoldP { u64 p, p3, p8; u32 eps; };
#if defined(EVAB_BOUND_CHECK) && !defined(__CUDA_ARCH__)
#include <cstdio>
#include <cstdlib>
// test builds of the CPU emulator: every tracked bound is verified against the value it describes
#define EVAB_CHECK_BOUND(x, b, F) do { if ((unsigned __int128)(x) * 16 >= (unsigned __int128)(b) * (F).p || (b) > FB_MAX) { \
  fprintf(stderr, "bound violated at %s:%d: %llu !< %d/16 p\n", __FILE__, __LINE__, (unsigned long long)(x), (int)(b)); abort(); } } while (0)
#else
#define EVAB_CHECK_BOUND(x, b, F) do {} while (0)
#endif
template <class FPr> EVAB_HD FoldP fold_params(const FPr &P) { FoldP F; F.p = P.p; F.p3 = P.p3; F.p8 = P.p8; F.eps = P.eps; return F; }

template <int D> EVAB_HD void ffwd_stage(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, u32 tw0, const FoldP &F) {
  const u64x2 *twg = tw + (size_t)tw0;   // the stage's first group, addressed once; the groups are immediate offsets from it
#pragma unroll
  for (int g = 0; g < NTT_E / 2 / D; g++) {
    const u64x2 w = ldg_tw(twg + g);
#pragma unroll
    for (int j = 0; j < D; j++) {
      const int k = g * 2 * D + j;
      u64 X = x[k];
      int bx = bb[k];
      if (bx + 48 > FB_MAX) { X = fold61(X, F.eps); bx = FB_FOLD; }
      const u64 t = fold_mul(x[k + D], w.x, w.y, F.eps);   // < 2.2501 p
      x[k] = X + t;
      x[k + D] = X + F.p3 - t;
      bb[k] = bx + FB_MUL;
      bb[k + D] = bx + 48;
      EVAB_CHECK_BOUND(t, FB_MUL, F); EVAB_CHECK_BOUND(x[k], bb[k], F); EVAB_CHECK_BOUND(x[k + D], bb[k + D], F);
    }
  }
}
// the exchange between two passes hands register k of one thread to some other register of another thread:
// past a pass, every register takes the largest bound
EVAB_HD void bounds_merge(int (&bb)[NTT_E]) {
  int m = 0;
#pragma unroll
  for (int k = 0; k < NTT_E; k++) m = bb[k] > m ? bb[k] : m;
#pragma unroll
  for (int k = 0; k < NTT_E; k++) bb[k] = m;
}
template <int LOGN, int J> EVAB_HD void ffwd_pass_s(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, const FoldP &F, u32 tid) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(J);
  constexpr int s0 = NTT_EL * J;
  ffwd_stage<8>(x, bb, tw, (1u << (s0 + 0)) + (H << 0), F);
  ffwd_stage<4>(x, bb, tw, (1u << (s0 + 1)) + (H << 1), F);
  ffwd_stage<2>(x, bb, tw, (1u << (s0 + 2)) + (H << 2), F);
  ffwd_stage<1>(x, bb, tw, (1u << (s0 + 3)) + (H << 3), F);
  bounds_merge(bb);
}
template <int LOGN> EVAB_HD void ffwd_pass_c(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, const FoldP &F, u32 tid) {
  constexpr int R = NttGeom<LOGN>::R;
  if (R >= 4) ffwd_stage<8>(x, bb, tw, (1u << (LOGN - 4)) + (tid << 0), F);
  if (R >= 3) ffwd_stage<4>(x, bb, tw, (1u << (LOGN - 3)) + (tid << 1), F);
  if (R >= 2) ffwd_stage<2>(x, bb, tw, (1u << (LOGN - 2)) + (tid << 2), F);
  if (R >= 1) ffwd_stage<1>(x, bb, tw, (1u << (LOGN - 1)) + (tid << 3), F);
}
// every register (< 16p) to canonical [0,p)
EVAB_HD void fcanon(u64 (&x)[NTT_E], const FoldP &F) {
#pragma unroll
  for (int k = 0; k < NTT_E; k++) x[k] = fold_canon(x[k], F.eps, F.p);
}

// Gentleman-Sande butterfly: X' = X + Y, Y' = (X - Y + C p) w with C p >= Y.  Folds X / Y first when a sum would leave the u64.
EVAB_HD void finv_bfly(u64 &xa, u64 &xb, int &ba, int &bby, const u64x2 &w, const FoldP &F) {
  u64 X = xa, Y = xb;
  int bx = ba, by = bby;
  if (by > 128) { Y = fold61(Y, F.eps); by = FB_FOLD; }
  const bool big = by > 48;                       // bias 8p instead of 3p
  if (bx + (big ? 128 : 48) > FB_MAX || bx + by > FB_MAX) { X = fold61(X, F.eps); bx = FB_FOLD; }
  xa = X + Y;
  xb = fold_mul(X - Y + (big ? F.p8 : F.p3), w.x, w.y, F.eps);
  ba = bx + by;
  bby = FB_MUL;
  EVAB_CHECK_BOUND(X, bx, F); EVAB_CHECK_BOUND(Y, by, F); EVAB_CHECK_BOUND(xa, ba, F); EVAB_CHECK_BOUND(xb, bby, F);
}
template <int D> EVAB_HD void finv_stage(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, u32 tw0, const FoldP &F) {
  const u64x2 *twg = tw + (size_t)tw0;   // as in ffwd_stage
#pragma unroll
  for (int g = 0; g < NTT_E / 2 / D; g++) {
    const u64x2 w = ldg_tw(twg + g);
#pragma unroll
    for (int j = 0; j < D; j++) {
      const int k = g * 2 * D + j;
      finv_bfly(x[k], x[k + D], bb[k], bb[k + D], w, F);
    }
  }
}
template <int LOGN> EVAB_HD void finv_pass_c(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, const FoldP &F, u32 tid) {
  constexpr int R = NttGeom<LOGN>::R;
  if (R >= 1) finv_stage<1>(x, bb, tw, (1u << (LOGN - 1)) + (tid << 3), F);
  if (R >= 2) finv_stage<2>(x, bb, tw, (1u << (LOGN - 2)) + (tid << 2), F);
  if (R >= 3) finv_stage<4>(x, bb, tw, (1u << (LOGN - 3)) + (tid << 1), F);
  if (R >= 4) finv_stage<8>(x, bb, tw, (1u << (LOGN - 4)) + (tid << 0), F);
  bounds_merge(bb);
}
template <int LOGN, int J> EVAB_HD void finv_pass_s(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, const FoldP &F, u32 tid) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(J);
  constexpr int s0 = NTT_EL * J;
  finv_stage<1>(x, bb, tw, (1u << (s0 + 3)) + (H << 3), F);
  finv_stage<2>(x, bb, tw, (1u << (s0 + 2)) + (H << 2), F);
  finv_stage<4>(x, bb, tw, (1u << (s0 + 1)) + (H << 1), F);
  finv_stage<8>(x, bb, tw, (1u << (s0 + 0)) + (H << 0), F);
  bounds_merge(bb);
}
// strided pass 0 of the inverse, N^-1 folded into its last stage (see inv_pass0_scaled); `half` != 0
// adds floor(p/2) before the canonicalisation (EPI_ADDHALF).  Output canonical.
template <int LOGN, class FPr> EVAB_HD void finv_pass0_scaled(u64 (&x)[NTT_E], int (&bb)[NTT_E], const u64x2 *tw, const FoldP &F, u32 tid, const FPr &P, u64 half) {
  const u32 H = tid >> NttGeom<LOGN>::lowbits(0);
  finv_stage<1>(x, bb, tw, (1u << 3) + (H << 3), F);
  finv_stage<2>(x, bb, tw, (1u << 2) + (H << 2), F);
  finv_stage<4>(x, bb, tw, (1u << 1) + (H << 1), F);
#pragma unroll
  for (int k = 0; k < NTT_E / 2; k++) {
    u64 X = x[k], Y = x[k + NTT_E / 2];
    int bx = bb[k], by = bb[k + NTT_E / 2];
    if (by > 128) { Y = fold61(Y, F.eps); by = FB_FOLD; }
    const bool big = by > 48;
    if (bx + (big ? 128 : 48) > FB_MAX || bx + by > FB_MAX) { X = fold61(X, F.eps); bx = FB_FOLD; }
    // products < 2.2501 p, + half < 2.7501 p: fold_canon takes anything below 16p
    x[k] = fold_canon(fold_mul(X + Y, P.ninv, P.ninv_v, F.eps) + half, F.eps, F.p);
    x[k + NTT_E / 2] = fold_canon(fold_mul(X - Y + (big ? F.p8 : F.p3), P.itw1n, P.itw1n_v, F.eps) + half, F.eps, F.p);
    bb[k] = bb[k + NTT_E / 2] = FB_CANON;
  }
}
