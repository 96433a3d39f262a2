// evab200.cu -- C-ABI implementation (include/evab200.h): CUDA backend for the
// op compositions in ops_impl.hpp, sm_90a kernels around the bodies in
// ntt_kernels.cuh / ops_kernels.cuh.  Product code: never includes or links
// anything under oracle/.
#include "../../include/evab200.h"
#include "host_tables.hpp"
#include "ops_impl.hpp"
#include "key_expand.cuh"
#include "compact_kernels.cuh"
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

static thread_local std::string g_err;
static int fail(const std::string &m) { g_err = m; return 1; }
#define CUDA_OK(x)                                                                       \
  do {                                                                                   \
    cudaError_t e_ = (x);                                                                \
    if (e_ != cudaSuccess) return fail(std::string(#x) + ": " + cudaGetErrorString(e_)); \
  } while (0)

extern "C" const char *evab_last_error(void) { return g_err.c_str(); }
extern "C" int evab_version(void) { return 1; }

struct evab_ctx {
  CtxView v;
  int device, sms;
  int ntt_cluster = 0;         // CTAs per residue (0 = automatic), evab_ctx_set_ntt_cluster
  std::vector<u64> primes;
  std::vector<FoldPrime> fold_host;
  PrimeDev *d_primes = nullptr;
  u64x2 *d_tw = nullptr;
  u64x2 *d_qinv = nullptr;
  u64x2 *d_qinv_f = nullptr;
  u64 *d_halfmod = nullptr;
  u64 *d_zeros = nullptr;
  cplx *d_roots = nullptr;
  u32 *d_slot = nullptr;
  u64 *d_pow2 = nullptr;
  std::map<u64, u32 *> perms;  // galois elt -> device permutation table (NTT domain)
  std::map<u64, u32 *> cperms; // galois elt -> device signed gather table (coefficient domain)
  std::mutex mu;
  mutable std::atomic<unsigned long long> launches{0};
};
static cudaStream_t S(void *s) { return (cudaStream_t)s; }

// thread-local batched-issue state (evab_set_batch)
struct BatchState { int batch = 1; long long stride = 0, vstride = 0; };
static thread_local BatchState g_batch;
extern "C" int evab_set_ntt_cluster(int ctas_per_residue);
extern "C" int evab_set_batch(int batch, size_t stride_words, size_t value_stride) {
  if (batch < 1 || batch > 65535) return fail("evab_set_batch: batch must be in [1, 65535]");
  g_batch.batch = batch; g_batch.stride = (long long)stride_words; g_batch.vstride = (long long)value_stride;
  return 0;
}
// thread-local key selection (evab_set_key_bank): instance b reads its keys at + tenant[b] * stride words
// c1: the c1 region of every instance (evab_set_key_c1_rows), read by the C1 instances only
struct KeyBankSel { const int32_t *tenant = nullptr; long long stride = 0; const int32_t *c1 = nullptr; };
static thread_local KeyBankSel g_bank;
extern "C" int evab_set_key_bank(const int32_t *d_tenant_of_instance, size_t tenant_stride_words) {
  g_bank.tenant = d_tenant_of_instance;
  g_bank.stride = d_tenant_of_instance ? (long long)tenant_stride_words : 0;
  return 0;
}
// thread-local cached c1 rows (evab_set_key_c1_rows): instance b of a seeded bank launch reads its keys' c1 rows at + region[b] *
// stride words, or draws them (region[b] < 0)
extern "C" int evab_set_key_c1_rows(const int32_t *d_region_of_instance) {
  g_bank.c1 = d_region_of_instance;
  return 0;
}
// thread-local inline hoist constants (evab_set_hoist_inline): the cadd operands of the hoisted rotations are indicator rows
static thread_local bool g_inline = false;
extern "C" int evab_set_hoist_inline(int on) {
  g_inline = on != 0;
  return 0;
}
// thread-local seeded keys (evab_set_key_seeded): the key operands of the key switches are seeded images, c1 drawn in the kernels
static thread_local bool g_seeded = false;
extern "C" int evab_set_key_seeded(int on) {
  g_seeded = on != 0;
  return 0;
}


// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
// ---- cluster protocol of the one exchange that crosses CTAs (CL > 1) ---------------------------------------
// barrier.cluster.arrive.release / wait.acquire around the distributed-shared-memory stores would put a GPU-scope
// memory fence on the arrive and an L1 invalidate on the wait of every exchange.  Instead every CTA owns
// two mbarriers behind its exchange slice:
//   full : completes when the N/CL * 8 bytes of the distributed exchange have landed in this CTA's slice.  The
//          writers use st.async (asynchronous DSMEM store that reports its bytes to the receiver's mbarrier), the
//          receiver's threads spin on try_wait: no fence, no block barrier, no L1 invalidate.
//   free : (inverse only) counts one arrival per warp of the whole cluster once that warp has read its slice for
//          the last time; a CTA waits on its own copy before it stores into its peers.
// One relaxed cluster barrier at kernel start makes the initialised mbarriers visible (as in CUTLASS prologues).
__device__ __forceinline__ u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
template <int LOGN, int CL> struct DevCluster {
  static constexpr u32 SLICE_BYTES = (u32)(NttGeom<LOGN>::N / CL) * 8u;
  static constexpr u32 WARPS = (u32)(NttGeom<LOGN>::T / CL) / 32u;
  u32 full, free_;   // shared::cta addresses of this CTA's barriers
};
template <int LOGN, int CL> struct DevSmemView {
  u64 *local;
  u32 peer32[CL];    // shared::cluster address of every rank's slice; its `full` barrier sits SLICE_BYTES behind
  __device__ __forceinline__ void put(int r, u32 idx, u64 v) const {
    const u32 a = peer32[r] + (idx << 3), mb = peer32[r] + DevCluster<LOGN, CL>::SLICE_BYTES;
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];" ::"r"(a), "l"(v), "r"(mb) : "memory");
  }
};
template <int LOGN, int CL> __device__ __forceinline__ DevSmemView<LOGN, CL> dev_smem_view(u64 *sm) {
  DevSmemView<LOGN, CL> v;
  v.local = sm;
  const u32 base = smem_u32(sm);
#pragma unroll
  for (int r = 0; r < CL; r++) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(v.peer32[r]) : "r"(base), "r"(r));
  return v;
}
template <int LOGN, int CL> struct DevHooks {
  DevCluster<LOGN, CL> c;
  __device__ __forceinline__ explicit DevHooks(u64 *sm) {
    c.full = smem_u32(sm) + DevCluster<LOGN, CL>::SLICE_BYTES;
    c.free_ = c.full + 8;
  }
  __device__ __forceinline__ void start() const {
    if (CL == 1) return;
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(c.full) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(c.free_), "r"((u32)CL * DevCluster<LOGN, CL>::WARPS) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      // the one arrival of `full`, announcing the bytes the peers (and this CTA) will deliver
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(c.full), "r"(DevCluster<LOGN, CL>::SLICE_BYTES) : "memory");
    }
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  }
  __device__ __forceinline__ void ready() const {
    if (CL > 1) asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
  }
  __device__ __forceinline__ void released() const {
    if (CL == 1) return;
    __syncwarp();
    if ((threadIdx.x & 31u) == 0) {
      const u32 mine = c.free_;
#pragma unroll
      for (int r = 0; r < CL; r++) {
        u32 remote;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(mine), "r"(r));
        asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
      }
    }
  }
  static __device__ __forceinline__ void spin(u32 bar) {
    asm volatile("{\n\t.reg .pred p;\n\tEVAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@!p bra EVAB_WAIT;\n\t}" ::"r"(bar) : "memory");
  }
  __device__ __forceinline__ void acquire_free() const { if (CL > 1) spin(c.free_); }
  __device__ __forceinline__ void landed() const { if (CL > 1) spin(c.full); }
};
// barrier after a phase: 0 = block, 1 = the distributed exchange has landed in this CTA's slice, 2 = none
template <int LOGN, int CL> struct DevSync {
  DevHooks<LOGN, CL> hk;
  __device__ __forceinline__ void operator()(int kind) const {
    if (CL > 1 && kind == 1) hk.landed();
    else if (kind != 2) __syncthreads();
  }
};
template <int CL> __device__ __forceinline__ SmemView<CL> smem_view(u64 *sm) {   // CL = 1: plain view
  SmemView<CL> v;
  v.local = sm;
#pragma unroll
  for (int r = 0; r < CL; r++) v.peer[r] = sm;
  return v;
}
// CL = 1: one CTA = one residue, T = N/16 threads, 64 registers.
// CL = 2, 4, 8: one residue over a cluster of CL CTAs of T/CL threads (ntt_core.cuh), CL CTAs per SM more.
template <int LOGN, int PRO, int EPI, int CL, int AR>
__global__ void __launch_bounds__(NttGeom<LOGN>::T / CL, 1024 / (NttGeom<LOGN>::T / CL)) k_ntt_fwd(const NttLaunch L, const long long bstride) {
  extern __shared__ __align__(16) u64 sm[];
  typedef FwdBody<LOGN, PRO, EPI, CL, AR> B;
  const NttJob J = ntt_job_qr(L, blockIdx.y, blockIdx.x / CL, blockIdx.x % CL, (long long)blockIdx.z * bstride);
  if (J.skip) return;
  NttState S;
  const u32 tid = threadIdx.x;
  if (PRO == PRO_PLAIN && EPI == EPI_STORE && J.bcast) { fwd_const_poly<LOGN>(J, B::vtid(J, tid)); return; }
  const DevHooks<LOGN, CL> hk(sm);
  hk.start();   // relaxed cluster arrive; the matching wait sits right before the first store into a peer (hk.ready in phase 0)
  if constexpr (CL > 1) PhaseLoop<B, 0, B::NPH>::run(S, L, J, tid, dev_smem_view<LOGN, CL>(sm), DevSync<LOGN, CL>{hk}, hk);
  else PhaseLoop<B, 0, B::NPH>::run(S, L, J, tid, smem_view<1>(sm), DevSync<LOGN, CL>{hk}, hk);
  B::phE(S, L, J, tid);
}
template <int LOGN, int PRO, int EPI, int CL, int AR>
__global__ void __launch_bounds__(NttGeom<LOGN>::T / CL, 1024 / (NttGeom<LOGN>::T / CL)) k_ntt_inv(const NttLaunch L, const long long bstride) {
  extern __shared__ __align__(16) u64 sm[];
  typedef InvBody<LOGN, PRO, EPI, CL, AR> B;
  const NttJob J = ntt_job_qr(L, blockIdx.y, blockIdx.x / CL, blockIdx.x % CL, (long long)blockIdx.z * bstride);
  if (J.skip) return;
  NttState S;
  const DevHooks<LOGN, CL> hk(sm);
  hk.start();   // the matching wait sits right before this CTA first signals its peers (hk.ready in the pass-1 phase)
  if constexpr (CL > 1) PhaseLoop<B, 0, B::NPH>::run(S, L, J, threadIdx.x, dev_smem_view<LOGN, CL>(sm), DevSync<LOGN, CL>{hk}, hk);
  else PhaseLoop<B, 0, B::NPH>::run(S, L, J, threadIdx.x, smem_view<1>(sm), DevSync<LOGN, CL>{hk}, hk);
}
template <int OP> __global__ void __launch_bounds__(256) k_dyadic(const DyArgs A, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 4; j < A.N; j += gridDim.x * blockDim.x * 4)
    dyadic_elem<OP>(A, blockIdx.y, j, off);
}
__global__ void __launch_bounds__(256) k_mul_plain(const DyArgs A, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 4; j < A.N; j += gridDim.x * blockDim.x * 4)
    mulpt_elem(A, blockIdx.y, j, off);
}
template <bool SQ> __global__ void __launch_bounds__(256) k_mul_ct(const MulArgs A, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2)
    mulct_elem<SQ>(A, blockIdx.y, j, off);
}
__global__ void __launch_bounds__(256) k_sum_terms(const SumArgs A, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2)
    sum_terms_elem(A, blockIdx.y, j, off);
}
// key offset of this block's instance: BANK = false is the shared-key launch (offset 0, the table is not read)
template <bool BANK> __device__ __forceinline__ long long key_off(const KeyBankSel &K) { return BANK ? (long long)__ldg(K.tenant + blockIdx.z) * K.stride : 0; }
// SEED: the c1 tile of a seeded key, [ell][2 blockDim.x] words of dynamic shared memory (seed_tile_bytes; ops_kernels.cuh SeedTileDev).
// C1 (seeded bank launches with evab_set_key_c1_rows): the block's instance copies its c1 rows from region K.c1[blockIdx.z] when it
// has one; the tile's offset is taken from the tenant's image (key + koff) to the region (key + region * stride)
template <bool C1 = false> __device__ __forceinline__ SeedTileDev seed_tile(const KeyBankSel &K, long long koff) {
  extern __shared__ __align__(16) u64 sm[];
  SeedTileDev t{sm};
  if (C1) {
    const int r = __ldg(K.c1 + blockIdx.z);
    t.cached = r >= 0;
    t.c1d = (long long)r * K.stride - koff;
  }
  return t;
}
// INL: inline hoist constants (ks_inner_elem); SEED: seeded key images (every launch has N / 512 blocks per row or a multiple of
// them, so the tile loop is uniform over the block)
template <bool BANK, bool INL, bool SEED, bool C1 = false> __global__ void __launch_bounds__(256) k_ks_inner(const IpArgs A, const long long bstride, const KeyBankSel K) {
  const long long off = (long long)blockIdx.z * bstride;   // parameters stay in constant memory: no local copy
  const long long koff = key_off<BANK>(K);
  SeedTileDev tile = seed_tile<C1>(K, koff);
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2)
    ks_inner_elem<INL, SEED>(A, blockIdx.y, j, off, koff, SEED ? &tile : nullptr);
}
__global__ void __launch_bounds__(256) k_scale_c0(const u64 *c0, u64 *ext, const PrimeDev *primes, int ell, int k, int N, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) scale_c0_elem(c0, ext, primes, ell, k, N, blockIdx.y, j, off);
}
// INL: 3 blocks per SM (80 registers) -- at 4 the inline instance spills about 100 bytes
template <bool BANK, bool INL, bool SEED, bool C1 = false> __global__ void __launch_bounds__(256, INL ? 3 : 4) k_rot_many(const RotManyArgs A, const long long bstride, const KeyBankSel K) {
  const long long off = (long long)blockIdx.z * bstride, koff = key_off<BANK>(K);
  const int i = blockIdx.y / (A.ell + 1), mi = blockIdx.y % (A.ell + 1);
  SeedTileDev tile = seed_tile<C1>(K, koff);
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2)
    rot_many_elem<INL, SEED>(A, i, mi, j, off, koff, SEED ? &tile : nullptr);
}
// grid.y = row of the extended basis; every thread loops over the rotations, so blocks are kept small for more of them
template <int NOUT, bool BANK, bool INL, bool SEED, bool C1 = false> __global__ void __launch_bounds__(128) k_rot_wsum_ip(const WsumIpArgs A, const long long bstride, const KeyBankSel K) {
  const long long off = (long long)blockIdx.z * bstride, koff = key_off<BANK>(K);
  SeedTileDev tile = seed_tile<C1>(K, koff);
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2)
    rot_wsum_ip_elem<NOUT, INL, SEED>(A, blockIdx.y, j, off, koff, SEED ? &tile : nullptr);
}
// grid.y = (polynomial, residue) of the outputs
__global__ void __launch_bounds__(256) k_rot_wsum(const WsumArgs A, const long long bstride) {
  const long long off = (long long)blockIdx.z * bstride;
  const int c = blockIdx.y / A.ell, r = blockIdx.y % A.ell;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2) rot_wsum_elem(A, c, r, j, off);
}
// block = 32 element pairs x n rotations (one warp per rotation); the parts meet in shared memory, one output sum at a time
template <bool BANK> __global__ void __launch_bounds__(32 * LRS_MAX) k_lazy_rotsum(const LazyRotSumArgs A, const long long bstride, const KeyBankSel K) {
  __shared__ u64 sh[LRS_MAX][4][32];
  const long long off = (long long)blockIdx.z * bstride;
  const int j = (blockIdx.x * 32 + threadIdx.x) * 2, i = threadIdx.y, mi = blockIdx.y;
  u64 part[LRS_OUT][4];
  lazy_rotsum_part(A, mi, j, i, off, part, key_off<BANK>(K));
#pragma unroll
  for (int o = 0; o < LRS_OUT; o++) {
    if (o >= A.nout) break;
    if (o) __syncthreads();
#pragma unroll
    for (int c = 0; c < 4; c++) sh[i][c][threadIdx.x] = part[o][c];
    __syncthreads();
    if (i == o % A.n) {
      u64 sum[4];
#pragma unroll
      for (int c = 0; c < 4; c++) { u64 s = 0; for (int r = 0; r < A.n; r++) s += sh[r][c][threadIdx.x]; sum[c] = s; }
      lazy_rotsum_store(A, mi, j, o, off, sum);
    }
  }
}
__global__ void __launch_bounds__(256) k_hoist_const(const HoistConstArgs A) {
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2) hoist_const_elem(A, blockIdx.y, j);
}
// grid (coefficient tiles, prime m, key g)
__global__ void __launch_bounds__(256) k_hoist_const_levels(const HoistLevelsArgs A) {
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < A.N; j += gridDim.x * blockDim.x * 2) hoist_levels_elem(A, blockIdx.z, blockIdx.y, j);
}
// grid (blocks of 8 coefficients, c1 row r, key g): one ChaCha20 block per thread
__global__ void __launch_bounds__(256) k_expand_uniform(const ExpandArgs A) {
  const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < A.N / 8) expand_uniform_elem(A, blockIdx.z, blockIdx.y, t);
}
// grid (blocks of 8 coefficients, c1 row r, seeded image i): one ChaCha20 block per thread
__global__ void __launch_bounds__(256) k_expand_seeded_c1(const u64 *images, u64 *rows, const PrimeDev *primes, int k, int N) {
  const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < (u32)N / 8) expand_seeded_c1_elem(images, rows, primes, k, (size_t)N, blockIdx.z, blockIdx.y, t);
}
// grid (blocks of 8 coefficients, ciphertext row m, entry i of the launch): one ChaCha20 block per thread; rows m >= ell_i return
__global__ void __launch_bounds__(256) k_expand_cipher_uniform(const CipherExpandArgs A) {
  const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < A.N / 8 && blockIdx.y < A.e[blockIdx.z].ell) expand_cipher_elem(A, blockIdx.z, blockIdx.y, t);
}
// ---- server-resident ciphertexts (evab_gather_ciphers): n device ranges copied into arena slots.  The ranges travel by value in
// the launch arguments, GW_MAX_ENTRIES per launch under the 4 KB parameter limit, so the call needs no device table and a captured
// graph replays it as it is
#define GW_MAX_ENTRIES 160
#define GW_THREADS 128
#define GW_UNROLL 4                       // 16-byte vectors in flight per thread
struct GatherEntry { const u64x2 *src; u64x2 *dst; u64 vecs; };   // vecs: 16-byte vectors (2 words each)
struct GatherArgs { GatherEntry e[GW_MAX_ENTRIES]; };
static_assert(sizeof(GatherArgs) <= 4096, "the gather's arguments must fit the classic 4 KB parameter space");
// grid (tiles of GW_THREADS * GW_UNROLL vectors, entry i of the launch): GW_UNROLL loads in flight, then their stores
__global__ void __launch_bounds__(GW_THREADS) k_gather_words(const GatherArgs A) {
  const GatherEntry E = A.e[blockIdx.y];
  const u64 step = (u64)gridDim.x * GW_THREADS * GW_UNROLL;
  for (u64 i = (u64)blockIdx.x * GW_THREADS * GW_UNROLL + threadIdx.x; i < E.vecs; i += step) {
    u64x2 v[GW_UNROLL];
#pragma unroll
    for (int u = 0; u < GW_UNROLL; u++)
      if (i + u * GW_THREADS < E.vecs) v[u] = E.src[i + u * GW_THREADS];
#pragma unroll
    for (int u = 0; u < GW_UNROLL; u++)
      if (i + u * GW_THREADS < E.vecs) E.dst[i + u * GW_THREADS] = v[u];
  }
}
// ---- compact responses (evab_compact_ciphers): grid (tiles of output words, polynomial, entry of the launch); one thread per word
static_assert(sizeof(CompactArgs) <= 4096, "the compaction's arguments must fit the classic 4 KB parameter space");
__global__ void __launch_bounds__(CMP_THREADS) k_compact(const CompactArgs A) {
  const u32 w = blockIdx.x * CMP_THREADS + threadIdx.x;
  if (w < A.words) compact_word(A, blockIdx.z, blockIdx.y, w);
}
__global__ void __launch_bounds__(256) k_compact_unpack(const u64 *words, u32 b, u32 W, const PrimeDev *primes, u32 nres, u32 N, u64 *out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) compact_unpack_elem(words, b, W, primes, nres, N, out, i);
}
__global__ void __launch_bounds__(256) k_compact_finish(const CrtTables T, const PrimeDev *primes, u32 nres, u32 N, u32 b, const u64 *coef, u32 nout,
                                                        u64 *out, long long *z) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) compact_finish_elem(T, primes, nres, N, b, coef, nout, out, z, i);
}
__global__ void __launch_bounds__(256) k_hoist_indicator(u64 *out, const u32 *ctab, int N) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) hoist_indicator_elem(out, ctab, N, blockIdx.y, j);
}
__global__ void __launch_bounds__(256) k_dec_compose(const DecArgs A) {
  for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < A.N; j += gridDim.x * blockDim.x) dec_compose(A, j);
}
__global__ void __launch_bounds__(256) k_dec_fft(const DecArgs A, u32 m) {
  for (u32 b = blockIdx.x * blockDim.x + threadIdx.x; b < A.N / 2; b += gridDim.x * blockDim.x) dec_fft_bfly(A, m, b);
}
__global__ void __launch_bounds__(256) k_dec_gather(const DecArgs A) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < A.N / 2; i += gridDim.x * blockDim.x) dec_gather(A, i);
}
__global__ void __launch_bounds__(256) k_enc_scatter(const EncBatch B, const long long bstride, const long long vstride) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B.N / 2; i += gridDim.x * blockDim.x)
    enc_scatter(B, blockIdx.y, i, (long long)blockIdx.z * bstride, (long long)blockIdx.z * vstride);
}
__global__ void __launch_bounds__(256) k_enc_fft(const EncBatch B, u32 g, int nstages, const long long bstride) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < B.N / 8; t += gridDim.x * blockDim.x)
    enc_fft8(B, blockIdx.y, t, g, nstages, (long long)blockIdx.z * bstride);
}
__global__ void __launch_bounds__(256) k_enc_round(const EncBatch B, const long long bstride) {
  for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < B.N; j += gridDim.x * blockDim.x)
    enc_round(B, blockIdx.y, j, (long long)blockIdx.z * bstride);
}
__global__ void __launch_bounds__(256) k_enc_uniform(const EncUniform B, const long long bstride) {
  const u32 e = blockIdx.y / B.ell, i = blockIdx.y % B.ell;
  for (u32 j = (blockIdx.x * blockDim.x + threadIdx.x) * 2; j < B.N; j += gridDim.x * blockDim.x * 2)
    enc_uniform_elem(B, e, i, j, (long long)blockIdx.z * bstride);
}

// ---------------------------------------------------------------------------
// CUDA backend
// ---------------------------------------------------------------------------
// CTAs per residue (evab_set_ntt_cluster); 0 = automatic: 128-thread CTAs, i.e. N/2048 CTAs per residue
// (N=16384: 8, 8192: 4, 4096: 2).  Sobel ops/s and single-instance latency at N=16384 (bench.py --ntt-cluster,
// H100 SXM at 700 W): 1: 572k 0.85 ms, 2: 635k 0.55, 4: 683k 0.40, 8: 691k 0.34.
static std::atomic<int> g_ntt_cluster{0};   // default for contexts created afterwards (evab_set_ntt_cluster)
template <int LOGN> static int ntt_cluster_for(int requested) {
  int most = NttGeom<LOGN>::T / 128 < 1 ? 1 : NttGeom<LOGN>::T / 128;   // keep CTAs at >= 128 threads
  if (most > 8) most = 8;                                                 // portable cluster size
  int cl = requested ? requested : most;
  if (cl > most) cl = most;
  if (LOGN == 15 && cl < 2) cl = 2;                                       // 2048 threads never fit one CTA
  return cl;
}

// grid = (inner * cluster, q, batch instance); more than 65535 q's are issued in slices
template <class K> static int launch_ntt(K kernel, const NttLaunch &L0, size_t jobs, int threads, size_t smem, int cluster, cudaStream_t st, std::atomic<bool> *done) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (!done[dev & 63].load()) {
    CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    done[dev & 63].store(true);
  }
  const size_t inner = (size_t)L0.inner, nq = (jobs + inner - 1) / inner;
  if (nq * inner != jobs) return fail("NTT launch: job count must be a multiple of the inner dimension");
  if (nq > 65535 && L0.prime_on_q) return fail("NTT launch: too many polynomials for a prime-per-polynomial launch");
  for (size_t q0 = 0; q0 < nq; q0 += 65535) {
    NttLaunch L = L0;
    const long long o = (long long)q0;
    L.src += o * L.src_sq; L.dst += o * L.dst_sq;
    if (L.aux0) L.aux0 += o * L.aux0_sq;
    if (L.aux1) L.aux1 += o * L.aux1_sq;
    if (L.cflags) L.cflags += o;
    L.aux1_polys = L0.aux1_polys - (int)(o > (1 << 30) ? (1 << 30) : o);
    const size_t n = nq - q0 < 65535 ? nq - q0 : 65535;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(inner * cluster), (unsigned)n, (unsigned)g_batch.batch);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, L, g_batch.stride));
  }
  return 0;
}
template <int LOGN, int PRO, int EPI, int CL, int AR> static int launch_fwd_m(const NttLaunch &L, size_t jobs, cudaStream_t st) {
  static std::atomic<bool> done[64];
  return launch_ntt(k_ntt_fwd<LOGN, PRO, EPI, CL, AR>, L, jobs, NttGeom<LOGN>::T / CL, (size_t)NttGeom<LOGN>::N / CL * sizeof(u64) + (CL > 1 ? 16 : 0), CL, st, done);
}
template <int LOGN, int CL, int AR> static int launch_fwd_c(const NttLaunch &L, size_t jobs, cudaStream_t st) {
  if (L.pro == PRO_PLAIN && L.epi == EPI_STORE) return launch_fwd_m<LOGN, PRO_PLAIN, EPI_STORE, CL, AR>(L, jobs, st);
  if (L.pro == PRO_MODRED && L.epi == EPI_STORE) return launch_fwd_m<LOGN, PRO_MODRED, EPI_STORE, CL, AR>(L, jobs, st);
  if (L.pro == PRO_MODRED && L.epi == EPI_STORE_LAZY) return launch_fwd_m<LOGN, PRO_MODRED, EPI_STORE_LAZY, CL, AR>(L, jobs, st);
  if (L.pro == PRO_MODRED && L.epi == EPI_DIVROUND) return launch_fwd_m<LOGN, PRO_MODRED, EPI_DIVROUND, CL, AR>(L, jobs, st);
  if (L.pro == PRO_PLAIN && L.epi == EPI_DIVROUND) return launch_fwd_m<LOGN, PRO_PLAIN, EPI_DIVROUND, CL, AR>(L, jobs, st);
  if (L.pro == PRO_MODRED_SG && L.epi == EPI_STORE_LAZY) return launch_fwd_m<LOGN, PRO_MODRED_SG, EPI_STORE_LAZY, CL, AR>(L, jobs, st);
  return fail("unsupported forward NTT prologue/epilogue combination");
}
template <int LOGN, int AR> static int launch_fwd_a(const NttLaunch &L, size_t jobs, cudaStream_t st, int cluster) {
  if constexpr (LOGN >= 12) {
    const int cl = ntt_cluster_for<LOGN>(cluster);
    if constexpr (LOGN >= 13) {
      if (cl == 4) return launch_fwd_c<LOGN, 4, AR>(L, jobs, st);
      if (cl == 8) return launch_fwd_c<LOGN, 8, AR>(L, jobs, st);
    }
    if (cl == 2 || LOGN == 15) return launch_fwd_c<LOGN, 2, AR>(L, jobs, st);
  }
  if constexpr (LOGN <= 14) return launch_fwd_c<LOGN, 1, AR>(L, jobs, st);
  return fail("unsupported cluster size");
}
template <int LOGN> static int launch_fwd_t(const NttLaunch &L, size_t jobs, cudaStream_t st, bool fold, int cluster) {
  return fold ? launch_fwd_a<LOGN, 1>(L, jobs, st, cluster) : launch_fwd_a<LOGN, 0>(L, jobs, st, cluster);
}
template <int LOGN, int PRO, int EPI, int CL, int AR> static int launch_inv_m(const NttLaunch &L, size_t jobs, cudaStream_t st) {
  static std::atomic<bool> done[64];
  return launch_ntt(k_ntt_inv<LOGN, PRO, EPI, CL, AR>, L, jobs, NttGeom<LOGN>::T / CL, (size_t)NttGeom<LOGN>::N / CL * sizeof(u64) + (CL > 1 ? 16 : 0), CL, st, done);
}
template <int LOGN, int CL, int AR> static int launch_inv_c(const NttLaunch &L, size_t jobs, cudaStream_t st) {
  if (L.pro == PRO_PLAIN && L.epi == EPI_STORE) return launch_inv_m<LOGN, PRO_PLAIN, EPI_STORE, CL, AR>(L, jobs, st);
  if (L.pro == PRO_PLAIN && L.epi == EPI_ADDHALF) return launch_inv_m<LOGN, PRO_PLAIN, EPI_ADDHALF, CL, AR>(L, jobs, st);
  if (L.pro == PRO_GATHER && L.epi == EPI_STORE) return launch_inv_m<LOGN, PRO_GATHER, EPI_STORE, CL, AR>(L, jobs, st);
  if (L.pro == PRO_PLAIN && L.epi == EPI_STORE_ZFLAG) return launch_inv_m<LOGN, PRO_PLAIN, EPI_STORE_ZFLAG, CL, AR>(L, jobs, st);
  return fail("unsupported inverse NTT prologue/epilogue combination");
}
template <int LOGN, int AR> static int launch_inv_a(const NttLaunch &L, size_t jobs, cudaStream_t st, int cluster) {
  if constexpr (LOGN >= 12) {
    const int cl = ntt_cluster_for<LOGN>(cluster);
    if constexpr (LOGN >= 13) {
      if (cl == 4) return launch_inv_c<LOGN, 4, AR>(L, jobs, st);
      if (cl == 8) return launch_inv_c<LOGN, 8, AR>(L, jobs, st);
    }
    if (cl == 2 || LOGN == 15) return launch_inv_c<LOGN, 2, AR>(L, jobs, st);
  }
  if constexpr (LOGN <= 14) return launch_inv_c<LOGN, 1, AR>(L, jobs, st);
  return fail("unsupported cluster size");
}
template <int LOGN> static int launch_inv_t(const NttLaunch &L, size_t jobs, cudaStream_t st, bool fold, int cluster) {
  return fold ? launch_inv_a<LOGN, 1>(L, jobs, st, cluster) : launch_inv_a<LOGN, 0>(L, jobs, st, cluster);
}

// bytes of a seeded launch's c1 tile: [ell][2 threads] words
static size_t seed_tile_bytes(int ell, int threads) { return (size_t)ell * 2 * threads * sizeof(u64); }
// the largest dynamic shared memory a seeded instance needs on a context of k primes (ell = k - 1), allowed once per device and
// never lowered (contexts of different k share the device).  The 128-thread k_rot_wsum_ip tile stays under the 48 KB default for
// every k <= 24 (47 104 bytes at ell = 23); the 256-thread k_ks_inner and k_rot_many tiles pass it from ell = 13
template <class Kern> static int seed_smem_allow(Kern kern, size_t bytes) {
  if (bytes <= 48 * 1024) return 0;
  cudaFuncAttributes fa;
  CUDA_OK(cudaFuncGetAttributes(&fa, kern));
  if ((size_t)fa.maxDynamicSharedSizeBytes < bytes) CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}
static int seeded_smem_opt_in(int k) {
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  const size_t b = seed_tile_bytes(k - 1, 256);
  if (seed_smem_allow(k_ks_inner<false, false, true>, b) || seed_smem_allow(k_ks_inner<false, true, true>, b) ||
      seed_smem_allow(k_ks_inner<true, false, true>, b) || seed_smem_allow(k_ks_inner<true, true, true>, b) ||
      seed_smem_allow(k_rot_many<false, true, true>, b) || seed_smem_allow(k_rot_many<true, true, true>, b) ||
      seed_smem_allow(k_ks_inner<true, false, true, true>, b) || seed_smem_allow(k_ks_inner<true, true, true, true>, b) ||
      seed_smem_allow(k_rot_many<true, true, true, true>, b))
    return 1;
  static_assert(24 * 2 * 128 * sizeof(u64) <= 48 * 1024, "the k_rot_wsum_ip seeded tile fits the default shared memory");
  return 0;
}

struct CudaBE {
  const evab_ctx *c;
  cudaStream_t st;
  int error(const char *m) { return fail(m); }
  bool hoist_inline() const { return g_inline; }
  bool key_seeded() const { return g_seeded; }
  bool key_bank() const { return g_bank.tenant != nullptr; }
  // cached c1 rows: checked by require_c1_rows (seeded keys and a key-bank table), so the C1 instances are bank instances only
  bool key_c1_rows() const { return g_bank.c1 != nullptr; }
  // dynamic shared memory of a seeded launch (the c1 tile, SeedTileDev); the instances whose tile can pass the 48 KB default were
  // allowed their largest one when the context was created (seeded_smem_opt_in), so a launch -- or a graph capture -- sets nothing
  static size_t seed_smem(int ell, int threads) { return seed_tile_bytes(ell, threads); }
  void count(unsigned n = 1) const { c->launches.fetch_add(n, std::memory_order_relaxed); }
  dim3 grid(int rows, int per_thread = 2) const {
    int per_row = (int)(c->v.N / per_thread / 256);
    if (per_row < 1) per_row = 1;
    return dim3(per_row, rows, g_batch.batch);
  }
  int fwd(const NttLaunch &L, size_t jobs) {
    count();
    const bool fold = c->v.arith == 0 && ntt_launch_folds(L, jobs, c->v.foldmask);
    switch (c->v.logN) {
      case 10: return launch_fwd_t<10>(L, jobs, st, fold, c->ntt_cluster);
      case 11: return launch_fwd_t<11>(L, jobs, st, fold, c->ntt_cluster);
      case 12: return launch_fwd_t<12>(L, jobs, st, fold, c->ntt_cluster);
      case 13: return launch_fwd_t<13>(L, jobs, st, fold, c->ntt_cluster);
      case 14: return launch_fwd_t<14>(L, jobs, st, fold, c->ntt_cluster);
      case 15: return launch_fwd_t<15>(L, jobs, st, fold, c->ntt_cluster);
    }
    return fail("unsupported N");
  }
  int inv(const NttLaunch &L, size_t jobs) {
    count();
    const bool fold = c->v.arith == 0 && ntt_launch_folds(L, jobs, c->v.foldmask);
    switch (c->v.logN) {
      case 10: return launch_inv_t<10>(L, jobs, st, fold, c->ntt_cluster);
      case 11: return launch_inv_t<11>(L, jobs, st, fold, c->ntt_cluster);
      case 12: return launch_inv_t<12>(L, jobs, st, fold, c->ntt_cluster);
      case 13: return launch_inv_t<13>(L, jobs, st, fold, c->ntt_cluster);
      case 14: return launch_inv_t<14>(L, jobs, st, fold, c->ntt_cluster);
      case 15: return launch_inv_t<15>(L, jobs, st, fold, c->ntt_cluster);
    }
    return fail("unsupported N");
  }
  int dyadic(int op, const DyArgs &A) {
    count();
    dim3 g = grid(A.sout * A.ell, 4);
    switch (op) {
      case DY_ADD: k_dyadic<DY_ADD><<<g, 256, 0, st>>>(A, g_batch.stride); break;
      case DY_SUB: k_dyadic<DY_SUB><<<g, 256, 0, st>>>(A, g_batch.stride); break;
      case DY_NEG: k_dyadic<DY_NEG><<<g, 256, 0, st>>>(A, g_batch.stride); break;
      case DY_COPY: k_dyadic<DY_COPY><<<g, 256, 0, st>>>(A, g_batch.stride); break;
      default: k_mul_plain<<<grid(A.ell, 4), 256, 0, st>>>(A, g_batch.stride); break;   // one thread: the same coefficients of every polynomial
    }
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int sum(const SumArgs &A) {
    count();
    k_sum_terms<<<grid(A.sout * A.ell), 256, 0, st>>>(A, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int mulct(bool sq, const MulArgs &A) {
    count();
    if (sq) k_mul_ct<true><<<grid(A.ell), 256, 0, st>>>(A, g_batch.stride);
    else k_mul_ct<false><<<grid(A.ell), 256, 0, st>>>(A, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  template <bool BANK, bool C1 = false> void inner_seeded(dim3 g, const IpArgs &A, bool inl) {
    if (inl) k_ks_inner<BANK, true, true, C1><<<g, 256, seed_smem(A.ell, 256), st>>>(A, g_batch.stride, g_bank);
    else k_ks_inner<BANK, false, true, C1><<<g, 256, seed_smem(A.ell, 256), st>>>(A, g_batch.stride, g_bank);
  }
  int inner(const IpArgs &A) {
    count();
    const dim3 g = grid(A.ell + 1);
    const bool inl = g_inline && A.cadd;   // only the hoisted form has a constant to form
    if (g_seeded) {
      if (g_bank.c1) inner_seeded<true, true>(g, A, inl);
      else if (g_bank.tenant) inner_seeded<true>(g, A, inl);
      else inner_seeded<false>(g, A, inl);
    }
    else if (g_bank.tenant) { if (inl) k_ks_inner<true, true, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank); else k_ks_inner<true, false, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank); }
    else if (inl) k_ks_inner<false, true, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank);
    else k_ks_inner<false, false, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int scale_c0(const u64 *c0, u64 *ext, int ell) {
    count();
    k_scale_c0<<<grid(ell, 1), 256, 0, st>>>(c0, ext, c->v.primes, ell, c->v.k, (int)c->v.N, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int rot_many(const RotManyArgs &A) {
    count();
    const dim3 g = grid(A.n * (A.ell + 1));
    if (g_seeded) {   // inline constants (require_seeded_inline)
      if (g_bank.c1) k_rot_many<true, true, true, true><<<g, 256, seed_smem(A.ell, 256), st>>>(A, g_batch.stride, g_bank);
      else if (g_bank.tenant) k_rot_many<true, true, true><<<g, 256, seed_smem(A.ell, 256), st>>>(A, g_batch.stride, g_bank);
      else k_rot_many<false, true, true><<<g, 256, seed_smem(A.ell, 256), st>>>(A, g_batch.stride, g_bank);
    }
    else if (g_bank.tenant) { if (g_inline) k_rot_many<true, true, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank); else k_rot_many<true, false, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank); }
    else if (g_inline) k_rot_many<false, true, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank);
    else k_rot_many<false, false, false><<<g, 256, 0, st>>>(A, g_batch.stride, g_bank);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  template <int NOUT> void wsum_ip(dim3 g, const WsumIpArgs &A, bool bank) {
    if (g_seeded) {   // inline constants (require_seeded_inline)
      if (g_bank.c1) k_rot_wsum_ip<NOUT, true, true, true, true><<<g, 128, seed_smem(A.ell, 128), st>>>(A, g_batch.stride, g_bank);
      else if (bank) k_rot_wsum_ip<NOUT, true, true, true><<<g, 128, seed_smem(A.ell, 128), st>>>(A, g_batch.stride, g_bank);
      else k_rot_wsum_ip<NOUT, false, true, true><<<g, 128, seed_smem(A.ell, 128), st>>>(A, g_batch.stride, g_bank);
    }
    else if (bank) { if (g_inline) k_rot_wsum_ip<NOUT, true, true, false><<<g, 128, 0, st>>>(A, g_batch.stride, g_bank); else k_rot_wsum_ip<NOUT, true, false, false><<<g, 128, 0, st>>>(A, g_batch.stride, g_bank); }
    else if (g_inline) k_rot_wsum_ip<NOUT, false, true, false><<<g, 128, 0, st>>>(A, g_batch.stride, g_bank);
    else k_rot_wsum_ip<NOUT, false, false, false><<<g, 128, 0, st>>>(A, g_batch.stride, g_bank);
  }
  int rot_wsum_ip(const WsumIpArgs &A) {
    count();
    const dim3 g(A.N / 2 / 128, A.ell + 1, g_batch.batch);   // N >= 1024
    const bool bank = g_bank.tenant != nullptr;
    switch (A.nout) {
      case 1: wsum_ip<1>(g, A, bank); break;
      case 2: wsum_ip<2>(g, A, bank); break;
      case 3: wsum_ip<3>(g, A, bank); break;
      case 4: wsum_ip<4>(g, A, bank); break;
      default: return fail("rotate_wsum: 1..4 output sums");
    }
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int rot_wsum(const WsumArgs &A) {
    count();
    k_rot_wsum<<<grid(2 * A.ell), 256, 0, st>>>(A, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int lazy_rotsum(const LazyRotSumArgs &A) {
    count();
    const dim3 g(A.N / 64, A.ell + 1, g_batch.batch), b(32, A.n);
    if (g_bank.tenant) k_lazy_rotsum<true><<<g, b, 0, st>>>(A, g_batch.stride, g_bank);
    else k_lazy_rotsum<false><<<g, b, 0, st>>>(A, g_batch.stride, g_bank);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int hoist_indicator(u64 *out, const u32 *ctab, int N, int rows) {
    count();
    k_hoist_indicator<<<dim3((N + 255) / 256, rows), 256, 0, st>>>(out, ctab, N);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int hoist_const(const HoistConstArgs &A) {
    count();
    k_hoist_const<<<dim3((A.N / 2 + 255) / 256, A.ell + 1), 256, 0, st>>>(A);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int hoist_levels(const HoistLevelsArgs &A, int n) {
    if (n > 65535) return fail("hoist constants: at most 65535 keys per call");
    count();
    k_hoist_const_levels<<<dim3((A.N / 2 + 255) / 256, A.k, n), 256, 0, st>>>(A);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int dec_compose(const DecArgs &A) { count(); k_dec_compose<<<(A.N + 255) / 256, 256, 0, st>>>(A); CUDA_OK(cudaGetLastError()); return 0; }
  int dec_fft(const DecArgs &A, u32 m) { count(); k_dec_fft<<<(A.N / 2 + 255) / 256, 256, 0, st>>>(A, m); CUDA_OK(cudaGetLastError()); return 0; }
  int dec_gather(const DecArgs &A) { count(); k_dec_gather<<<(A.N / 2 + 255) / 256, 256, 0, st>>>(A); CUDA_OK(cudaGetLastError()); return 0; }
  int enc_scatter(const EncBatch &B) {
    count();
    k_enc_scatter<<<dim3((B.N / 2 + 255) / 256, B.count, g_batch.batch), 256, 0, st>>>(B, g_batch.stride, g_batch.vstride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int enc_fft(const EncBatch &B, u32 g, int ns) {
    count();
    k_enc_fft<<<dim3((B.N / 8 + 255) / 256, B.count, g_batch.batch), 256, 0, st>>>(B, g, ns, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int enc_uniform(const EncUniform &B) {
    count();
    k_enc_uniform<<<dim3((B.N / 2 + 255) / 256, B.count * B.ell, g_batch.batch), 256, 0, st>>>(B, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  int enc_round(const EncBatch &B) {
    count();
    k_enc_round<<<dim3((B.N + 255) / 256, B.count, g_batch.batch), 256, 0, st>>>(B, g_batch.stride);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
};

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------
static void ctx_free(evab_ctx *c) {
  for (auto &kv : c->perms) cudaFree(kv.second);
  for (auto &kv : c->cperms) cudaFree(kv.second);
  cudaFree(c->d_tw); cudaFree(c->d_primes); cudaFree(c->d_qinv); cudaFree(c->d_qinv_f); cudaFree(c->d_halfmod); cudaFree(c->d_zeros);
  cudaFree(c->d_roots); cudaFree(c->d_slot); cudaFree(c->d_pow2);
  delete c;
}
// device copy of a host table; on failure the caller frees the whole context (no leak on any error path)
template <class T> static int to_device(T **dst, const T *src, size_t n) {
  CUDA_OK(cudaMalloc(dst, n * sizeof(T)));
  CUDA_OK(cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}
static int ctx_build(evab_ctx *c, uint64_t N, int logN, const uint64_t *primes, int k) {
  const size_t tw_elems = (size_t)k * 4 * N;   // Shoup rows + fold rows (host_tables.hpp)
  CUDA_OK(cudaMalloc(&c->d_tw, tw_elems * sizeof(u64x2)));
  evab_host::Tables T;
  const char *err = evab_host::build_tables(N, logN, primes, k, c->d_tw, T);
  if (err[0]) return fail(std::string("evab_ctx_create: ") + err);
  CUDA_OK(cudaMemcpy(c->d_tw, T.tw.data(), tw_elems * sizeof(u64x2), cudaMemcpyHostToDevice));
  if (to_device(&c->d_primes, T.pd.data(), (size_t)k)) return 1;
  if (to_device(&c->d_qinv, T.qinv.data(), T.qinv.size())) return 1;
  if (to_device(&c->d_qinv_f, T.qinv_f.data(), T.qinv_f.size())) return 1;
  if (to_device(&c->d_halfmod, T.halfmod.data(), T.halfmod.size())) return 1;
  CUDA_OK(cudaMalloc(&c->d_zeros, 32 * sizeof(u64)));
  CUDA_OK(cudaMemset(c->d_zeros, 0, 32 * sizeof(u64)));
  if (to_device(&c->d_roots, reinterpret_cast<const cplx *>(T.roots.data()), (size_t)N)) return 1;
  if (to_device(&c->d_slot, T.slot_index.data(), (size_t)N)) return 1;
  if (to_device(&c->d_pow2, T.pow2.data(), T.pow2.size())) return 1;
  c->v.roots = c->d_roots; c->v.slot_index = c->d_slot; c->v.pow2 = c->d_pow2;
  c->v.N = N; c->v.logN = logN; c->v.k = k;
  c->v.primes = c->d_primes; c->v.qinv = c->d_qinv; c->v.qinv_f = c->d_qinv_f; c->v.halfmod = c->d_halfmod; c->v.zeros = c->d_zeros;
  c->v.foldmask = T.foldmask;
  c->fold_host = T.fp; c->v.fold_host = c->fold_host.data();
  c->v.arith = getenv("EVAB_NTT_SHOUP") ? 1 : 0;
  return 0;
}
extern "C" int evab_ctx_create(uint64_t N, const uint64_t *primes, int k, int device, evab_ctx **out) {
  if (!out) return fail("evab_ctx_create: null out");
  *out = nullptr;
  int logN = 0;
  while ((1ull << logN) < N) logN++;
  if ((1ull << logN) != N || logN < 10 || logN > 15) return fail("evab_ctx_create: N must be a power of two in [2^10, 2^15]");
  if (k < 1 || k > 24) return fail("evab_ctx_create: prime count must be in [1,24]");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("evab_ctx_create: no CUDA device (this backend has no CPU fallback)");
  if (device < 0 || device >= ndev) return fail("evab_ctx_create: bad device index");
  CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  cudaMemPool_t pool;
  CUDA_OK(cudaDeviceGetDefaultMemPool(&pool, device));
  unsigned long long thresh = ~0ull;  // keep freed blocks cached in the pool
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);

  evab_ctx *c = new evab_ctx();
  c->device = device; c->sms = prop.multiProcessorCount;
  c->ntt_cluster = g_ntt_cluster.load();
  c->primes.assign(primes, primes + k);
  if (ctx_build(c, N, logN, primes, k)) { ctx_free(c); return 1; }   // g_err is set; every partial allocation is released
  if (k >= 2 && seeded_smem_opt_in(k)) { ctx_free(c); return 1; }
  *out = c;
  return 0;
}
extern "C" void evab_ctx_destroy(evab_ctx *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  ctx_free(c);
}
// per-context tuning knobs (no process-global state): CTAs per residue, NTT arithmetic
extern "C" int evab_ctx_set_ntt_cluster(evab_ctx *c, int cl) {
  if (cl != 0 && cl != 1 && cl != 2 && cl != 4 && cl != 8) return fail("evab_ctx_set_ntt_cluster: 0 (automatic), 1, 2, 4 or 8 CTAs per residue");
  c->ntt_cluster = cl;
  return 0;
}
extern "C" int evab_ctx_set_ntt_arith(evab_ctx *c, int mode) {
  if (mode != 0 && mode != 1) return fail("evab_ctx_set_ntt_arith: 0 (two-row fold where the primes allow it) or 1 (lazy Shoup everywhere)");
  c->v.arith = mode;
  return 0;
}
extern "C" unsigned evab_ctx_foldmask(const evab_ctx *c) { return c->v.foldmask; }
extern "C" uint64_t evab_ctx_N(const evab_ctx *c) { return c->v.N; }
extern "C" int evab_ctx_k(const evab_ctx *c) { return c->v.k; }
extern "C" int evab_ctx_device(const evab_ctx *c) { return c->device; }
extern "C" int evab_ctx_sm_count(const evab_ctx *c) { return c->sms; }
extern "C" int evab_mem_info(evab_ctx *c, size_t *free_bytes, size_t *total_bytes) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMemGetInfo(free_bytes, total_bytes));
  return 0;
}

extern "C" int evab_malloc(evab_ctx *c, size_t bytes, void **p, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMallocAsync(p, bytes ? bytes : 8, S(stream)));
  return 0;
}
extern "C" int evab_free(evab_ctx *c, void *p, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaFreeAsync(p, S(stream)));
  return 0;
}
extern "C" int evab_upload(evab_ctx *c, void *d, const void *h, size_t bytes, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, S(stream)));
  return 0;
}
extern "C" int evab_upload_2d(evab_ctx *c, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyHostToDevice, S(stream)));
  return 0;
}
extern "C" int evab_download(evab_ctx *c, void *h, const void *d, size_t bytes, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, S(stream)));
  return 0;
}
extern "C" int evab_host_alloc(size_t bytes, void **p) {
  CUDA_OK(cudaHostAlloc(p, bytes ? bytes : 8, cudaHostAllocPortable));
  return 0;
}
extern "C" int evab_host_free(void *p) {
  CUDA_OK(cudaFreeHost(p));
  return 0;
}
extern "C" int evab_sync(evab_ctx *c, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaStreamSynchronize(S(stream)));
  return 0;
}
extern "C" int evab_stream_create(evab_ctx *c, void **stream) {
  CUDA_OK(cudaSetDevice(c->device));
  cudaStream_t s;
  CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *stream = (void *)s;
  return 0;
}
extern "C" int evab_stream_destroy(evab_ctx *c, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaStreamDestroy(S(stream)));
  return 0;
}
extern "C" int evab_event_create(evab_ctx *c, void **event) {
  CUDA_OK(cudaSetDevice(c->device));
  cudaEvent_t e;
  CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  *event = (void *)e;
  return 0;
}
extern "C" int evab_event_destroy(evab_ctx *c, void *event) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaEventDestroy((cudaEvent_t)event));
  return 0;
}
extern "C" int evab_event_record(evab_ctx *c, void *event, void *stream) {
  CUDA_OK(cudaEventRecord((cudaEvent_t)event, S(stream)));
  return 0;
}
extern "C" int evab_stream_wait_event(evab_ctx *c, void *stream, void *event) {
  CUDA_OK(cudaStreamWaitEvent(S(stream), (cudaEvent_t)event, 0));
  return 0;
}
extern "C" int evab_graph_begin(evab_ctx *c, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaStreamBeginCapture(S(stream), cudaStreamCaptureModeThreadLocal));
  return 0;
}
extern "C" int evab_graph_end(evab_ctx *c, void *stream, void **graph_exec) {
  cudaGraph_t g = nullptr;
  CUDA_OK(cudaStreamEndCapture(S(stream), &g));
  cudaGraphExec_t ge = nullptr;
  cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  if (e != cudaSuccess) return fail(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
  *graph_exec = (void *)ge;
  return 0;
}
extern "C" int evab_graph_launch(evab_ctx *c, void *graph_exec, void *stream) {
  CUDA_OK(cudaGraphLaunch((cudaGraphExec_t)graph_exec, S(stream)));
  return 0;
}
extern "C" int evab_graph_destroy(evab_ctx *c, void *graph_exec) {
  CUDA_OK(cudaGraphExecDestroy((cudaGraphExec_t)graph_exec));
  return 0;
}
extern "C" uint64_t evab_launch_count(const evab_ctx *c) { return c->launches.load(); }

// ---------------------------------------------------------------------------
// ops
// ---------------------------------------------------------------------------
#define BE_BEGIN                         \
  CUDA_OK(cudaSetDevice(c->device));     \
  CudaBE be{c, S(stream)};

extern "C" int evab_ntt_fwd(evab_ctx *c, uint64_t *d, size_t count, const int *pidx, int np, void *stream) {
  BE_BEGIN return ntt_batch_impl(be, c->v, false, d, count, pidx, np);
}
extern "C" int evab_ntt_inv(evab_ctx *c, uint64_t *d, size_t count, const int *pidx, int np, void *stream) {
  BE_BEGIN return ntt_batch_impl(be, c->v, true, d, count, pidx, np);
}
extern "C" int evab_set_ntt_cluster(int cl) {
  if (cl != 0 && cl != 1 && cl != 2 && cl != 4 && cl != 8) return fail("evab_set_ntt_cluster: 0 (automatic), 1, 2, 4 or 8 CTAs per residue");
  g_ntt_cluster.store(cl);   // default of contexts created from now on; existing contexts keep theirs
  return 0;
}
extern "C" int evab_encode_uniform(evab_ctx *c, int count, const double *values, const double *scales, int ell, uint64_t *out, void *stream) {
  BE_BEGIN return encode_uniform_impl(be, c->v, count, values, scales, ell, out);
}
extern "C" int evab_encode_uniform_ext(evab_ctx *c, int count, const double *values, const double *scales, int ell, int with_p, uint64_t *out, void *stream) {
  BE_BEGIN return encode_uniform_impl(be, c->v, count, values, scales, ell, out, with_p);
}
extern "C" int evab_encode_ext(evab_ctx *c, int count, const double *const *vals, const uint32_t *vec, const double *scales, int ell, int with_p,
                               uint64_t *out, void *work, void *stream) {
  BE_BEGIN return encode_impl(be, c->v, count, vals, vec, scales, ell, out, (cplx *)work, with_p);
}
extern "C" size_t evab_encode_work_bytes(const evab_ctx *c, int count) { return encode_work_bytes(c->v, count); }
extern "C" int evab_encode(evab_ctx *c, int count, const double *const *vals, const uint32_t *vec, const double *scales, int ell,
                           uint64_t *out, void *work, void *stream) {
  BE_BEGIN return encode_impl(be, c->v, count, vals, vec, scales, ell, out, (cplx *)work);
}
extern "C" size_t evab_decode_work_bytes(const evab_ctx *c, int ell) { return decode_tmp_elems(c->v, ell) * sizeof(u64) + (size_t)c->v.N * sizeof(cplx); }
extern "C" int evab_decode(evab_ctx *c, int ell, const uint64_t *pt, double scale, double *d_out, void *work, void *stream) {
  u64 *tmp = (u64 *)work;
  cplx *cw = (cplx *)(tmp + decode_tmp_elems(c->v, ell));
  BE_BEGIN return decode_impl(be, c->v, ell, c->primes.data(), pt, scale, d_out, tmp, cw);
}
extern "C" int evab_add(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *b, int sb, void *stream) {
  BE_BEGIN return dyadic_impl<DY_ADD>(be, c->v, ell, o, a, sa, b, sb, 0);
}
extern "C" int evab_sub(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *b, int sb, void *stream) {
  BE_BEGIN return dyadic_impl<DY_SUB>(be, c->v, ell, o, a, sa, b, sb, 0);
}
extern "C" int evab_add_plain(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt, void *stream) {
  BE_BEGIN return dyadic_impl<DY_ADD>(be, c->v, ell, o, a, sa, pt, 1, 1);
}
extern "C" int evab_sub_plain(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt, void *stream) {
  BE_BEGIN return dyadic_impl<DY_SUB>(be, c->v, ell, o, a, sa, pt, 1, 1);
}
extern "C" int evab_negate(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, void *stream) {
  BE_BEGIN return dyadic_impl<DY_NEG>(be, c->v, ell, o, a, sa, (const u64 *)nullptr, 0, 0);
}
extern "C" int evab_mul_plain(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, const uint64_t *pt, void *stream) {
  BE_BEGIN return dyadic_impl<DY_MULPT>(be, c->v, ell, o, a, sa, pt, 1, 1);
}
extern "C" int evab_sum_terms(evab_ctx *c, int ell, uint64_t *o, int n, const uint64_t *const *cts, const int *sizes, const uint64_t *const *pts, void *stream) {
  BE_BEGIN return sum_terms_impl(be, c->v, ell, o, n, cts, sizes, pts);
}
extern "C" int evab_sum_products(evab_ctx *c, int ell, uint64_t *o, int n, const uint64_t *const *cts, const int *sizes, const uint64_t *const *seconds, const int *kinds,
                                 void *stream) {
  BE_BEGIN return sum_terms_impl(be, c->v, ell, o, n, cts, sizes, seconds, kinds);
}
extern "C" int evab_mul(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *b, void *stream) {
  BE_BEGIN return mulct_impl(be, c->v, false, ell, o, a, b);
}
extern "C" int evab_square(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, void *stream) {
  BE_BEGIN return mulct_impl(be, c->v, true, ell, o, a, (const u64 *)nullptr);
}
extern "C" int evab_mod_switch(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, void *stream) {
  if (ell < 2 || ell > c->v.k) return fail("mod_switch needs 2 <= ell <= k");
  BE_BEGIN return copy_impl(be, c->v, ell, ell - 1, o, a, sa);
}
extern "C" int evab_copy(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, void *stream) {
  BE_BEGIN return copy_impl(be, c->v, ell, ell, o, a, sa);
}
extern "C" size_t evab_rescale_work_bytes(const evab_ctx *c, int sa) { return rescale_work_elems(c->v, sa) * sizeof(u64); }
extern "C" int evab_rescale(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, int sa, void *work, void *stream) {
  BE_BEGIN return rescale_impl(be, c->v, ell, o, a, sa, (u64 *)work);
}
extern "C" size_t evab_keyswitch_work_bytes(const evab_ctx *c, int ell) { return keyswitch_work_elems(c->v, ell) * sizeof(u64); }
extern "C" int evab_relinearize(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *key, void *work, void *stream) {
  BE_BEGIN return relinearize_impl(be, c->v, ell, o, a, key, (u64 *)work);
}
extern "C" uint64_t evab_galois_elt_from_step(uint64_t N, int steps) { return evab_host::galois_elt_from_step(N, steps); }
extern "C" int evab_galois_prepare(evab_ctx *c, uint64_t elt) {
  if (!(elt & 1) || elt >= 2 * c->v.N) return fail("galois element must be odd and < 2N");
  std::lock_guard<std::mutex> g(c->mu);
  if (c->perms.count(elt)) return 0;
  CUDA_OK(cudaSetDevice(c->device));
  std::vector<u32> tab;
  evab_host::galois_table(c->v.N, c->v.logN, elt, tab);
  u32 *d = nullptr;
  CUDA_OK(cudaMalloc(&d, tab.size() * sizeof(u32)));
  CUDA_OK(cudaMemcpy(d, tab.data(), tab.size() * sizeof(u32), cudaMemcpyHostToDevice));
  c->perms[elt] = d;
  evab_host::galois_coeff_table(c->v.N, elt, tab);
  u32 *dc = nullptr;
  CUDA_OK(cudaMalloc(&dc, tab.size() * sizeof(u32)));
  CUDA_OK(cudaMemcpy(dc, tab.data(), tab.size() * sizeof(u32), cudaMemcpyHostToDevice));
  c->cperms[elt] = dc;
  return 0;
}
extern "C" int evab_rotate_prepare(evab_ctx *c, int ell, uint64_t *hoist, const uint64_t *a, void *stream) {
  BE_BEGIN return rotate_prepare_impl(be, c->v, ell, hoist, a);
}
extern "C" int evab_rotate_prepared(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *hoist, uint64_t elt, const uint64_t *key, void *work,
                                    void *stream) {
  u32 *perm = nullptr, *ctab = nullptr;
  {
    std::lock_guard<std::mutex> g(c->mu);
    auto it = c->perms.find(elt);
    if (it == c->perms.end()) return fail("evab_rotate_prepared: call evab_galois_prepare(elt) first");
    perm = it->second; ctab = c->cperms.at(elt);
  }
  BE_BEGIN return rotate_prepared_impl(be, c->v, ell, o, a, hoist, perm, ctab, key, (u64 *)work);
}
static int galois_tables(evab_ctx *c, uint64_t elt, u32 **perm, u32 **ctab, const char *who) {
  std::lock_guard<std::mutex> g(c->mu);
  auto it = c->perms.find(elt);
  if (it == c->perms.end()) return fail(std::string(who) + ": call evab_galois_prepare(elt) first");
  *perm = it->second; *ctab = c->cperms.at(elt);
  return 0;
}
extern "C" size_t evab_rotate_modup_work_bytes(const evab_ctx *c, int ell) { return rotate_modup_work_elems(c->v, ell) * sizeof(u64); }
extern "C" size_t evab_rotate_modup_ext_bytes(const evab_ctx *c, int ell) { return (size_t)(ell + 1) * ell * c->v.N * sizeof(u64); }
extern "C" size_t evab_hoist_const_bytes(const evab_ctx *c, int ell) { return hoist_const_elems(c->v, ell) * sizeof(u64); }
extern "C" int evab_rotate_modup_prepare(evab_ctx *c, int ell, uint64_t *that, uint64_t *ext, const uint64_t *a, uint64_t *zflag, void *stream) {
  BE_BEGIN return rotate_modup_prepare_impl(be, c->v, ell, that, ext, a, zflag);
}
extern "C" int evab_rotate_hoist_const(evab_ctx *c, int ell, uint64_t elt, const uint64_t *key, uint64_t *out, uint64_t *tmp, void *stream) {
  u32 *perm = nullptr, *ctab = nullptr;
  if (galois_tables(c, elt, &perm, &ctab, "evab_rotate_hoist_const")) return 1;
  BE_BEGIN return hoist_const_impl(be, c->v, ell, ctab, key, out, tmp);
}
extern "C" size_t evab_seeded_key_bytes(const evab_ctx *c) { return seeded_key_words(c->v.k, c->v.N) * sizeof(u64); }
extern "C" size_t evab_hoist_indicators_bytes(const evab_ctx *c, int n) { return hoist_indicators_elems(c->v, n) * sizeof(u64); }
extern "C" int evab_hoist_indicators(evab_ctx *c, int n, const uint64_t *elts, uint64_t *out, void *stream) {
  if (n < 1) return fail("evab_hoist_indicators: n must be >= 1");
  std::vector<const u32 *> ctabs(n);
  for (int g = 0; g < n; g++) {
    u32 *perm = nullptr, *ctab = nullptr;
    if (galois_tables(c, elts[g], &perm, &ctab, "evab_hoist_indicators")) return 1;
    ctabs[g] = ctab;
  }
  BE_BEGIN return hoist_indicators_impl(be, c->v, n, ctabs.data(), out);
}
extern "C" size_t evab_hoist_const_levels_bytes(const evab_ctx *c) { return hoist_levels_words(c->v.k, c->v.N) * sizeof(u64); }
extern "C" size_t evab_rotate_hoist_const_levels_work_bytes(const evab_ctx *c, int n) { return hoist_const_levels_work_elems(c->v, n) * sizeof(u64); }
extern "C" int evab_rotate_hoist_const_levels(evab_ctx *c, int n, const uint64_t *elts, const uint64_t *keys, uint64_t *out, uint64_t *tmp, void *stream) {
  if (n < 1) return fail("evab_rotate_hoist_const_levels: n must be >= 1");
  std::vector<const u32 *> ctabs(n);
  for (int g = 0; g < n; g++) {
    u32 *perm = nullptr, *ctab = nullptr;
    if (galois_tables(c, elts[g], &perm, &ctab, "evab_rotate_hoist_const_levels")) return 1;
    ctabs[g] = ctab;
  }
  BE_BEGIN return hoist_const_levels_impl(be, c->v, n, ctabs.data(), keys, out, tmp);
}
extern "C" int evab_rotate_modup_prepared(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, const uint64_t *ext, uint64_t elt, const uint64_t *key,
                                          const uint64_t *cadd, void *work, void *stream) {
  u32 *perm = nullptr, *ctab = nullptr;
  if (galois_tables(c, elt, &perm, &ctab, "evab_rotate_modup_prepared")) return 1;
  BE_BEGIN return rotate_modup_prepared_impl(be, c->v, ell, o, a, ext, perm, key, cadd, (u64 *)work);
}
extern "C" int evab_rotate_modup_scale_c0(evab_ctx *c, int ell, uint64_t *ext, const uint64_t *a, void *stream) {
  BE_BEGIN return rotate_modup_scale_c0_impl(be, c->v, ell, ext, a);
}
extern "C" size_t evab_rotate_modup_many_work_bytes(const evab_ctx *c, int ell, int n) { return rotate_modup_many_work_elems(c->v, ell, n) * sizeof(u64); }
extern "C" int evab_rotate_modup_many(evab_ctx *c, int ell, int n, uint64_t *o, const uint64_t *a, const uint64_t *ext, const uint64_t *elts,
                                      const uint64_t *const *keys, const uint64_t *const *cadds, void *work, void *stream) {
  if (n < 1 || n > ROTMANY_MAX) return fail("evab_rotate_modup_many: 1..16 rotations");
  const u32 *perms[ROTMANY_MAX];
  for (int i = 0; i < n; i++) {
    u32 *perm = nullptr, *ctab = nullptr;
    if (galois_tables(c, elts[i], &perm, &ctab, "evab_rotate_modup_many")) return 1;
    perms[i] = perm;
  }
  BE_BEGIN return rotate_modup_many_impl(be, c->v, ell, n, o, a, ext, perms, keys, cadds, (u64 *)work);
}
extern "C" size_t evab_lazy_rotsum_work_bytes(const evab_ctx *c, int ell, int nout) { return lazy_rotsum_work_elems(c->v, ell, nout) * sizeof(u64); }
extern "C" int evab_lazy_rotsum(evab_ctx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts,
                                const uint64_t *const *keys, const uint64_t *const *cadds, const uint64_t *const *wts, void *work, void *stream) {
  if (n < 1 || n > LRS_MAX) return fail("evab_lazy_rotsum: 1..16 rotations");
  const u32 *perms[LRS_MAX];
  for (int i = 0; i < n; i++) {
    u32 *perm = nullptr, *ctab = nullptr;
    if (galois_tables(c, elts[i], &perm, &ctab, "evab_lazy_rotsum")) return 1;
    perms[i] = perm;
  }
  BE_BEGIN return lazy_rotsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, (u64 *)work);
}
extern "C" size_t evab_rotate_wsum_work_bytes(const evab_ctx *c, int ell, int n, int nout) { return rotate_wsum_work_elems(c->v, ell, n, nout) * sizeof(u64); }
extern "C" int evab_rotate_wsum(evab_ctx *c, int ell, int nout, uint64_t *o, const uint64_t *a, const uint64_t *ext, int n, const uint64_t *elts,
                                const uint64_t *const *keys, const uint64_t *const *cadds, const uint64_t *const *wts, int ntap,
                                const uint64_t *const *taps, const uint64_t *const *twts, void *work, void *stream) {
  if (n < 1 || n > WS_MAX) return fail("evab_rotate_wsum: 1..16 rotations");
  const u32 *perms[WS_MAX];
  for (int i = 0; i < n; i++) {
    u32 *perm = nullptr, *ctab = nullptr;
    if (galois_tables(c, elts[i], &perm, &ctab, "evab_rotate_wsum")) return 1;
    perms[i] = perm;
  }
  BE_BEGIN return rotate_wsum_impl(be, c->v, ell, nout, o, a, ext, n, perms, keys, cadds, wts, ntap, taps, twts, (u64 *)work);
}
extern "C" int evab_memset_zero(evab_ctx *c, void *d, size_t bytes, void *stream) {
  CUDA_OK(cudaSetDevice(c->device));
  CUDA_OK(cudaMemsetAsync(d, 0, bytes, S(stream)));
  return 0;
}
extern "C" int evab_rotate(evab_ctx *c, int ell, uint64_t *o, const uint64_t *a, uint64_t elt, const uint64_t *key, void *work, void *stream) {
  u32 *perm = nullptr;
  {
    std::lock_guard<std::mutex> g(c->mu);
    auto it = c->perms.find(elt);
    if (it == c->perms.end()) return fail("evab_rotate: call evab_galois_prepare(elt) first");
    perm = it->second;
  }
  BE_BEGIN return rotate_impl(be, c->v, ell, o, a, perm, key, (u64 *)work);
}
extern "C" int evab_expand_key_uniform(evab_ctx *c, int n, const uint8_t *seeds, const uint64_t *moduli, uint64_t *keys, void *stream) {
  if (n < 1 || n > 65535) return fail("evab_expand_key_uniform: n must be in [1, 65535]");
  if (c->v.k < 2 || c->v.k > KX_MAXK) return fail("evab_expand_key_uniform: 2 <= k <= 64 primes");
  if (!moduli) return fail("evab_expand_key_uniform: no moduli");
  ExpandArgs A{};
  A.seeds = reinterpret_cast<const uint32_t *>(seeds); A.keys = keys; A.N = (uint32_t)c->v.N; A.k = (uint32_t)c->v.k;
  for (int m = 0; m < c->v.k; m++) {
    if (moduli[m] < 2) return fail("evab_expand_key_uniform: every modulus must be >= 2");
    A.q[m] = moduli[m]; A.lim[m] = kx_limit(moduli[m]);
  }
  CUDA_OK(cudaSetDevice(c->device));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  k_expand_uniform<<<dim3((A.N / 8 + 255) / 256, (A.k - 1) * A.k, n), 256, 0, S(stream)>>>(A);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int evab_expand_seeded_c1(evab_ctx *c, int n, const uint64_t *images, uint64_t *rows, void *stream) {
  if (n < 1 || n > 65535) return fail("evab_expand_seeded_c1: n must be in [1, 65535]");
  if (!images || !rows) return fail("evab_expand_seeded_c1: d_images and d_rows must not be null");
  if (c->v.k < 2) return fail("evab_expand_seeded_c1: seeded keys need k >= 2 primes");
  if (reinterpret_cast<uintptr_t>(images) % 64 || reinterpret_cast<uintptr_t>(rows) % 64)
    return fail("evab_expand_seeded_c1: d_images and d_rows must be 64-byte aligned");
  CUDA_OK(cudaSetDevice(c->device));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  k_expand_seeded_c1<<<dim3(((unsigned)c->v.N / 8 + 255) / 256, (c->v.k - 1) * c->v.k, n), 256, 0, S(stream)>>>(images, rows, c->v.primes, c->v.k, (int)c->v.N);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int evab_expand_cipher_uniform(evab_ctx *c, int n, const uint8_t *seeds, uint64_t *const *c1, const int *ell, const uint64_t *moduli, void *stream) {
  if (n < 1 || n > 65535) return fail("evab_expand_cipher_uniform: n must be in [1, 65535]");
  if (!seeds) return fail("evab_expand_cipher_uniform: h_seeds is null");
  if (!c1) return fail("evab_expand_cipher_uniform: h_c1 is null");
  if (!ell) return fail("evab_expand_cipher_uniform: h_ell is null");
  if (!moduli) return fail("evab_expand_cipher_uniform: h_moduli is null");
  if (c->v.k < 2 || c->v.k > KX_MAXK) return fail("evab_expand_cipher_uniform: 2 <= k <= 64 primes");
  int maxEll = 0;
  for (int i = 0; i < n; i++) {
    if (ell[i] < 1 || ell[i] > c->v.k - 1)
      return fail("evab_expand_cipher_uniform: h_ell[" + std::to_string(i) + "] must be in [1, k-1] (k = " + std::to_string(c->v.k) + ")");
    if (!c1[i]) return fail("evab_expand_cipher_uniform: h_c1[" + std::to_string(i) + "] is null");
    if (reinterpret_cast<uintptr_t>(c1[i]) % 16) return fail("evab_expand_cipher_uniform: h_c1[" + std::to_string(i) + "] is not 16-byte aligned");
    maxEll = std::max(maxEll, ell[i]);
  }
  CipherExpandArgs A{};
  A.N = (uint32_t)c->v.N;
  for (int m = 0; m < maxEll; m++) {
    if (moduli[m] < 2) return fail("evab_expand_cipher_uniform: every modulus in h_moduli must be >= 2");
    A.q[m] = moduli[m]; A.lim[m] = kx_limit(moduli[m]);
  }
  CUDA_OK(cudaSetDevice(c->device));
  // the entries travel by value in the launch arguments (no device table to keep alive): CX_MAX_ENTRIES per launch, in order on
  // the caller's stream
  for (int i0 = 0; i0 < n; i0 += CX_MAX_ENTRIES) {
    const int nb = std::min(CX_MAX_ENTRIES, n - i0);
    int rows = 0;
    for (int b = 0; b < nb; b++) {
      std::memcpy(A.e[b].seed, seeds + (size_t)32 * (i0 + b), 32);
      A.e[b].c1 = c1[i0 + b]; A.e[b].ell = (uint32_t)ell[i0 + b];
      rows = std::max(rows, ell[i0 + b]);
    }
    c->launches.fetch_add(1, std::memory_order_relaxed);
    k_expand_cipher_uniform<<<dim3((A.N / 8 + 255) / 256, rows, nb), 256, 0, S(stream)>>>(A);
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}
extern "C" int evab_gather_ciphers(evab_ctx *c, int n, const uint64_t *const *src, uint64_t *const *dst, const uint64_t *words, void *stream) {
  if (n < 0) return fail("evab_gather_ciphers: n must be >= 0");
  if (!src) return fail("evab_gather_ciphers: h_src is null");
  if (!dst) return fail("evab_gather_ciphers: h_dst is null");
  if (!words) return fail("evab_gather_ciphers: h_words is null");
  for (int i = 0; i < n; i++) {
    const std::string at = "[" + std::to_string(i) + "]";
    if (!src[i] || reinterpret_cast<uintptr_t>(src[i]) % 16) return fail("evab_gather_ciphers: h_src" + at + " is null or not 16-byte aligned");
    if (!dst[i] || reinterpret_cast<uintptr_t>(dst[i]) % 16) return fail("evab_gather_ciphers: h_dst" + at + " is null or not 16-byte aligned");
    if (words[i] % 2) return fail("evab_gather_ciphers: h_words" + at + " must be even (16-byte vectors)");
  }
  CUDA_OK(cudaSetDevice(c->device));
  // in order on the caller's stream, GW_MAX_ENTRIES entries per launch
  for (int i0 = 0; i0 < n; i0 += GW_MAX_ENTRIES) {
    const int nb = std::min(GW_MAX_ENTRIES, n - i0);
    GatherArgs A{};
    u64 vecs = 0;
    for (int b = 0; b < nb; b++) {
      A.e[b].src = reinterpret_cast<const u64x2 *>(src[i0 + b]);
      A.e[b].dst = reinterpret_cast<u64x2 *>(dst[i0 + b]);
      A.e[b].vecs = words[i0 + b] / 2;
      vecs = std::max(vecs, A.e[b].vecs);
    }
    const u64 tiles = std::max<u64>(1, std::min<u64>((vecs + GW_THREADS * GW_UNROLL - 1) / (GW_THREADS * GW_UNROLL), 65535));
    c->launches.fetch_add(1, std::memory_order_relaxed);
    k_gather_words<<<dim3((unsigned)tiles, nb), GW_THREADS, 0, S(stream)>>>(A);
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

// ---- compact responses
extern "C" size_t evab_compact_work_bytes(const evab_ctx *c, int n, int ell) {
  return n < 1 || ell < 1 ? 0 : (size_t)2 * n * ell * c->v.N * sizeof(u64);
}
extern "C" int evab_compact_ciphers(evab_ctx *c, int n, const uint64_t *const *src, uint64_t *const *dst, int ell, int shift, int bits, void *work,
                                    void *stream) {
  if (n < 0 || n > 32767) return fail("evab_compact_ciphers: n must be in [0, 32767]");
  if (!src) return fail("evab_compact_ciphers: h_src is null");
  if (!dst) return fail("evab_compact_ciphers: h_dst is null");
  if (ell < 1 || ell > DEC_MAX_ELL || ell > c->v.k) return fail("evab_compact_ciphers: ell must be in [1, min(8, k)]");
  if (bits < 1 || bits > 62) return fail("evab_compact_ciphers: bits must be in [1, 62]");
  if (shift < bits) return fail("evab_compact_ciphers: shift must be >= bits");
  if (!work || reinterpret_cast<uintptr_t>(work) % 16) return fail("evab_compact_ciphers: d_work is null or not 16-byte aligned");
  for (int i = 0; i < n; i++) {
    const std::string at = "[" + std::to_string(i) + "]";
    if (!src[i] || reinterpret_cast<uintptr_t>(src[i]) % 16) return fail("evab_compact_ciphers: h_src" + at + " is null or not 16-byte aligned");
    if (!dst[i] || reinterpret_cast<uintptr_t>(dst[i]) % 8) return fail("evab_compact_ciphers: h_dst" + at + " is null or not 8-byte aligned");
  }
  if (n == 0) return 0;
  const size_t N = c->v.N, rows = (size_t)2 * ell * N;
  // 1. the ciphertexts side by side in d_work
  std::vector<uint64_t *> to(n);
  std::vector<uint64_t> words(n, rows);
  for (int i = 0; i < n; i++) to[i] = (uint64_t *)work + i * rows;
  if (int rc = evab_gather_ciphers(c, n, src, to.data(), words.data(), stream)) return rc;
  // 2. coefficient form: one transform of the 2 n ell rows (the call's own batch of one, whatever evab_set_batch says)
  {
    const BatchState saved = g_batch;
    g_batch = BatchState();
    int pidx[DEC_MAX_ELL];
    for (int i = 0; i < ell; i++) pidx[i] = i;
    int rc;
    { BE_BEGIN rc = ntt_batch_impl(be, c->v, true, (u64 *)work, (size_t)2 * n * ell, pidx, ell); }
    g_batch = saved;
    if (rc) return rc;
  }
  // 3. CRT of x' = 2^(shift-bits) x mod Q, exact rounding, packing
  CompactArgs A;
  compact_args(A, c->primes.data(), ell, shift, bits, (u32)N);
  A.primes = c->v.primes;
  CUDA_OK(cudaSetDevice(c->device));
  for (int i0 = 0; i0 < n; i0 += CMP_MAX_ENTRIES) {
    const int nb = std::min(CMP_MAX_ENTRIES, n - i0);
    A.src = (const u64 *)work + i0 * rows;
    for (int b = 0; b < nb; b++) A.dst[b] = dst[i0 + b];
    c->launches.fetch_add(1, std::memory_order_relaxed);
    k_compact<<<dim3((A.words + CMP_THREADS - 1) / CMP_THREADS, 2, nb), CMP_THREADS, 0, S(stream)>>>(A);
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}
extern "C" int evab_compact_unpack(evab_ctx *c, const uint64_t *words, int bits, int nres, uint64_t *out, void *stream) {
  if (!words || !out) return fail("evab_compact_unpack: d_words and d_out must not be null");
  if (bits < 1 || bits > 62) return fail("evab_compact_unpack: bits must be in [1, 62]");
  if (nres < 1 || nres > DEC_MAX_ELL || nres > c->v.k) return fail("evab_compact_unpack: nres must be in [1, min(8, k)]");
  const u32 N = (u32)c->v.N;
  CUDA_OK(cudaSetDevice(c->device));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  k_compact_unpack<<<(N + 255) / 256, 256, 0, S(stream)>>>(words, (u32)bits, (u32)(((u64)N * bits + 63) / 64), c->v.primes, (u32)nres, N, out);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int evab_compact_finish(evab_ctx *c, const uint64_t *coef, int nres, int bits, int nout, uint64_t *out, int64_t *z, void *stream) {
  if (!coef || !out) return fail("evab_compact_finish: d_coef and d_out must not be null");
  if (bits < 1 || bits > 62) return fail("evab_compact_finish: bits must be in [1, 62]");
  if (nres < 1 || nres > DEC_MAX_ELL || nres > c->v.k) return fail("evab_compact_finish: nres must be in [1, min(8, k)]");
  if (nout < 1 || nout > DEC_MAX_ELL || nout > c->v.k) return fail("evab_compact_finish: nout must be in [1, min(8, k)]");
  CrtTables T;
  crt_tables(T, c->primes.data(), nres);
  const u32 N = (u32)c->v.N;
  CUDA_OK(cudaSetDevice(c->device));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  k_compact_finish<<<(N + 255) / 256, 256, 0, S(stream)>>>(T, c->v.primes, (u32)nres, N, (u32)bits, coef, (u32)nout, out, (long long *)z);
  CUDA_OK(cudaGetLastError());
  return 0;
}
