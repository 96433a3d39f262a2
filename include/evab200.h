/*
 * evab200.h -- C-ABI of the H100-native (sm_90a) CKKS evaluator that replaces the
 * Microsoft SEAL calls made by microsoft/EVA's executor.
 *
 * The reference has no FFI for this path: eva/seal/seal_executor.h calls
 * seal::Evaluator / seal::CKKSEncoder directly (SURVEY.md section 8b).  This
 * header is the boundary a maintainer would bind instead; every entry point
 * names the reference call site it replaces.  Plain pointers and sizes only;
 * all `u64*` arguments named d_* are DEVICE pointers, `stream` is a
 * cudaStream_t passed as void* (NULL = default stream).  All calls enqueue
 * work and return immediately unless stated; return 0 on success, non-zero on
 * error with a message available from evab_last_error() (thread-local).  No
 * exceptions cross this boundary.  There is NO CPU fallback: without a CUDA
 * device evab_ctx_create fails.
 *
 * Layouts (identical to seal::Ciphertext::data() etc., SURVEY.md 8a T1-T3):
 *   ciphertext   u64 [size][ell][N]       NTT form, values in [0, q_i)
 *   plaintext    u64 [ell][N]             NTT form
 *   kswitch key  u64 [k-1][2][k][N]       (digit, component, key-level residue)
 * k = number of primes incl. the special key-switching prime (last);
 * EVA level j has ell = k-1-j residues (seal_executor.h:221-224).
 */
#ifndef EVAB200_H
#define EVAB200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct evab_ctx evab_ctx;

const char *evab_last_error(void);
int evab_version(void);

/* Replaces seal::SEALContext construction (eva/seal/seal.cpp:148-172,179-184):
 * builds NTT tables (minimal primitive 2N-th root per prime), Barrett/Shoup
 * constants and RNS divide-and-round constants for every level on `device`.
 * `primes` are the k moduli in SEAL order (last = special prime). N = 2^10..2^15. */
int evab_ctx_create(uint64_t N, const uint64_t *primes, int k, int device, evab_ctx **out);
void evab_ctx_destroy(evab_ctx *ctx);
uint64_t evab_ctx_N(const evab_ctx *ctx);
int evab_ctx_k(const evab_ctx *ctx);
int evab_ctx_device(const evab_ctx *ctx);
/* number of SMs of the context's device (grid sizing for callers/benchmarks) */
int evab_ctx_sm_count(const evab_ctx *ctx);
/* free / total device memory in bytes (the host layer bounds the number of concurrent plan replicas with it) */
int evab_mem_info(evab_ctx *ctx, size_t *free_bytes, size_t *total_bytes);

/* ---- device memory (stream-ordered pool) and transfers ---- */
int evab_malloc(evab_ctx *ctx, size_t bytes, void **d_ptr, void *stream);
int evab_free(evab_ctx *ctx, void *d_ptr, void *stream);
int evab_upload(evab_ctx *ctx, void *d_dst, const void *h_src, size_t bytes, void *stream);
/* `height` rows of `width` bytes, row i from h_src + i * spitch to d_dst + i * dpitch (one strided copy: the c0 rows of
 * compressed keys into their places in the key layout) */
int evab_upload_2d(evab_ctx *ctx, void *d_dst, size_t dpitch, const void *h_src, size_t spitch, size_t width, size_t height, void *stream);
int evab_download(evab_ctx *ctx, void *h_dst, const void *d_src, size_t bytes, void *stream);
int evab_sync(evab_ctx *ctx, void *stream); /* blocks the calling thread */
/* page-locked host memory for ciphertext / plaintext buffers that cross the boundary: uploads and
 * downloads from it are truly asynchronous and run at full PCIe rate (replaces the seal::Ciphertext
 * heap buffers copied at reference seal.cpp:104-122) */
int evab_host_alloc(size_t bytes, void **h_ptr);
int evab_host_free(void *h_ptr);

/* ---- scheduler glue: streams, events and CUDA-graph capture.  These replace
 * the Galois worklist + atomics of MulticoreProgramTraversal::forwardPass
 * (eva/common/multicore_program_traversal.h:24-84): independent DAG terms are
 * enqueued on different streams, dependencies become events, and a whole
 * execute() can be captured once and replayed as one graph launch. ---- */
int evab_stream_create(evab_ctx *ctx, void **stream);
int evab_stream_destroy(evab_ctx *ctx, void *stream);
int evab_event_create(evab_ctx *ctx, void **event);            /* timing disabled */
int evab_event_destroy(evab_ctx *ctx, void *event);
int evab_event_record(evab_ctx *ctx, void *event, void *stream);
int evab_stream_wait_event(evab_ctx *ctx, void *stream, void *event);
/* begin/end capture on `stream` (other streams join through event waits);
 * end returns an executable graph handle */
int evab_graph_begin(evab_ctx *ctx, void *stream);
int evab_graph_end(evab_ctx *ctx, void *stream, void **graph_exec);
int evab_graph_launch(evab_ctx *ctx, void *graph_exec, void *stream);
int evab_graph_destroy(evab_ctx *ctx, void *graph_exec);
/* Batched issue (thread-local): until reset with batch = 1, every op enqueued by this
 * thread is applied to `batch` independent instances laid out at a fixed distance:
 * instance b uses every ciphertext / plaintext / workspace device pointer shifted by
 * b * stride_words (u64 words) and every evab_encode value pointer shifted by
 * b * value_stride (doubles); keys and tables are shared.  One fat launch replaces
 * `batch` launches (horizontal fusion across program instances, SURVEY.md 8f-3). */
int evab_set_batch(int batch, size_t stride_words, size_t value_stride);
/* Per-instance keys (thread-local, next to evab_set_batch): until reset with NULL, every
 * key pointer and hoist-constant pointer that the relinearize / rotate / rotate_prepared /
 * rotate_modup_prepared / rotate_modup_many / rotate_wsum / lazy_rotsum kernels read is,
 * for batch instance b, shifted by d_tenant_of_instance[b] * tenant_stride_words (u64
 * words).  The caller passes tenant 0's pointers of a key bank whose tenants share one
 * layout.  The table is device memory read when the kernels run, so a captured graph
 * follows a table rewritten (stream-ordered) before its launch. */
int evab_set_key_bank(const int32_t *d_tenant_of_instance, size_t tenant_stride_words);
/* Inline hoist constants, thread-local like evab_set_key_bank (on != 0: on).  While on, the d_cadd / d_cadds[i] arguments of
 * evab_rotate_modup_prepared, evab_rotate_modup_many and evab_rotate_wsum are read as the Galois element's indicator rows
 * [k][N] (evab_hoist_indicators) instead of its hoist constant, the constant being formed inside the key-switch inner product
 * from the key rows it loads (same bits); those rows are shared by all tenants of a key bank and are NOT shifted by the
 * key-bank offset.  evab_lazy_rotsum fails while it is on. */
int evab_set_hoist_inline(int on);
/* Seeded keys, thread-local like evab_set_key_bank (on != 0: on).  While on, the d_key / d_keys[i] arguments of
 * evab_relinearize, evab_rotate, evab_rotate_prepared, evab_rotate_modup_prepared, evab_rotate_modup_many and evab_rotate_wsum
 * point at seeded key images of evab_seeded_key_bytes bytes: the key's [k-1][k][N] c0 rows, then its 32-byte seed padded to 64
 * bytes.  The c1 rows are never stored: the key-switch inner products draw them from the seed by the rule of
 * eva_b200/csrc/key_expand.cuh (the words evab_expand_key_uniform writes), so the outputs are those of the expanded key.  The
 * key-bank offset moves the whole image.  The hoisted calls need evab_set_hoist_inline on; evab_lazy_rotsum,
 * evab_rotate_hoist_const and evab_rotate_hoist_const_levels fail while it is on. */
int evab_set_key_seeded(int on);
size_t evab_seeded_key_bytes(const evab_ctx *ctx);
/* Cached c1 rows, thread-local like evab_set_key_bank (null: off).  d_region_of_instance is a device table of one int32 per batch
 * instance, read by the kernels at run time (a captured graph follows a rewritten table): instance b with region r = table[b] >= 0
 * reads the c1 rows of every key it switches with from key operand + r * tenant_stride_words, where key i's c1 rows [k-1][k][N]
 * sit at the word offset of its c0 rows in a seeded image (evab_expand_seeded_c1 writes them); an instance with r < 0 draws them
 * from the seed.  The outputs are the same either way.  Valid only while evab_set_key_seeded is on and a key-bank table is set:
 * otherwise the key-switch calls fail, naming the missing setting. */
int evab_set_key_c1_rows(const int32_t *d_region_of_instance);
/* the c1 rows of the n consecutive seeded images at d_images (evab_seeded_key_bytes apart) -> d_rows, in the geometry above: image
 * i's row (J, m) at d_rows + i * evab_seeded_key_bytes / 8 + (J k + m) N words (the 8 seed words of every image are not written).
 * Both pointers 64-byte aligned; device memory; stream-ordered */
int evab_expand_seeded_c1(evab_ctx *ctx, int n, const uint64_t *d_images, uint64_t *d_rows, void *stream);
/* number of kernel launches issued through this context so far */
uint64_t evab_launch_count(const evab_ctx *ctx);

/* ---- negacyclic NTT / iNTT (microbenchmark entry, BASELINE config 2) ----
 * d_data holds `count` residue polynomials of N coefficients; polynomial r is
 * transformed in place modulo primes[prime_idx[r % nprimes]].  Semantics:
 * seal::util::ntt_negacyclic_harvey / inverse_ntt_negacyclic_harvey
 * (out[i] = a(psi^(2*bitrev(i)+1)), canonical output; SURVEY Appendix A.3). */
int evab_ntt_fwd(evab_ctx *ctx, uint64_t *d_data, size_t count, const int *prime_idx, int nprimes, void *stream);
int evab_ntt_inv(evab_ctx *ctx, uint64_t *d_data, size_t count, const int *prime_idx, int nprimes, void *stream);

/* Tuning knob (process-wide): spread every residue transform of 4096 <= N <= 16384 over a thread-block
 * cluster of 1, 2, 4 or 8 CTAs (distributed shared memory exchange), capped so that a CTA keeps at least
 * 128 threads; 0 (default) = that cap.  Results are identical. */
int evab_set_ntt_cluster(int ctas_per_residue);   /* default for contexts created afterwards */
/* The same knob per context (no process-global state on the op path), and the NTT arithmetic:
 * 0 (default) = "two-row fold" butterflies (5 wide multiplies) in every launch whose primes are all
 * SEAL-style 60-bit primes p = 2^60 - delta, delta < 2^25 (evab_ctx_foldmask: bit i = prime i qualifies),
 * lazy Shoup butterflies otherwise; 1 = lazy Shoup everywhere.  Results are identical bit for bit. */
int evab_ctx_set_ntt_cluster(evab_ctx *ctx, int ctas_per_residue);
int evab_ctx_set_ntt_arith(evab_ctx *ctx, int mode);
unsigned evab_ctx_foldmask(const evab_ctx *ctx);

/* ---- CKKS encoder on the device: seal::CKKSEncoder::encode at seal_executor.h:242
 * (and seal.cpp:68,80).  Encodes `count` vectors in one batch: vector e has
 * vec_sizes[e] doubles at d_values[e] (device), is replicated over the N/2 slots
 * and encoded at absolute scale scales[e] into d_out[e][ell][N] (NTT form).
 * h_* arguments are host arrays read during the call.  d_work:
 * evab_encode_work_bytes(ctx, count) bytes (FP64 FFT buffer + one flag word per vector:
 * vectors that encode to a constant polynomial -- scalar constants -- skip the NTT,
 * their transform is the constant itself). ---- */
size_t evab_encode_work_bytes(const evab_ctx *ctx, int count);
int evab_encode(evab_ctx *ctx, int count, const double *const *h_d_values, const uint32_t *h_vec_sizes, const double *h_scales,
                int ell, uint64_t *d_out, void *d_work, void *stream);
/* The same encoder for vectors whose elements are all equal (every scalar constant of an EVA program,
 * constant_value.h:64-71): encodes h_values[e] replicated over all slots at scale h_scales[e] into
 * d_out[e][ell][N].  All FFT butterflies are exact for equal inputs, so the result -- the constant
 * polynomial round(value * scale), whose NTT is that constant -- is bit-identical to evab_encode of the
 * replicated vector, in one launch and without workspace. */
int evab_encode_uniform(evab_ctx *ctx, int count, const double *h_values, const double *h_scales, int ell, uint64_t *d_out, void *stream);

/* ---- evaluator ops; one per SEAL call site of eva/seal/seal_executor.h ----
 * `ell` = residues of the inputs' level.  Outputs must not alias inputs unless
 * stated.  Sizes: sa/sb in {2,3}. */
/* Evaluator::add :124 / sub :140 -- out size = max(sa,sb); may alias a or b */
int evab_add(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, const uint64_t *d_b, int sb, void *stream);
int evab_sub(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, const uint64_t *d_b, int sb, void *stream);
/* Evaluator::add_plain :127 / sub_plain :143 -- out size = sa; may alias a */
int evab_add_plain(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, const uint64_t *d_pt, void *stream);
int evab_sub_plain(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, const uint64_t *d_pt, void *stream);
/* Evaluator::negate :194 -- may alias */
int evab_negate(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, void *stream);
/* Evaluator::multiply_plain :168 -- may alias a */
int evab_mul_plain(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, const uint64_t *d_pt, void *stream);
/* A chain of Evaluator::multiply_plain :168 and Evaluator::add :124 calls in one pass:
 * out = sum_t (h_d_pts[t] ? cts[t] * pts[t] : cts[t]), 1 <= nterms <= 32, out size = max size.
 * Products are accumulated in 128 bits and reduced once: the canonical result is identical to
 * performing the calls one by one.  h_* are host arrays of device pointers read during the call. */
int evab_sum_terms(evab_ctx *ctx, int ell, uint64_t *d_out, int nterms, const uint64_t *const *h_d_cts, const int *h_sizes,
                   const uint64_t *const *h_d_pts, void *stream);
/* The same with ciphertext products among the terms: h_kinds[t] = 0 (cts[t]), 1 (cts[t] * plaintext
 * h_d_seconds[t], multiply_plain :168) or 2 (cts[t] (x) ciphertext h_d_seconds[t], both of size 2: the
 * size-3 result of Evaluator::multiply :164 / square :162).  A sum of products -- e.g. the reduction of
 * the wide test DAGs -- never materialises the individual products. */
int evab_sum_products(evab_ctx *ctx, int ell, uint64_t *d_out, int nterms, const uint64_t *const *h_d_cts, const int *h_sizes,
                      const uint64_t *const *h_d_seconds, const int *h_kinds, void *stream);
/* Evaluator::multiply :164 (2x2 -> 3) and square :162 */
int evab_mul(evab_ctx *ctx, int ell, uint64_t *d_out3, const uint64_t *d_a2, const uint64_t *d_b2, void *stream);
int evab_square(evab_ctx *ctx, int ell, uint64_t *d_out3, const uint64_t *d_a2, void *stream);
/* Evaluator::rescale_to_next :213 -- [sa][ell][N] -> [sa][ell-1][N].
 * d_work: evab_rescale_work_bytes(ctx, sa) bytes of scratch. */
size_t evab_rescale_work_bytes(const evab_ctx *ctx, int sa);
int evab_rescale(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, void *d_work, void *stream);
/* plain copy of a ciphertext (rotate_vector by 0 steps) */
int evab_copy(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, void *stream);
/* Evaluator::mod_switch_to_next :206 -- drop the last residue */
int evab_mod_switch(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, int sa, void *stream);
/* Evaluator::relinearize :200 (size 3 -> 2) and rotate_vector :181,188.
 * d_key: key-switch key for relinearisation / for galois_elt, layout above.
 * d_work: evab_keyswitch_work_bytes(ctx, ell) bytes of scratch. */
size_t evab_keyswitch_work_bytes(const evab_ctx *ctx, int ell);
int evab_relinearize(evab_ctx *ctx, int ell, uint64_t *d_out2, const uint64_t *d_a3, const uint64_t *d_key, void *d_work, void *stream);
/* Galois element of rotate_vector(steps) (steps>0 left; SEAL GaloisTool::get_elt_from_step) */
uint64_t evab_galois_elt_from_step(uint64_t N, int steps);
/* builds and caches the permutation tables of galois_elt on the device (NTT domain and signed
 * coefficient domain; blocking); must be called once before evab_rotate* uses that element */
int evab_galois_prepare(evab_ctx *ctx, uint64_t galois_elt);
int evab_rotate(evab_ctx *ctx, int ell, uint64_t *d_out2, const uint64_t *d_a2, uint64_t galois_elt, const uint64_t *d_key, void *d_work, void *stream);
/* Rotations of the SAME ciphertext share the inverse NTT of its c1 (the automorphism commutes with
 * the transform; SEAL recomputes it inside every rotate_vector :181,:188).  evab_rotate_prepare
 * writes it to d_hoist [ell][N]; evab_rotate_prepared(…, d_hoist, …) then equals evab_rotate bit
 * for bit with ell fewer transforms.  Same workspace as evab_rotate; ell <= 15. */
int evab_rotate_prepare(evab_ctx *ctx, int ell, uint64_t *d_hoist, const uint64_t *d_a, void *stream);
int evab_rotate_prepared(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, const uint64_t *d_hoist, uint64_t galois_elt,
                         const uint64_t *d_key, void *d_work, void *stream);
/* Rotations of the same ciphertext also share the MOD-UP of its c1, exactly (SEAL decomposes sigma_g(c1) inside every
 * rotate_vector :181,:188; the digit of the rotated ciphertext reduced to an output modulus m equals the NTT-domain permutation
 * of the unrotated extended digit plus (q_J mod m) * NTT_m(indicator of the negated coefficients), a term that depends on the
 * Galois key only -- eva_b200/csrc/ops_impl.hpp "hoisted_modup").
 *   evab_rotate_modup_prepare : d_that [ell][N] = iNTT(c1), d_ext [ell+1][ell][N] = the extended digits, once per ciphertext;
 *                               *d_zflag |= 1 when a digit holds a zero coefficient: the identity above then does not hold
 *                               (negate(0) = 0) and the caller must use evab_rotate / evab_rotate_prepared for that ciphertext.
 *   evab_rotate_hoist_const   : d_cadd [2][ell+1][N] for (galois_elt, key, ell), once per key and level; d_tmp (ell+1)*N words.
 *   evab_rotate_modup_prepared: == evab_rotate bit for bit, with ell*ell + ell fewer transforms (10 instead of 26 at ell = 4).
 * ell <= 15. */
size_t evab_rotate_modup_ext_bytes(const evab_ctx *ctx, int ell);
size_t evab_rotate_modup_work_bytes(const evab_ctx *ctx, int ell);
size_t evab_hoist_const_bytes(const evab_ctx *ctx, int ell);
int evab_rotate_modup_prepare(evab_ctx *ctx, int ell, uint64_t *d_that, uint64_t *d_ext, const uint64_t *d_a, uint64_t *d_zflag, void *stream);
int evab_rotate_hoist_const(evab_ctx *ctx, int ell, uint64_t galois_elt, const uint64_t *d_key, uint64_t *d_cadd, uint64_t *d_tmp, void *stream);
int evab_rotate_modup_prepared(evab_ctx *ctx, int ell, uint64_t *d_out, const uint64_t *d_a, const uint64_t *d_ext, uint64_t galois_elt,
                               const uint64_t *d_key, const uint64_t *d_cadd, void *d_work, void *stream);
/* evab_rotate_hoist_const of EVERY level ell = 1 .. k-1 for n Galois keys in one pass: d_keys holds the n keys back to back
 * ([n][k-1][2][k][N]; key g is for galois_elts[g], each prepared with evab_galois_prepare), d_out receives for key g the block
 * [ell = 1 .. k-1][2][ell+1][N] at g * evab_hoist_const_levels_bytes(ctx) / 8 words -- level ell's [2][ell+1][N] equals
 * evab_rotate_hoist_const(ell) bit for bit.  One batched forward transform of the n indicators over all k primes and one
 * element-wise launch that reads every key row once.  d_tmp: evab_rotate_hoist_const_levels_work_bytes(ctx, n) bytes (n k N
 * words).  Stream-ordered; does not synchronise.  k >= 2, n <= 65535. */
size_t evab_hoist_const_levels_bytes(const evab_ctx *ctx);
size_t evab_rotate_hoist_const_levels_work_bytes(const evab_ctx *ctx, int n);
int evab_rotate_hoist_const_levels(evab_ctx *ctx, int n, const uint64_t *galois_elts, const uint64_t *d_keys, uint64_t *d_out, uint64_t *d_tmp,
                                   void *stream);
/* The key-independent half of the hoist constants: d_out [n][k][N] receives NTT_m(I_g) for every prime m of the n Galois elements
 * (each prepared with evab_galois_prepare), I_g the indicator of the coefficients the automorphism negates -- the rows that
 * evab_rotate_hoist_const_levels multiplies by the key sums, and that evab_set_hoist_inline reads.  Stream-ordered. */
size_t evab_hoist_indicators_bytes(const evab_ctx *ctx, int n);
int evab_hoist_indicators(evab_ctx *ctx, int n, const uint64_t *galois_elts, uint64_t *d_out, void *stream);
/* Seed-compressed key-switch keys: a key whose c1 rows (the uniform halves) are not stored but expanded from a 32-byte seed by
 * the rule of eva_b200/csrc/key_expand.cuh (ChaCha20 blocks keyed by the seed, rejection sampling mod q; DESIGN §2).  Writes the
 * c1 rows of n keys d_keys [n][k-1][2][k][N]: row (J, m) of key g from the seed d_seeds[g] (device, [n][32] bytes) modulo
 * h_moduli[m] (host array of the k moduli, read during the call; the context's primes for real keys, any moduli >= 2 for
 * tests).  The c0 rows are not touched.  One launch; stream-ordered, does not synchronise.  1 <= n <= 65535, k <= 64. */
int evab_expand_key_uniform(evab_ctx *ctx, int n, const uint8_t *d_seeds, const uint64_t *h_moduli, uint64_t *d_keys, void *stream);
/* Seed-compressed input ciphertexts: the c1 rows of n fresh secret-key encryptions (c0, c1) = (-(a s + e) + m, a), expanded from
 * their 32-byte seeds by the same rule with the row ids 2^62 | m (key_expand.cuh; DESIGN §2).  Entry i writes the ell_i rows
 * [h_ell[i]][N] at h_c1[i] (a device pointer, 16-byte aligned: the c1 half of a ciphertext [2][ell_i][N] that starts ell_i N words
 * before) from h_seeds[i] (host, [n][32] bytes), row m modulo h_moduli[m] (host, >= max ell entries; the context's primes for real
 * ciphertexts, any moduli >= 2 for tests).  Nothing else is written.  The pointers are explicit: evab_set_batch does not apply.
 * All arrays are read during the call (the entries travel in the launch arguments, up to 56 per launch; larger n is split into
 * several launches on `stream`).  Stream-ordered, does not synchronise.  1 <= n <= 65535, 1 <= h_ell[i] <= k-1. */
int evab_expand_cipher_uniform(evab_ctx *ctx, int n, const uint8_t *h_seeds, uint64_t *const *h_c1, const int *h_ell, const uint64_t *h_moduli,
                               void *stream);
/* Server-resident ciphertexts: copy n device ranges, entry i the h_words[i] words at h_src[i] to h_dst[i] (device pointers, both
 * 16-byte aligned; h_words[i] even; the ranges of one call must not overlap a destination).  Nothing else is written.  The host
 * tables are read during the call (the entries travel in the launch arguments, up to 160 per launch; larger n is split into
 * several launches on `stream`), so a captured graph replays the copies as they were.  Stream-ordered, does not synchronise;
 * evab_set_batch does not apply.  n >= 0 (0: no launch); the tables must not be null. */
int evab_gather_ciphers(evab_ctx *ctx, int n, const uint64_t *const *h_src, uint64_t *const *h_dst, const uint64_t *h_words, void *stream);
/* Compact responses (compact_kernels.cuh; DESIGN §4): n size-2 ciphertexts [2][ell][N] in NTT form at h_src[i] (device, 16-byte
 * aligned), all with the same ell, switched to the modulus 2^bits and bit-packed into h_dst[i] (device, 8-byte aligned, [2][W] words,
 * W = ceil(N bits / 64)).  Every coefficient x of c0 and c1 becomes floor((2^(shift+1) x + Q) / (2Q)) mod 2^bits, exactly
 * (Q = q_0 ... q_{ell-1}).  d_work (16-byte aligned) holds evab_compact_work_bytes(ctx, n, ell) bytes: the coefficient form of the
 * n ciphertexts.  Launches: ceil(n / 160) gathers into d_work, one inverse transform of the 2 n ell rows and ceil(n / 256)
 * compactions, whatever the data.  The host tables are read during the call; evab_set_batch does not apply.  Stream-ordered, does
 * not synchronise.  0 <= n <= 32767 (0: no launch), 1 <= ell <= min(8, k), 1 <= bits <= 62, shift >= bits. */
size_t evab_compact_work_bytes(const evab_ctx *ctx, int n, int ell);
int evab_compact_ciphers(evab_ctx *ctx, int n, const uint64_t *const *h_src, uint64_t *const *h_dst, int ell, int shift, int bits, void *d_work,
                         void *stream);
/* The client side of a compact value [2][W] at d_words: evab_compact_unpack writes both polynomials' fields as residues modulo the
 * primes 0 .. nres-1, d_out [2][nres][N] in coefficient form.  evab_compact_finish takes y0 + y1 s in coefficient form over those
 * nres primes (d_coef [nres][N]; exact when their product exceeds 2 (N+1) 2^bits), reduces it mod 2^bits, centres it to
 * (-2^(bits-1), 2^(bits-1)] and writes that integer z as residues modulo the primes 0 .. nout-1 (d_out [nout][N], coefficient form)
 * and, if d_z is not null, as int64 values d_z [N].  1 <= nres, nout <= min(8, k), 1 <= bits <= 62.  Stream-ordered. */
int evab_compact_unpack(evab_ctx *ctx, const uint64_t *d_words, int bits, int nres, uint64_t *d_out, void *stream);
int evab_compact_finish(evab_ctx *ctx, const uint64_t *d_coef, int nres, int bits, int nout, uint64_t *d_out, int64_t *d_z, void *stream);
/* n <= 16 rotations of ONE ciphertext (seal::Evaluator::rotate_vector, seal_executor.h:176-189) in three kernel launches instead of
 * 3 n: d_out [n][2][ell][N], rotation i by galois_elts[i]; same bits as n calls of evab_rotate_modup_prepared.  d_ext, keys, cadds as there. */
/* evab_rotate_modup_many and evab_lazy_rotsum read P * c0 from the diagonal of d_ext (ext[m][J] has no entry for m = q_J): call this once
 * per ciphertext after evab_rotate_modup_prepare and before either of them.  evab_rotate_wsum does not need it (it reads c0 itself). */
int evab_rotate_modup_scale_c0(evab_ctx *ctx, int ell, uint64_t *d_ext, const uint64_t *d_a, void *stream);
size_t evab_rotate_modup_many_work_bytes(const evab_ctx *ctx, int ell, int n);
int evab_rotate_modup_many(evab_ctx *ctx, int ell, int n, uint64_t *d_out, const uint64_t *d_a, const uint64_t *d_ext, const uint64_t *galois_elts,
                           const uint64_t *const *d_keys, const uint64_t *const *d_cadds, void *d_work, void *stream);
/* Bit-exact weighted rotation sums: d_out [nout][2][ell][N], out_o = sum_i w_oi (.) rotate(x, g_i) + sum_t v_ot (.) c_t for n <= 16
 * rotations of ONE ciphertext x = d_a, nout <= 4 sums and ntap <= 16 size-2 ciphertexts c_t = d_taps[t] at level ell; the same bits as
 * rotate -> multiply_plain -> add (every rotation keeps its own rounding by P), in four launches and 2 n + 2 nout ell transforms instead of
 * n (2 + 2 ell).  Every weight is a SCALAR plaintext [ell][N] (the encoding of a replicated constant: one value per residue);
 * d_wts[o * n + i] weighs rotation i in sum o, d_twts[o * ntap + t] tap t, NULL for weight 0.  d_ext, keys, cadds as for
 * evab_rotate_modup_many; the diagonal of d_ext is not read. */
size_t evab_rotate_wsum_work_bytes(const evab_ctx *ctx, int ell, int n, int nout);
int evab_rotate_wsum(evab_ctx *ctx, int ell, int nout, uint64_t *d_out, const uint64_t *d_a, const uint64_t *d_ext, int n, const uint64_t *galois_elts,
                     const uint64_t *const *d_keys, const uint64_t *const *d_cadds, const uint64_t *const *d_wts, int ntap,
                     const uint64_t *const *d_taps, const uint64_t *const *d_twts, void *d_work, void *stream);
/* OPT-IN, NOT bit-exact (SURVEY 8f-4; graded by the reference's MSE criterion only): d_out [nout][2][ell][N],
 * out_o = sum_i w_oi (.) rotate(x, g_i) for n <= 16 rotations of ONE ciphertext x = d_a and nout <= 4 sets of plaintext weights, rounding
 * each weighted sum down by P ONCE instead of every rotation (2 + 2 ell transforms per sum instead of n (2 + 2 ell)); the key-switch
 * inner product of a rotation is shared by the sums it appears in.  d_ext: evab_rotate_modup_prepare of x; keys / cadds: per rotation
 * as for evab_rotate_modup_prepared; d_wts[o * n + i]: plaintext [ell+1][N] with the residue mod P as last row (evab_encode_ext /
 * evab_encode_uniform_ext with_p = 1), NULL when rotation i does not appear in sum o. */
size_t evab_lazy_rotsum_work_bytes(const evab_ctx *ctx, int ell, int nout);
int evab_lazy_rotsum(evab_ctx *ctx, int ell, int nout, uint64_t *d_out, const uint64_t *d_a, const uint64_t *d_ext, int n, const uint64_t *galois_elts,
                     const uint64_t *const *d_keys, const uint64_t *const *d_cadds, const uint64_t *const *d_wts, void *d_work, void *stream);
/* evab_encode / evab_encode_uniform with an extra last row: the residue mod the key-switch prime (with_p = 1: ell + 1 rows) */
int evab_encode_ext(evab_ctx *ctx, int count, const double *const *d_values, const uint32_t *h_vec_sizes, const double *h_scales, int ell, int with_p,
                    uint64_t *d_out, void *d_work, void *stream);
int evab_encode_uniform_ext(evab_ctx *ctx, int count, const double *h_values, const double *h_scales, int ell, int with_p, uint64_t *d_out, void *stream);
/* seal::CKKSEncoder::decode (seal.cpp:132-146): plaintext d_pt [ell][N] (NTT form) at absolute scale -> N/2 slot values
 * (doubles, device) -- inverse NTT, CRT composition to a centred multi-word integer, FP64 forward special FFT, all on the
 * device and bit-identical to the host / oracle decoders.  ell <= 8.  d_work: evab_decode_work_bytes(ctx, ell) bytes. */
size_t evab_decode_work_bytes(const evab_ctx *ctx, int ell);
int evab_decode(evab_ctx *ctx, int ell, const uint64_t *d_pt, double scale, double *d_out, void *d_work, void *stream);
/* stream-ordered zero fill (the executor clears its zero-coefficient flags at the start of every run) */
int evab_memset_zero(evab_ctx *ctx, void *d, size_t bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif
