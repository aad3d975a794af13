/* b200_bfv.h — layer-1 C ABI of the B200-native BFV backend ("slab" interface).
 *
 * Plain pointers and sizes only.  Every ciphertext argument is a dense device (or, for the *_host entry
 * points, host) array of uint64 words in the reference's own ciphertext word order
 *     data[((item * size + poly) * k + residue) * n + coeff]            (S/ciphertext.h:337,701-715)
 * key-switching keys use the reference's KSwitchKeys word order for one key list
 *     key[((J * 2 + comp) * (k_key) + residue) * n + coeff]             (S/kswitchkeys.h:340; NTT form)
 * `level` is the index in the modulus-switching chain: 0 = key level (all primes), 1 = first data level
 * (what SEALContext::first_parms_id() names), 2 = after one mod_switch_to_next, ...
 *
 * Each function replaces the arithmetic behind one reference entry point; the SEAL-named handle layer
 * (include/b200_sealc.h) is a thin wrapper over these:
 *   b200_multiply        Evaluator_Multiply        S/c/evaluator.cpp:218-243  -> Evaluator::bfv_multiply  S/evaluator.cpp:395-567
 *   b200_square          Evaluator_Square          S/c/evaluator.cpp          -> Evaluator::bfv_square    S/evaluator.cpp:864-1020
 *   b200_relinearize     Evaluator_Relinearize     S/c/evaluator.cpp:333      -> relinearize_internal     S/evaluator.cpp:1104-1159
 *   b200_apply_galois    Evaluator_ApplyGalois / RotateRows / RotateColumns   -> apply_galois_inplace     S/evaluator.cpp:2221-2323
 *   b200_apply_galois_add    apply_galois_inplace + add_inplace (one step of a rotate-and-sum reduction)
 *   b200_multiply_relin_sum  a chain of multiply + relinearize + add_inplace (encrypted inner products)
 *   b200_add/sub/negate  Evaluator_Add/Sub/Negate                             -> S/evaluator.cpp:130-350
 *   b200_multiply_plain  Evaluator_MultiplyPlain                              -> multiply_plain_normal    S/evaluator.cpp:1858-1992
 *   b200_plain_to_ntt    Evaluator_TransformToNTT1                            -> transform_to_ntt_inplace S/evaluator.cpp:2033-2124
 *   b200_multiply_plain_sum  a chain of multiply_plain + add_inplace (plaintext matrix x ciphertext vector)
 *   b200_apply_galois_many   apply_galois_inplace over items with their own element and key, one key switch
 *   b200_linear_transform    the baby-step giant-step chain of rotate_rows + multiply_plain + add_inplace (slot-wise matrix)
 *   b200_add_plain / b200_sub_plain   Evaluator_AddPlain/SubPlain             -> S/util/scalingvariant.cpp:69-188
 *   b200_mod_switch_to_next           Evaluator_ModSwitchToNext1              -> S/util/rns.cpp:801-840
 *   b200_ntt_forward / b200_ntt_inverse  (util level)                         -> S/util/ntt.cpp:393-474
 * All functions return 0 on success or a negative B200_E_* code; b200_last_error() gives the message.
 * There is NO CPU fallback: without a CUDA device every compute entry point fails with B200_E_CUDA.
 */
#ifndef B200_BFV_H
#define B200_BFV_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_E_INVALID (-1) /* invalid argument (reference: std::invalid_argument -> E_INVALIDARG) */
#define B200_E_LOGIC (-2)   /* invalid operation (reference: std::logic_error -> COR_E_INVALIDOPERATION) */
#define B200_E_CUDA (-3)    /* CUDA runtime/driver failure or no device */
#define B200_E_NULL (-4)    /* null pointer (reference: E_POINTER) */
#define B200_E_NOMEM (-5)

typedef struct b200_ctx b200_ctx;

typedef struct b200_info
{
    uint64_t n;
    uint64_t plain_modulus;
    int32_t key_primes;      /* K: primes at the key level */
    int32_t levels;          /* number of chain levels (key level included) */
    int32_t first_level;     /* 1 when key switching is available, else 0 */
    int32_t using_batching;
    int32_t device;
    int32_t sm_count;
} b200_info;

typedef struct b200_level_info
{
    int32_t k;               /* residues at this level */
    int32_t nB, nBsk;        /* BEHZ aux base sizes */
    uint64_t parms_id[4];    /* BLAKE2b-256 of (scheme, n, q_0.., t) — equals the reference's parms_id */
    uint64_t m_sk, gamma;
    uint64_t q[64];          /* the k primes */
    uint64_t bsk[66];        /* B primes then m_sk */
    uint64_t roots[64];      /* minimal primitive 2n-th roots of the k primes */
    uint64_t delta[64];      /* floor(Q/t) mod q_i */
    uint64_t q_mod_t;
} b200_level_info;

const char *b200_last_error(void);
int b200_device_count(void);

int b200_ctx_create(uint64_t poly_modulus_degree, const uint64_t *coeff_modulus, uint64_t coeff_modulus_count,
                    uint64_t plain_modulus, int device, b200_ctx **out);
void b200_ctx_destroy(b200_ctx *ctx);
int b200_ctx_info(const b200_ctx *ctx, b200_info *out);
int b200_ctx_level_info(const b200_ctx *ctx, int level, b200_level_info *out);
int b200_galois_elt_from_step(const b200_ctx *ctx, int steps, uint32_t *elt);

/* device memory helpers so that non-CUDA callers (Rust/C via FFI, Python via ctypes) can stage data */
int b200_malloc(b200_ctx *ctx, size_t bytes, void **dptr);
int b200_free(b200_ctx *ctx, void *dptr);
/* free ordered after the work already enqueued on `stream`; b200_malloc/b200_free use the stream-ordered pool, and
   b200_free requires that nothing still in flight uses the buffer */
int b200_free_async(b200_ctx *ctx, void *dptr, void *stream);
/* non-blocking streams for callers that overlap independent operations (the SEAL-named layer runs each calling thread's
   operations on its own) */
int b200_stream_create(b200_ctx *ctx, void **stream);
int b200_stream_destroy(b200_ctx *ctx, void *stream);
int b200_malloc_host(size_t bytes, void **hptr); /* pinned */
int b200_free_host(void *hptr);
int b200_memcpy_h2d(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream);
int b200_memcpy_d2h(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream);
int b200_memcpy_d2d(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream);
/* zero a device buffer (secret material is wiped before its memory returns to the pool; S/memorymanager.h clear_on_destruction) */
int b200_memzero(b200_ctx *ctx, void *dst, size_t bytes, void *stream);
int b200_stream_synchronize(b200_ctx *ctx, void *stream);

/* ---- NTT over a slab [items][k(level)][n], in place, canonical in -> canonical out ---- */
int b200_ntt_forward(b200_ctx *ctx, int level, uint64_t *data, uint64_t items, void *stream);
int b200_ntt_inverse(b200_ctx *ctx, int level, uint64_t *data, uint64_t items, void *stream);

/* negacyclic NTT modulo the plain modulus t over [items][n] (BatchEncoder encode = inverse, decode = forward) */
int b200_plain_ntt(b200_ctx *ctx, uint64_t *data, uint64_t items, int inverse, void *stream);

/* ---- slots in and out (BatchEncoder, S/batchencoder.cpp), batched; B200_E_INVALID when the parameters do not batch ---- */
/* values: device [items][count] (count <= n; NULL allowed when count == 0), read as int64_t when is_signed -> plain_out:
   device [items][n] coefficients mod t, the words of BatchEncoder_Encode1 (unsigned: each value reduced mod t) or
   BatchEncoder_Encode2 (signed: a negative x becomes t + x); slots at and beyond count are zero.  Multiply-ready operands:
   follow with b200_plain_to_ntt. */
int b200_batch_encode(b200_ctx *ctx, const uint64_t *values, uint64_t count, int is_signed, uint64_t *plain_out, uint64_t items,
                      void *stream);
/* plain: device [items][n] coefficient form (zero-padded, not modified) -> slots_out: device [items][n], uint64_t mod t
   (BatchEncoder_Decode1) or, with is_signed, int64_t centred v > t/2 ? v - t : v (BatchEncoder_Decode2) */
int b200_batch_decode(b200_ctx *ctx, const uint64_t *plain, int is_signed, uint64_t *slots_out, uint64_t items, void *stream);
/* b200_decrypt followed by b200_batch_decode, and with norm_out != NULL also b200_noise_norm, from one secret-key phase per
   call: slots_out device [batch][n]; norm_out HOST [batch][words] as b200_noise_norm fills it (the call then returns after
   completion; with norm_out == NULL it is asynchronous and `words` is not read) */
int b200_decrypt_slots(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, int is_signed,
                       uint64_t *slots_out, uint64_t *norm_out, int words, uint64_t batch, void *stream);

/* ---- encryption (S/encryptor.cpp), batched, in two steps.  The host step samples the random stream with the reference's
   generators (sampling.h): item i from Blake2xbPrng(seeds[i]), seeds HOST [batch][8], the items in parallel on the context's
   host threads (one item on the calling thread); it touches no device state.  Ternary and clipped-normal samples are int8.
   The device step is one launch sequence per call whatever the batch; it is asynchronous, and the host samples must stay
   unchanged until the stream has passed it (they are not wiped by the library: the caller owns them).  Device scratch that
   held u, e or products with the secret key is wiped in stream order.  Device memory: about 3 n + 24 k_e n bytes of scratch
   per pk item, 8 k n + n per sk item. ---- */
/* u, e0, e1 of each item in the order of Encryptor_EncryptReturnComponentsSetSeed: samples_out HOST [batch][3][n] */
int b200_sample_pk(b200_ctx *ctx, const uint64_t *seeds, int8_t *samples_out, uint64_t batch);
/* the public seed from the bootstrap PRNG, the uniform c1 (NTT form, first data level) from it, then e, as
   Encryptor_EncryptSymmetricReturnComponentsSetSeed draws them: c1_out HOST [batch][k1][n], noise_out HOST [batch][n] */
int b200_sample_sk(b200_ctx *ctx, const uint64_t *seeds, uint64_t *c1_out, int8_t *noise_out, uint64_t batch);
/* pk encryption of `batch` plaintexts from b200_sample_pk's samples.  pk: device [2][K][n] NTT form at the key level; plain:
   device [batch][n] coefficients mod t; out: device [batch][2][k1][n] at the first data level (encrypted at the key level and
   switched down, or with disable_special_modulus encrypted there directly) */
int b200_encrypt_pk_samples(b200_ctx *ctx, const uint64_t *pk, const int8_t *samples, const uint64_t *plain,
                            int disable_special_modulus, uint64_t *out, uint64_t batch, void *stream);
/* sk encryption at the first data level from b200_sample_sk's c1 and e: c0 = -(s c1 + e) + Delta m.  sk: device [K][n] NTT
   form.  On failure `out` is wiped (it holds s (*) c1 on the way). */
int b200_encrypt_sk_samples(b200_ctx *ctx, const uint64_t *sk, const uint64_t *c1, const int8_t *noise, const uint64_t *plain,
                            uint64_t *out, uint64_t batch, void *stream);
/* both steps in one call, returning after completion: item i gives the words of Encryptor_EncryptReturnComponentsSetSeed
   (Encryptor_EncryptSymmetricReturnComponentsSetSeed) with seeds[i]; samples_out (NULL or HOST [batch][3][n]) / noise_out
   (NULL or HOST [batch][n]) receive the samples */
int b200_encrypt_pk(b200_ctx *ctx, const uint64_t *pk, const uint64_t *seeds, const uint64_t *plain, int disable_special_modulus,
                    uint64_t *out, int8_t *samples_out, uint64_t batch, void *stream);
int b200_encrypt_sk(b200_ctx *ctx, const uint64_t *sk, const uint64_t *seeds, const uint64_t *plain, uint64_t *out,
                    int8_t *noise_out, uint64_t batch, void *stream);

/* ---- ciphertext arithmetic, batched over `batch` independent items (device pointers) ---- */
int b200_add(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, uint64_t *out, int size, uint64_t batch,
             void *stream);
int b200_sub(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, uint64_t *out, int size, uint64_t batch,
             void *stream);
int b200_negate(b200_ctx *ctx, int level, const uint64_t *a, uint64_t *out, int size, uint64_t batch, void *stream);
int b200_multiply(b200_ctx *ctx, int level, const uint64_t *a, int size_a, const uint64_t *b, int size_b, uint64_t *out,
                  uint64_t batch, void *stream);
int b200_square(b200_ctx *ctx, int level, const uint64_t *a, uint64_t *out, uint64_t batch, void *stream);
/* in: size-3 cts, relin_key: one key list (k digits) at the key level, out: size-2 cts (may alias in's first two polys) */
int b200_relinearize(b200_ctx *ctx, int level, const uint64_t *in3, const uint64_t *relin_key, uint64_t *out2,
                     uint64_t batch, void *stream);
/* multiply (2,2->3) followed by relinearize (3->2) without materialising the size-3 result in the caller's memory */
int b200_multiply_relin(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, const uint64_t *relin_key,
                        uint64_t *out2, uint64_t batch, void *stream);
/* out2[r] = sum_{j<m} relinearize(multiply(a[r][j], b[r][j])); a, b: [rows][m][2][k][n], out2: [rows][2][k][n].
   b may equal a (squares).  out2 must not overlap a or b.  m == 0: B200_E_INVALID; rows == 0: no work.  The words of
   b200_multiply_relin followed by m - 1 b200_add, with the adds folded into the key switch's mod-down. */
int b200_multiply_relin_sum(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, const uint64_t *relin_key,
                            uint64_t m, uint64_t *out2, uint64_t rows, void *stream);
/* size-2 cts: out = (sigma_g(c0), 0) + KeySwitch(sigma_g(c1), galois_key) */
int b200_apply_galois(b200_ctx *ctx, int level, const uint64_t *in2, uint32_t galois_elt, const uint64_t *galois_key,
                      uint64_t *out2, uint64_t batch, void *stream);
/* out = addend + apply_galois(in): the words of b200_apply_galois followed by b200_add (apply_galois + add_inplace), with the
   automorphism applied inside the key switch's digit loads and mod-down and the add folded into the mod-down.  addend2 ==
   NULL: no addend (the words of b200_apply_galois).  addend2 may equal in2 or out2; out2 must not overlap in2.  One step of a
   rotate-and-sum slot reduction (c = c + rotate_rows(c, s)). */
int b200_apply_galois_add(b200_ctx *ctx, int level, const uint64_t *in2, uint32_t galois_elt, const uint64_t *galois_key,
                          const uint64_t *addend2, uint64_t *out2, uint64_t batch, void *stream);
/* out2[i] = apply_galois(in2[src_idx ? src_idx[i] : i], elts[i]) with key list keys[i], word for word, as one key switch whose
   items carry their own element and key.  src_idx, elts and keys are HOST arrays of `batch` entries; keys[i] are device key
   lists as b200_apply_galois takes them.  Items with one key should be adjacent: below the key switch's cluster rule the
   MAC runs once per run of equal keys.  out2 must not overlap the sources in2[0 .. max src_idx]. */
int b200_apply_galois_many(b200_ctx *ctx, int level, const uint64_t *in2, const uint64_t *src_idx, const uint32_t *elts,
                           const uint64_t *const *keys, uint64_t *out2, uint64_t batch, void *stream);
/* plain: [batch or 1][n] coefficients mod t (plain_batch = 1 broadcasts one plaintext to every item).  multiply_plain
   follows the reference per plaintext item: an item with exactly one nonzero coefficient m is multiplied by m itself
   (its monomial path); any other item, and a monomial item when some q_i <= t, by the lifted plaintext
   (m + (Q - t) for m >= (t+1)/2).  The two are congruent mod t but give different ciphertext words. */
int b200_multiply_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t plain_batch,
                        uint64_t *out, uint64_t batch, void *stream);
/* plain: [pb][n] coefficients -> out: [pb][k][n] in NTT form at `level`.  `rule` selects the lift:
     B200_PLAIN_NTT_TRANSFORM  Evaluator::transform_to_ntt_inplace(Plaintext &, parms_id) (S/evaluator.cpp:2033-2124): every
                               coefficient m >= (t+1)/2 becomes m + (Q - t)
     B200_PLAIN_NTT_MULTIPLY   the operand b200_multiply_plain multiplies by, monomial path included (S/evaluator.cpp:1885-1933)
   The two differ only for a monomial with its coefficient in the upper half under the fast plain lift (every q_i > t). */
#define B200_PLAIN_NTT_TRANSFORM 0
#define B200_PLAIN_NTT_MULTIPLY 1
int b200_plain_to_ntt(b200_ctx *ctx, int level, const uint64_t *plain, uint64_t pb, uint64_t *out, int rule, void *stream);
/* plaintext matrix x ciphertext vector: out[i] = sum_{j<m} multiply_plain(cts[j], plain i,j) for i < R, word for word.
   cts: [m][size][k][n] coefficient form; plain_ntt: [R][m][k][n] from b200_plain_to_ntt; out: [R][size][k][n], must not
   overlap cts.  Each ciphertext is transformed once and each output once; m or R = 0 is a no-op. */
int b200_multiply_plain_sum(b200_ctx *ctx, int level, const uint64_t *cts, int size, uint64_t m, const uint64_t *plain_ntt,
                            uint64_t R, uint64_t *out, void *stream);
/* Baby-step giant-step slot-wise linear transform of V ciphertexts, word for word the chain
       inner_g = sum_{j < baby} multiply_plain(apply_galois(ct, elts[j - 1]), P[g][j])    (j = 0: ct itself)
       out     = inner_0 + sum_{1 <= g < giant} apply_galois(inner_g, elts[baby - 1 + g - 1])   (add, in order of g)
   cts, out: [V][2][k][n] coefficient form (out may be cts, or must not overlap it).  elts, keys: HOST arrays of the baby - 1
   baby-step then giant - 1 giant-step elements and device key lists.  plain_ntt: [giant][baby][k][n] from b200_plain_to_ntt
   (B200_PLAIN_NTT_MULTIPLY).  present: HOST [giant][baby] mask of terms, or NULL for all; an absent term is skipped, a step no
   present term uses needs no element or key, and a row without a present term is dropped.  No present term: an error. */
int b200_linear_transform(b200_ctx *ctx, int level, const uint64_t *cts, uint64_t V, int baby, int giant, const uint32_t *elts,
                          const uint64_t *const *keys, const uint64_t *plain_ntt, const uint8_t *present, uint64_t *out, void *stream);
int b200_add_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t plain_batch,
                   uint64_t *out, uint64_t batch, void *stream);
int b200_sub_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t plain_batch,
                   uint64_t *out, uint64_t batch, void *stream);
/* out = x (*) y coefficient-wise mod q_r, y broadcast over polys (and over items when y_batch == 1) */
int b200_dyadic_product(b200_ctx *ctx, int level, const uint64_t *x, int size, const uint64_t *y, uint64_t y_batch,
                        uint64_t *out, uint64_t batch, void *stream);
/* residues of small signed values (host-sampled ternary secrets / clipped-normal noise, S/util/rlwe.cpp:23-67):
   vals [polys][n] int64 (device) -> out [polys][k][n], out = v < 0 ? v + q_r : v */
int b200_expand_signed(b200_ctx *ctx, int level, const int64_t *vals, int polys, uint64_t *out, void *stream);
/* [batch][size][k][n] at `level` -> [batch][size][k-1][n] at level+1 */
int b200_mod_switch_to_next(b200_ctx *ctx, int level, const uint64_t *a, int size, uint64_t *out, uint64_t batch,
                            void *stream);
/* ct (size polys) . secret-key powers (NTT form, [size-1][k][n]) -> plaintext coefficients [batch][n] mod t */
int b200_decrypt(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *plain_out,
                 uint64_t batch, void *stream);
/* phase = c0 + sum_j c_j * s^j in coefficient form: [batch][k][n] (Decryptor::dot_product_ct_sk_array, S/decryptor.cpp:340-422) */
int b200_ct_sk_phase(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *phase_out,
                     uint64_t batch, void *stream);
/* infinity norm of the centred t * phase mod Q of each item, as little-endian multi-precision words; norm_out is a HOST
   array [batch][words], words >= ceil(bits(Q)/64) + 1; returns after completion (Decryptor::invariant_noise_internal,
   S/decryptor.cpp:424-485: the quantity behind invariant_noise_budget and the fork's invariant_noise) */
int b200_noise_norm(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *norm_out,
                    int words, uint64_t batch, void *stream);
/* any-nonzero test over polys [1, size) of each item (transparent-ciphertext guard, S/ciphertext.h:451-456);
   flags_out: device array [batch] of 0/1 ("is transparent") */
int b200_is_transparent(b200_ctx *ctx, int level, const uint64_t *ct, int size, uint32_t *flags_out, uint64_t batch,
                        void *stream);

/* the same test without clearing: flags[item] = 1 when polys [1, size) of the item hold a nonzero word; the caller zeroes
   `flags` beforehand, and `flags` may be pinned host memory from b200_malloc_host (no fill kernel, no copy back) */
int b200_any_nonzero(b200_ctx *ctx, int level, const uint64_t *ct, int size, uint32_t *flags, uint64_t batch, void *stream);

/* ---- host-buffer (end-to-end) variants: pinned or pageable host memory in, host memory out;
        H2D / compute / D2H are chunked and overlapped on internal streams; returns after completion ---- */
int b200_multiply_relin_host(b200_ctx *ctx, int level, const uint64_t *a_host, const uint64_t *b_host,
                             const uint64_t *relin_key_dev, uint64_t *out_host, uint64_t batch);

/* gather (`gather` != 0: slab[i*words..] <- *host_ptrs[i]) or scatter (*host_ptrs[i] <- slab[i*words..]) of `count` device
   buffers of `words` words in one launch; `host_ptrs` is a HOST array of device pointers and must stay valid until the
   stream has consumed it (pageable memory is copied at call time) */
int b200_gather_scatter(b200_ctx *ctx, uint64_t *const *host_ptrs, uint64_t count, uint64_t *slab, uint64_t words, int gather,
                        void *stream);
/* the same with the pointer table already in device-accessible memory (pinned host memory qualifies): one launch, no copy */
int b200_gather_scatter_table(b200_ctx *ctx, uint64_t *const *table, uint64_t count, uint64_t *slab, uint64_t words, int gather,
                              void *stream);
/* CUDA-graph capture of a fixed launch sequence on `stream` (kernels by value, stream-ordered allocations as memory nodes);
   capture_end instantiates and returns an executable handle for b200_graph_launch / b200_graph_destroy */
int b200_capture_begin(b200_ctx *ctx, void *stream);
int b200_capture_end(b200_ctx *ctx, void *stream, void **graph_exec);
int b200_graph_launch(b200_ctx *ctx, void *graph_exec, void *stream);
int b200_graph_destroy(b200_ctx *ctx, void *graph_exec);
/* wait for `stream` without spinning (blocking-sync event cached in *event_slot; release it with b200_event_destroy) */
int b200_stream_synchronize_blocking(b200_ctx *ctx, void *stream, void **event_slot);
int b200_event_destroy(b200_ctx *ctx, void *event);
/* make the context's GPU the calling thread's current device (new host threads start on device 0) */
int b200_bind_thread(b200_ctx *ctx);
/* stream-ordered allocation for work enqueued on `stream` afterwards (release with b200_free_async on the same stream) */
int b200_malloc_async(b200_ctx *ctx, size_t bytes, void **dptr, void *stream);

/* number of kernel launches issued by this library since the context was created (bench.py: gpu_launches) */
uint64_t b200_launch_count(const b200_ctx *ctx);
/* developer aid: with B200_TRACE=1 in the environment every kernel launch is bracketed by CUDA events;
   this prints the per-kernel totals to stderr and clears the log (no-op otherwise) */
void b200_trace_dump(void);
/* developer aid: resident CTAs per SM of the FP64 NTT kernel (log2 n, forward != 0, threads per CTA), as the launcher
   queries it to size the grid of the persistent kernel; B200_E_INVALID when no such kernel exists.
   Meaningful once a context exists (context creation raises the kernels' shared-memory limit) */
int b200_debug_ntt_ctas_per_sm(int logn, int forward, int threads);
/* developer aid: device prime `prime_index` (key primes, then the auxiliary primes, then the plain modulus when batching) in
   *prime (0: no such prime), and its FP64 transform's renorm masks (bit i: renormalise the inputs of pass i in execution
   order).  schedule 0: the masks the context's transforms use; 1: those of the generic pass schedule; 2: those of the
   statically scheduled kernels (n = 4096 ... 16384 only).  B200_E_INVALID for no such prime, a prime off the FP64 path or a
   schedule the size does not have */
int b200_debug_fp_masks(const b200_ctx *ctx, int prime_index, int schedule, uint64_t *prime, unsigned *fwd, unsigned *inv);

#ifdef __cplusplus
}
#endif
#endif
