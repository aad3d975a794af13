/* b200_sealc.h — layer-2 C ABI: the SEAL C export names that Sunscreen's `seal_fhe` crate binds to
 * (seal_fhe/build.rs:157-180 allow-list, seal_fhe/bindgen_wrapper.h), re-implemented over the B200 backend.
 *
 * Same calling convention as the reference's S/c/defines.h:26-56: every function returns an HRESULT in a
 * `long`, objects are opaque `void*` handles created by *_Create* and released by *_Destroy, out-parameters are
 * pointers.  Error mapping follows S/c/evaluator.cpp:58-80: NULL handle -> E_POINTER, what the reference throws
 * as std::invalid_argument -> E_INVALIDARG, std::logic_error -> COR_E_INVALIDOPERATION.
 *
 * Ciphertexts live in GPU memory; the host mirror is materialised lazily by the accessors that read words
 * (Ciphertext_GetDataAt*, B200_Ciphertext_GetWords).  Evaluator calls are re-entrant (one internal stream per
 * SEALContext, enqueue under a mutex), matching the reference's thread-safety contract for the rayon DAG
 * executor (sunscreen_runtime/src/run.rs:415-469).
 *
 * Covered: all 121 functions seal_fhe references (grep `bindgen::` in seal_fhe/src) — parameter objects,
 * SEALContext, Ciphertext/Plaintext/PublicKey/SecretKey/KSwitchKeys data objects and their wire format
 * (SaveSize/Save/Load, S/serialization.h), the whole BFV Evaluator surface, Decryptor (decrypt, invariant noise and
 * noise budget), KeyGenerator and Encryptor incl. the fork's ReturnComponents variants (sampling on the host with the
 * reference's PRNG stream, arithmetic on the GPU), BatchEncoder, PolynomialArray.
 * B200_* names are extensions (bulk word access, batching) that the reference does not have.
 */
#ifndef B200_SEALC_H
#define B200_SEALC_H
#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef SEAL_C_FUNC
#define SEAL_C_FUNC long
#endif

/* HRESULT values (S/c/defines.h:29-41) */
#define B200_S_OK 0L
#define B200_E_POINTER_HR 0x80004003L
#define B200_E_INVALIDARG_HR 0x80070057L
#define B200_E_OUTOFMEMORY_HR 0x8007000EL
#define B200_E_UNEXPECTED_HR 0x8000FFFFL
#define B200_COR_E_INVALIDOPERATION_HR 0x80131509L
#define B200_ERROR_INVALID_INDEX_HR 0x80070585L /* HRESULT_FROM_WIN32(ERROR_INVALID_INDEX) */

/* ---- Modulus / CoeffModulus (S/c/modulus.h) ---- */
SEAL_C_FUNC Modulus_Create1(uint64_t value, void **small_modulus);
SEAL_C_FUNC Modulus_Create2(void *copy, void **small_modulus);
SEAL_C_FUNC Modulus_Destroy(void *thisptr);
SEAL_C_FUNC Modulus_Value(void *thisptr, uint64_t *value);
SEAL_C_FUNC Modulus_BitCount(void *thisptr, int *bit_count);
SEAL_C_FUNC CoeffModulus_MaxBitCount(uint64_t poly_modulus_degree, int sec_level, int *bit_count);
SEAL_C_FUNC CoeffModulus_BFVDefault(uint64_t poly_modulus_degree, int sec_level, uint64_t *length, void **coeffs);
SEAL_C_FUNC CoeffModulus_Create1(uint64_t poly_modulus_degree, uint64_t length, int *bit_sizes, void **coeffs);

/* ---- EncryptionParameters (S/c/encryptionparameters.h) ---- */
SEAL_C_FUNC EncParams_Create1(uint8_t scheme, void **enc_params);
SEAL_C_FUNC EncParams_Destroy(void *thisptr);
SEAL_C_FUNC EncParams_GetPolyModulusDegree(void *thisptr, uint64_t *degree);
SEAL_C_FUNC EncParams_SetPolyModulusDegree(void *thisptr, uint64_t degree);
SEAL_C_FUNC EncParams_GetCoeffModulus(void *thisptr, uint64_t *length, void **coeffs);
SEAL_C_FUNC EncParams_SetCoeffModulus(void *thisptr, uint64_t length, void **coeffs);
SEAL_C_FUNC EncParams_GetScheme(void *thisptr, uint8_t *scheme);
SEAL_C_FUNC EncParams_GetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC EncParams_GetPlainModulus(void *thisptr, void **plain_modulus);
SEAL_C_FUNC EncParams_SetPlainModulus1(void *thisptr, void *modulus);
SEAL_C_FUNC EncParams_SetPlainModulus2(void *thisptr, uint64_t plain_modulus);

/* ---- SEALContext (S/c/sealcontext.h) ---- */
SEAL_C_FUNC SEALContext_Create(void *encryptionParams, bool expand_mod_chain, int sec_level, void **context);
SEAL_C_FUNC SEALContext_Destroy(void *thisptr);
SEAL_C_FUNC SEALContext_KeyParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC SEALContext_FirstParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC SEALContext_LastParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC SEALContext_ParametersSet(void *thisptr, bool *params_set);
SEAL_C_FUNC SEALContext_UsingKeyswitching(void *thisptr, bool *using_keyswitching);

/* ---- Ciphertext (S/c/ciphertext.h) ---- */
SEAL_C_FUNC Ciphertext_Create1(void *pool, void **cipher);
SEAL_C_FUNC Ciphertext_Create2(void *copy, void **cipher);
SEAL_C_FUNC Ciphertext_Set(void *thisptr, void *assign);
SEAL_C_FUNC Ciphertext_Destroy(void *thisptr);
SEAL_C_FUNC Ciphertext_Size(void *thisptr, uint64_t *size);
SEAL_C_FUNC Ciphertext_PolyModulusDegree(void *thisptr, uint64_t *poly_modulus_degree);
SEAL_C_FUNC Ciphertext_CoeffModulusSize(void *thisptr, uint64_t *coeff_modulus_size);
SEAL_C_FUNC Ciphertext_ParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC Ciphertext_SetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC Ciphertext_Resize1(void *thisptr, void *context, uint64_t *parms_id, uint64_t size);
SEAL_C_FUNC Ciphertext_GetDataAt1(void *thisptr, uint64_t index, uint64_t *data);
SEAL_C_FUNC Ciphertext_GetDataAt2(void *thisptr, uint64_t poly_index, uint64_t coeff_index, uint64_t *data);
SEAL_C_FUNC Ciphertext_SetDataAt(void *thisptr, uint64_t index, uint64_t value);
SEAL_C_FUNC Ciphertext_IsNTTForm(void *thisptr, bool *is_ntt_form);
SEAL_C_FUNC Ciphertext_SetIsNTTForm(void *thisptr, bool is_ntt_form);
SEAL_C_FUNC Ciphertext_Scale(void *thisptr, double *scale);
SEAL_C_FUNC Ciphertext_IsTransparent(void *thisptr, bool *result);

/* ---- Plaintext (S/c/plaintext.h) ---- */
SEAL_C_FUNC Plaintext_Create1(void *memoryPoolHandle, void **plaintext);
SEAL_C_FUNC Plaintext_Create2(uint64_t coeffCount, void *memoryPoolHandle, void **plaintext);
SEAL_C_FUNC Plaintext_Create4(uint8_t *hex_poly, void *memoryPoolHandle, void **plaintext);
SEAL_C_FUNC Plaintext_Create5(void *copy, void **plaintext);
SEAL_C_FUNC Plaintext_Destroy(void *thisptr);
SEAL_C_FUNC Plaintext_CoeffCount(void *thisptr, uint64_t *coeff_count);
SEAL_C_FUNC Plaintext_CoeffAt(void *thisptr, uint64_t index, uint64_t *coeff);
SEAL_C_FUNC Plaintext_SetCoeffAt(void *thisptr, uint64_t index, uint64_t value);
SEAL_C_FUNC Plaintext_Resize(void *thisptr, uint64_t coeff_count);
SEAL_C_FUNC Plaintext_GetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC Plaintext_SetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC Plaintext_IsNTTForm(void *thisptr, bool *is_ntt_form);
SEAL_C_FUNC Plaintext_IsZero(void *thisptr, bool *is_zero);

/* ---- PublicKey / SecretKey (S/c/publickey.h, secretkey.h) ---- */
SEAL_C_FUNC PublicKey_Create1(void **public_key);
SEAL_C_FUNC PublicKey_Create2(void *copy, void **public_key);
SEAL_C_FUNC PublicKey_Data(void *thisptr, void **data);
SEAL_C_FUNC PublicKey_ParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC PublicKey_Destroy(void *thisptr);
SEAL_C_FUNC SecretKey_Create1(void **secret_key);
SEAL_C_FUNC SecretKey_Create2(void *copy, void **secret_key);
SEAL_C_FUNC SecretKey_Data(void *thisptr, void **data);
SEAL_C_FUNC SecretKey_ParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC SecretKey_Destroy(void *thisptr);

/* ---- KSwitchKeys / RelinKeys / GaloisKeys (S/c/kswitchkeys.h, relinkeys.h, galoiskeys.h) ---- */
SEAL_C_FUNC KSwitchKeys_Create1(void **kswitch_keys);
SEAL_C_FUNC KSwitchKeys_Create2(void *copy, void **kswitch_keys);
SEAL_C_FUNC KSwitchKeys_Destroy(void *thisptr);
SEAL_C_FUNC KSwitchKeys_Size(void *thisptr, uint64_t *size);
SEAL_C_FUNC KSwitchKeys_RawSize(void *thisptr, uint64_t *key_count);
SEAL_C_FUNC KSwitchKeys_GetKeyList(void *thisptr, uint64_t index, uint64_t *count, void **key_list);
SEAL_C_FUNC KSwitchKeys_ClearDataAndReserve(void *thisptr, uint64_t size);
SEAL_C_FUNC KSwitchKeys_AddKeyList(void *thisptr, uint64_t count, void **key_list);
SEAL_C_FUNC KSwitchKeys_GetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC KSwitchKeys_SetParmsId(void *thisptr, uint64_t *parms_id);
SEAL_C_FUNC RelinKeys_GetIndex(uint64_t key_power, uint64_t *index);
SEAL_C_FUNC GaloisKeys_GetIndex(uint32_t galois_elt, uint64_t *index);

/* ---- Evaluator (S/c/evaluator.h:16-79) ---- */
SEAL_C_FUNC Evaluator_Create(void *context, void **evaluator);
SEAL_C_FUNC Evaluator_Destroy(void *thisptr);
SEAL_C_FUNC Evaluator_Negate(void *thisptr, void *encrypted, void *destination);
SEAL_C_FUNC Evaluator_Add(void *thisptr, void *encrypted1, void *encrypted2, void *destination);
SEAL_C_FUNC Evaluator_AddMany(void *thisptr, uint64_t count, void **encrypteds, void *destination);
SEAL_C_FUNC Evaluator_AddPlain(void *thisptr, void *encrypted, void *plain, void *destination);
SEAL_C_FUNC Evaluator_Sub(void *thisptr, void *encrypted1, void *encrypted2, void *destination);
SEAL_C_FUNC Evaluator_SubPlain(void *thisptr, void *encrypted, void *plain, void *destination);
SEAL_C_FUNC Evaluator_Multiply(void *thisptr, void *encrypted1, void *encrypted2, void *destination, void *pool);
SEAL_C_FUNC Evaluator_MultiplyMany(void *thisptr, uint64_t count, void **encrypteds, void *relin_keys, void *destination,
                                   void *pool);
SEAL_C_FUNC Evaluator_MultiplyPlain(void *thisptr, void *encrypted, void *plain, void *destination, void *pool);
SEAL_C_FUNC Evaluator_Square(void *thisptr, void *encrypted, void *destination, void *pool);
SEAL_C_FUNC Evaluator_Relinearize(void *thisptr, void *encrypted, void *relinKeys, void *destination, void *pool);
SEAL_C_FUNC Evaluator_ModSwitchToNext1(void *thisptr, void *encrypted, void *destination, void *pool);
SEAL_C_FUNC Evaluator_ModSwitchToNext2(void *thisptr, void *plain, void *destination);
SEAL_C_FUNC Evaluator_Exponentiate(void *thisptr, void *encrypted, uint64_t exponent, void *relin_keys, void *destination,
                                   void *pool);
SEAL_C_FUNC Evaluator_ApplyGalois(void *thisptr, void *encrypted, uint32_t galois_elt, void *galois_keys, void *destination,
                                  void *pool);
SEAL_C_FUNC Evaluator_RotateRows(void *thisptr, void *encrypted, int steps, void *galoisKeys, void *destination, void *pool);
SEAL_C_FUNC Evaluator_RotateColumns(void *thisptr, void *encrypted, void *galois_keys, void *destination, void *pool);
SEAL_C_FUNC Evaluator_ContextUsingKeyswitching(void *thisptr, bool *using_keyswitching);

/* ---- Decryptor (S/c/decryptor.h) ---- */
SEAL_C_FUNC Decryptor_Create(void *context, void *secret_key, void **decryptor);
SEAL_C_FUNC Decryptor_Destroy(void *thisptr);
SEAL_C_FUNC Decryptor_Decrypt(void *thisptr, void *encrypted, void *destination);
SEAL_C_FUNC Decryptor_InvariantNoiseBudget(void *thisptr, void *encrypted, int *invariant_noise_budget);
SEAL_C_FUNC Decryptor_InvariantNoise(void *thisptr, void *encrypted, double *invariant_noise);

/* ---- KeyGenerator (S/c/keygenerator.h) : host-side sampling (the reference's Blake2xb stream), GPU arithmetic ---- */
SEAL_C_FUNC KeyGenerator_Create1(void *context, void **key_generator);
SEAL_C_FUNC KeyGenerator_Create2(void *context, void *secret_key, void **key_generator);
SEAL_C_FUNC KeyGenerator_Destroy(void *thisptr);
SEAL_C_FUNC KeyGenerator_SecretKey(void *thisptr, void **secret_key);
SEAL_C_FUNC KeyGenerator_CreatePublicKey(void *thisptr, bool save_seed, void **public_key);
SEAL_C_FUNC KeyGenerator_CreateRelinKeys(void *thisptr, bool save_seed, void **relin_keys);
SEAL_C_FUNC KeyGenerator_CreateGaloisKeysFromElts(void *thisptr, uint64_t count, uint32_t *galois_elts, bool save_seed,
                                                  void **galois_keys);
SEAL_C_FUNC KeyGenerator_CreateGaloisKeysFromSteps(void *thisptr, uint64_t count, int *steps, bool save_seed, void **galois_keys);
SEAL_C_FUNC KeyGenerator_CreateGaloisKeysAll(void *thisptr, bool save_seed, void **galois_keys);

/* ---- Encryptor (S/c/encryptor.h) ---- */
SEAL_C_FUNC Encryptor_Create(void *context, void *public_key, void *secret_key, void **encryptor);
SEAL_C_FUNC Encryptor_Destroy(void *thisptr);
SEAL_C_FUNC Encryptor_Encrypt(void *thisptr, void *plaintext, void *destination, void *pool_handle);
SEAL_C_FUNC Encryptor_EncryptSymmetric(void *thisptr, void *plaintext, bool save_seed, void *destination, void *pool_handle);
/* the Sunscreen fork's entry points that also return u, e (PolynomialArray handles) and the rounding remainder
   (S/c/encryptor.h:24-40, S/c/encryptor.cpp:136-240,300-372) */
SEAL_C_FUNC Encryptor_EncryptReturnComponents(void *thisptr, void *plaintext, bool disable_special_modulus, void *destination,
                                              void *u_destination, void *e_destination, void *remainder_destination,
                                              void *pool_handle);
SEAL_C_FUNC Encryptor_EncryptReturnComponentsSetSeed(void *thisptr, void *plaintext, bool disable_special_modulus,
                                                     void *destination, void *u_destination, void *e_destination,
                                                     void *remainder_destination, void *seed, void *pool_handle);
SEAL_C_FUNC Encryptor_EncryptSymmetricReturnComponents(void *thisptr, void *plaintext, void *destination, void *e_destination,
                                                       void *remainder_destination, void *pool_handle);
SEAL_C_FUNC Encryptor_EncryptSymmetricReturnComponentsSetSeed(void *thisptr, void *plaintext, void *destination,
                                                              void *e_destination, void *remainder_destination, void *seed,
                                                              void *pool_handle);

/* ---- BatchEncoder (S/c/batchencoder.h): slot permutation and negacyclic NTT mod t on the GPU ---- */
SEAL_C_FUNC BatchEncoder_Create(void *context, void **batch_encoder);
SEAL_C_FUNC BatchEncoder_Destroy(void *thisptr);
SEAL_C_FUNC BatchEncoder_Encode1(void *thisptr, uint64_t count, uint64_t *values, void *destination);
SEAL_C_FUNC BatchEncoder_Encode2(void *thisptr, uint64_t count, int64_t *values, void *destination);
SEAL_C_FUNC BatchEncoder_Decode1(void *thisptr, void *plain, uint64_t *count, uint64_t *destination, void *pool);
SEAL_C_FUNC BatchEncoder_Decode2(void *thisptr, void *plain, uint64_t *count, int64_t *destination, void *pool);
SEAL_C_FUNC BatchEncoder_GetSlotCount(void *thisptr, uint64_t *slot_count);

/* ---- wire format (S/c/ciphertext.h:80-86, plaintext.h:82-88, kswitchkeys.h:40-46, publickey.h:30-36,
        secretkey.h:30-36 -> S/serialization.h): compr_mode 0 none, 1 zlib, 2 zstd ---- */
#define B200_COR_E_IO_HR 0x80131620L
SEAL_C_FUNC Ciphertext_SaveSize(void *thisptr, uint8_t compr_mode, int64_t *result);
SEAL_C_FUNC Ciphertext_Save(void *thisptr, uint8_t *outptr, uint64_t size, uint8_t compr_mode, int64_t *out_bytes);
SEAL_C_FUNC Ciphertext_UnsafeLoad(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC Ciphertext_Load(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC Plaintext_SaveSize(void *thisptr, uint8_t compr_mode, int64_t *result);
SEAL_C_FUNC Plaintext_Save(void *thisptr, uint8_t *outptr, uint64_t size, uint8_t compr_mode, int64_t *out_bytes);
SEAL_C_FUNC Plaintext_UnsafeLoad(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC Plaintext_Load(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC PublicKey_SaveSize(void *thisptr, uint8_t compr_mode, int64_t *result);
SEAL_C_FUNC PublicKey_Save(void *thisptr, uint8_t *outptr, uint64_t size, uint8_t compr_mode, int64_t *out_bytes);
SEAL_C_FUNC PublicKey_UnsafeLoad(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC PublicKey_Load(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC SecretKey_SaveSize(void *thisptr, uint8_t compr_mode, int64_t *result);
SEAL_C_FUNC SecretKey_Save(void *thisptr, uint8_t *outptr, uint64_t size, uint8_t compr_mode, int64_t *out_bytes);
SEAL_C_FUNC SecretKey_UnsafeLoad(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC SecretKey_Load(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC KSwitchKeys_SaveSize(void *thisptr, uint8_t compr_mode, int64_t *result);
SEAL_C_FUNC KSwitchKeys_Save(void *thisptr, uint8_t *outptr, uint64_t size, uint8_t compr_mode, int64_t *out_bytes);
SEAL_C_FUNC KSwitchKeys_UnsafeLoad(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);
SEAL_C_FUNC KSwitchKeys_Load(void *thisptr, void *context, uint8_t *inptr, uint64_t size, int64_t *in_bytes);

/* ---- PolynomialArray (S/c/polyarray.h, added by the Sunscreen fork) ---- */
SEAL_C_FUNC PolynomialArray_Create(void *memoryPoolHandle, void **poly_array);
SEAL_C_FUNC PolynomialArray_CreateFromCiphertext(void *memoryPoolHandle, void *context, void *ciphertext, void **poly_array);
SEAL_C_FUNC PolynomialArray_CreateFromPublicKey(void *memoryPoolHandle, void *context, void *public_key, void **poly_array);
SEAL_C_FUNC PolynomialArray_CreateFromSecretKey(void *memoryPoolHandle, void *context, void *secret_key, void **poly_array);
SEAL_C_FUNC PolynomialArray_Copy(void *copy, void **poly_array);
SEAL_C_FUNC PolynomialArray_Destroy(void *thisptr);
SEAL_C_FUNC PolynomialArray_IsReserved(void *thisptr, bool *is_reserved);
SEAL_C_FUNC PolynomialArray_IsRns(void *thisptr, bool *is_rns);
SEAL_C_FUNC PolynomialArray_IsMultiprecision(void *thisptr, bool *is_multiprecision);
SEAL_C_FUNC PolynomialArray_ToRns(void *thisptr);
SEAL_C_FUNC PolynomialArray_ToMultiprecision(void *thisptr);
SEAL_C_FUNC PolynomialArray_GetPolynomial(void *thisptr, uint64_t poly_index, uint64_t *data);
SEAL_C_FUNC PolynomialArray_ExportSize(void *thisptr, uint64_t *size);
SEAL_C_FUNC PolynomialArray_PerformExport(void *thisptr, uint64_t *data);
SEAL_C_FUNC PolynomialArray_PolySize(void *thisptr, uint64_t *size);
SEAL_C_FUNC PolynomialArray_PolyModulusDegree(void *thisptr, uint64_t *size);
SEAL_C_FUNC PolynomialArray_CoeffModulusSize(void *thisptr, uint64_t *size);
SEAL_C_FUNC PolynomialArray_Drop(void *thisptr, void **poly_array);

/* ---- extensions (not in the reference) ---- */
/* deterministic pk-encryption from a 64-byte seed: the same random stream (and therefore the same ciphertext words)
   as the reference's Encryptor_EncryptReturnComponentsSetSeed (S/c/encryptor.cpp:185-240) */
/* 1: Zstandard 1.4.5 is compiled in (compressed bytes == the reference's); 0: system libzstd bound at run time */
SEAL_C_FUNC B200_VendoredZstd(void);
SEAL_C_FUNC B200_Encryptor_EncryptSetSeed(void *thisptr, void *plaintext, const uint64_t *seed8, void *destination);
/* bulk word access: the reference only offers word-at-a-time accessors */
SEAL_C_FUNC B200_Ciphertext_SetWords(void *thisptr, void *context, uint64_t *parms_id, uint64_t size, bool is_ntt_form,
                                     const uint64_t *words);
SEAL_C_FUNC B200_Ciphertext_GetWords(void *thisptr, uint64_t *words, uint64_t capacity_words);
/* the same for `count` handles at once: `words` is one contiguous host buffer [count][size][k][n] (pinned memory moves
   asynchronously at link speed); one transfer + one device-side scatter / gather instead of a copy per handle */
SEAL_C_FUNC B200_Ciphertext_SetWordsBatch(void *context, uint64_t count, void **ciphertexts, uint64_t *parms_id, uint64_t size,
                                          bool is_ntt_form, const uint64_t *words);
SEAL_C_FUNC B200_Ciphertext_GetWordsBatch(void *context, uint64_t count, void **ciphertexts, uint64_t *words,
                                          uint64_t capacity_words);
SEAL_C_FUNC B200_Plaintext_SetCoeffs(void *thisptr, uint64_t count, const uint64_t *coeffs);
/* Key list `index` <- `decomp` size-2 key-level NTT-form ciphertexts given as one flat word array */
SEAL_C_FUNC B200_KSwitchKeys_SetKeyWords(void *thisptr, void *context, uint64_t index, uint64_t decomp, const uint64_t *words);
/* SecretKey <- key-level NTT-form words [K][n] */
SEAL_C_FUNC B200_SecretKey_SetWords(void *thisptr, void *context, const uint64_t *words);
/* wait until every enqueued operation of this context has finished */
SEAL_C_FUNC B200_SEALContext_Synchronize(void *context);
/* multiply + relinearize over `count` independent pairs in one launch sequence (DAG-level batching seam) */
SEAL_C_FUNC B200_Evaluator_MultiplyRelinBatch(void *thisptr, uint64_t count, void **encrypteds1, void **encrypteds2,
                                              void *relin_keys, void **destinations);

/* the other DAG node kinds as batches of independent size-2 ciphertexts at one level (same words as the per-handle calls) */
SEAL_C_FUNC B200_Evaluator_AddSubBatch(void *thisptr, uint64_t count, void **encrypteds1, void **encrypteds2, bool subtract,
                                       void **destinations);
/* which: 0 add_plain, 1 sub_plain, 2 multiply_plain; plains[i] goes with encrypteds[i] */
SEAL_C_FUNC B200_Evaluator_PlainBatch(void *thisptr, int which, uint64_t count, void **encrypteds, void **plains,
                                      void **destinations);
/* one row rotation for all items; the Galois key for `steps` must be present */
SEAL_C_FUNC B200_Evaluator_RotateRowsBatch(void *thisptr, uint64_t count, void **encrypteds, int steps, void *galois_keys,
                                           void **destinations);
/* plaintext matrix x ciphertext vector: destinations[i] receives the words of multiply_plain(encrypteds[0], plains[i*cols])
   followed by add_inplace(multiply_plain(encrypteds[j], plains[i*cols + j])) for j = 1 ... cols-1 (plains row-major,
   rows x cols).  Same checks and HRESULTs as those calls, except: all encrypteds must have one size, and a transparent
   partial sum is not detected (only a transparent final result).  Destinations may alias encrypteds. */
SEAL_C_FUNC B200_Evaluator_MultiplyPlainSum(void *thisptr, uint64_t rows, uint64_t cols, void **encrypteds, void **plains,
                                            void **destinations);
/* rotate-and-sum slot reduction: destinations[i] receives the words of
       c = encrypteds[i]; for s in steps: c = Evaluator_Add(c, Evaluator_RotateRows(c, s));
       if columns: c = Evaluator_Add(c, Evaluator_RotateColumns(c))
   Steps follow RotateRows: 0 adds c to itself, a step without its own key goes through its NAF parts.  Same checks and
   HRESULTs as that chain, except that a transparent intermediate is not detected (only a transparent final result; a
   transparent input stays transparent).  All encrypteds at one level; destinations may alias encrypteds. */
SEAL_C_FUNC B200_Evaluator_RotateSumBatch(void *thisptr, uint64_t count, void **encrypteds, int nsteps, const int *steps, bool columns,
                                          void *galois_keys, void **destinations);
/* encrypted inner products: destinations[i] receives the words of
       c = Relinearize(Multiply(encrypteds1[i*cols], encrypteds2[i*cols]));
       for j = 1 ... cols-1: c = Add(c, Relinearize(Multiply(encrypteds1[i*cols + j], encrypteds2[i*cols + j])))
   (both arrays row-major, rows x cols; the same handle twice in one term squares it).  Same checks and HRESULTs as that
   chain, all made before any work, except: every operand must be a size-2 ciphertext (the chain's Relinearize refuses larger
   products with single-key relinearization keys) at one level for the whole call, and a transparent intermediate is not
   detected (only a term whose two operands are both transparent, and a transparent final result).  Destinations may alias
   encrypteds. */
SEAL_C_FUNC B200_Evaluator_MultiplyRelinSum(void *thisptr, uint64_t rows, uint64_t cols, void **encrypteds1, void **encrypteds2,
                                            void *relin_keys, void **destinations);
/* row rotations by a step per item: destinations[i] receives the words of Evaluator_RotateRows(encrypteds[i], steps[i]), with
   one key switch for the whole batch.  Same checks and HRESULTs as those calls, all made before any work, except: a step
   without its own Galois key is E_INVALIDARG (RotateRows would split it into NAF parts), and all encrypteds are at one level.
   Destinations may alias encrypteds. */
SEAL_C_FUNC B200_Evaluator_RotateRowsStepsBatch(void *thisptr, uint64_t count, void **encrypteds, const int *steps, void *galois_keys,
                                                void **destinations);
/* baby-step giant-step slot-wise linear transform: destinations[i] receives the words of
       inner_g = Add over j of MultiplyPlain(RotateRows(encrypteds[i], j), plains[g*baby + j])   (j = 0: encrypteds[i] itself)
       c = inner_0;  for g = 1 ... giant-1: c = Add(c, RotateRows(inner_g, g*baby))
   plains: giant x baby coefficient-form plaintexts (BatchEncoder output), row-major; a NULL handle is an absent term (skipped;
   a row without terms is dropped).  Same checks and HRESULTs as that chain, all made before any work, except: a step without
   its own Galois key is E_INVALIDARG (create the keys with KeyGenerator_CreateGaloisKeysFromSteps for steps 1 ... baby-1 and
   g*baby), all encrypteds are at one level, and a transparent partial sum is not detected (only a transparent final result).
   baby or giant 0 and a call where every term is absent are E_INVALIDARG.  Destinations may alias encrypteds. */
SEAL_C_FUNC B200_Evaluator_LinearTransform(void *thisptr, uint64_t count, void **encrypteds, uint64_t baby, uint64_t giant, void **plains,
                                           void *galois_keys, void **destinations);

/* slots in and out for many plaintexts / ciphertexts at once, one transfer each way and one launch sequence per call:
   EncodeBatch: destinations[i] receives the plaintext BatchEncoder_Encode1 (is_signed: Encode2, the words read as int64_t)
   gives for row i of `values`, one host buffer [count][values_per_item].  Same checks and HRESULTs as those calls.
   DecodeBatch: slots_out (host [count][n], uint64_t or with is_signed int64_t) receives BatchEncoder_Decode1/2 of plains[i].
   Same checks and HRESULTs as those calls, all made before any work.
   DecryptSlotsBatch: slots_out (host [count][n]) receives BatchEncoder_Decode1/2(Decryptor_Decrypt(encrypteds[i])) and, when
   budgets != NULL, budgets[i] Decryptor_InvariantNoiseBudget(encrypteds[i]), from one secret-key phase per item.  Same checks
   and HRESULTs as those calls, all made before any work, except: all encrypteds must have one size and one level
   (E_INVALIDARG).  A decryptor and an encoder of different contexts are E_INVALIDARG. */
SEAL_C_FUNC B200_BatchEncoder_EncodeBatch(void *encoder, uint64_t count, uint64_t values_per_item, const uint64_t *values,
                                          bool is_signed, void **destinations);
SEAL_C_FUNC B200_BatchEncoder_DecodeBatch(void *encoder, uint64_t count, void **plains, bool is_signed, void *slots_out);
SEAL_C_FUNC B200_Decryptor_DecryptSlotsBatch(void *decryptor, void *encoder, uint64_t count, void **encrypteds, bool is_signed,
                                             void *slots_out, int *budgets);
/* encryption of many plaintexts at once: every item is sampled on the host from its own seed, in parallel over items, and the
   samples cross in one int8 transfer; the arithmetic is one launch sequence per call.
   EncryptBatch: destinations[i] receives Encryptor_Encrypt(plains[i]) (symmetric: Encryptor_EncryptSymmetric).  seeds: host
   [count][8], item i then gives the words of B200_Encryptor_EncryptSetSeed(plains[i], seeds + 8 i) (symmetric: of
   Encryptor_EncryptSymmetricReturnComponentsSetSeed), or NULL for a fresh random seed per item.  Same checks and HRESULTs
   as those calls, all made before any work (a missing key first, then the plaintexts).
   EncryptSlotsBatch: the same for the plaintexts B200_BatchEncoder_EncodeBatch gives for `values` (host
   [count][values_per_item], int64_t when is_signed), encoded on the device with no plaintext handles in between: the mirror
   of DecryptSlotsBatch.  Same checks and HRESULTs as EncodeBatch and EncryptBatch, all made before any work, except: an
   encoder of another context, and parameters that do not batch, are E_INVALIDARG.
   Destinations must be distinct (E_INVALIDARG).  Destinations are untouched when a call is refused.  The sampling runs
   before the call takes the context, so other threads' operations proceed meanwhile. */
SEAL_C_FUNC B200_Encryptor_EncryptBatch(void *encryptor, uint64_t count, void **plains, const uint64_t *seeds, bool symmetric,
                                        void **destinations);
SEAL_C_FUNC B200_Encryptor_EncryptSlotsBatch(void *encryptor, void *encoder, uint64_t count, uint64_t values_per_item,
                                             const uint64_t *values, bool is_signed, const uint64_t *seeds, bool symmetric,
                                             void **destinations);

/* ---- debug aids (tests only; not part of the seal_fhe surface) ---- */
/* `count` (1 ... 64) per-handle calls of one kind run as if they had arrived together at the combiner: kind 0
   Evaluator_Multiply(a[i], b[i]), 1 Evaluator_Relinearize(a[i], keys), 2 Evaluator_ApplyGalois(a[i], galois_elt, keys) as
   Evaluator_RotateRows / RotateColumns combine it; results go to destinations[i], HRESULTs to hresults[i].  Every item is
   validated as its call validates it, then the combinable ones run as one leader's batch (compatible items together) on
   the calling thread, so the batch size and the graph state it meets are known.  COR_E_INVALIDOPERATION when combining is
   off (B200_NO_COMBINE). */
SEAL_C_FUNC B200_Evaluator_CombinedBatchDebug(void *thisptr, int kind, uint64_t count, void **encrypteds1, void **encrypteds2,
                                              void *keys, uint32_t galois_elt, void **destinations, long *hresults);
/* counts of what the combiner did with its batches, summed over the context's lanes: out[0] first sights of a graph shape
   (run kernel by kernel), [1] captures, [2] refused captures, [3] graph replays, [4] LRU evictions of a lane's graph,
   [5] batches run without a graph (graphs off, an operand that is also a destination of another shape, or a shape whose
   capture was refused) */
SEAL_C_FUNC B200_Context_GraphStatsDebug(void *context, uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif
