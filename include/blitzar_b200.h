/* blitzar_b200 — C ABI of the H100-native (sm_90a) MSM / Pedersen-commitment backend.
 *
 * Part 1 ("sxt_*") is the drop-in boundary: the same 18 symbols, struct layouts and argument
 * meaning as the reference's cbindings/blitzar_api.h (line numbers of the reference declaration
 * each entry replaces are cited). A consumer that was linked against libblitzar (e.g. the
 * blitzar-sys crate, rust/blitzar-sys/build.rs:21-56) links against libblitzar_b200.so unchanged.
 * All pointers are caller-owned HOST memory; calls block until results are written.
 * Misuse aborts the process with a message on stderr (reference convention, blitzar_api.h:230-237).
 *
 * Part 2 ("b200_*") is an extension for callers that already hold inputs in HBM and for the
 * one-process-per-GPU multi-GPU layout (device-resident inputs, partial results, device events).
 */
#ifndef BLITZAR_B200_H
#define BLITZAR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- constants (blitzar_api.h:25-34) ---- */
#define SXT_CPU_BACKEND 1
#define SXT_GPU_BACKEND 2
#define SXT_CURVE_RISTRETTO255 0
#define SXT_CURVE_BLS_381 1
#define SXT_CURVE_BN_254 2
#define SXT_CURVE_GRUMPKIN 3
#define SXT_FIELD_SCALAR255 0
#define SXT_FIELD_GRUMPKIN 1

/* ---- types (blitzar_api.h:37-131) ---- */
struct sxt_config { int backend; uint64_t num_precomputed_generators; };
struct sxt_ristretto255_compressed { uint8_t ristretto_bytes[32]; };
struct sxt_bls12_381_g1_compressed { uint8_t g1_bytes[48]; };
struct sxt_curve25519_scalar { uint8_t bytes[32]; };
struct sxt_transcript { uint8_t bytes[203]; };
/* ed25519 extended coordinates, radix-2^51 limbs (not necessarily reduced) */
struct sxt_ristretto255 { uint64_t X[5]; uint64_t Y[5]; uint64_t Z[5]; uint64_t T[5]; };
/* Montgomery-form limbs, R = 2^384. NOTE: arrays of generators passed to the bls12-381 commitment
 * entry point are read with a 104-byte stride ({X, Y, uint8 infinity} padded), exactly as the
 * reference does (cbindings/pedersen.cc:215-217); see INTEGRATION.md "ABI quirks". */
struct sxt_bls12_381_g1 { uint64_t X[6]; uint64_t Y[6]; };
struct sxt_bls12_381_g1_p2 { uint64_t X[6]; uint64_t Y[6]; uint64_t Z[6]; };
/* Montgomery-form limbs, R = 2^256 */
struct sxt_bn254_g1 { uint64_t X[4]; uint64_t Y[4]; uint8_t infinity; };
struct sxt_bn254_g1_p2 { uint64_t X[4]; uint64_t Y[4]; uint64_t Z[4]; };
struct sxt_grumpkin { uint64_t X[4]; uint64_t Y[4]; uint8_t infinity; };
struct sxt_grumpkin_p2 { uint64_t X[4]; uint64_t Y[4]; uint64_t Z[4]; };
/* one column of scalars: n little-endian integers of element_nbytes (1..32) bytes; signed columns
 * are two's complement with element_nbytes a power of two <= 16 */
struct sxt_sequence_descriptor {
  uint8_t element_nbytes;
  uint64_t n;
  const uint8_t* data;
  int is_signed;
};
/* blitzar_api.h:133-183 (sumcheck is outside this library's scope; the type is kept for ABI) */
struct sumcheck_descriptor {
  const void* mles;
  const void* product_table;
  const unsigned* product_terms;
  unsigned n;
  unsigned num_mles;
  unsigned num_products;
  unsigned num_product_terms;
  unsigned round_degree;
};
struct sxt_multiexp_handle; /* opaque: device-resident generators of one curve */

/* ---- Part 1: drop-in entry points ---- */

/* blitzar_api.h:200. 0 on success. Only SXT_GPU_BACKEND is provided (non-zero for anything else);
 * env BLITZAR_BACKEND=gpu|cpu overrides config->backend as in cbindings/backend.cc:72-89. */
int sxt_init(const struct sxt_config* config);

/* blitzar_api.h:243. commitments[i] = sum_j a_ij * g(offset_generators + j), built-in generators */
void sxt_curve25519_compute_pedersen_commitments(struct sxt_ristretto255_compressed* commitments,
                                                 uint32_t num_sequences,
                                                 const struct sxt_sequence_descriptor* descriptors,
                                                 uint64_t offset_generators);
/* blitzar_api.h:284 */
void sxt_curve25519_compute_pedersen_commitments_with_generators(
    struct sxt_ristretto255_compressed* commitments, uint32_t num_sequences,
    const struct sxt_sequence_descriptor* descriptors, const struct sxt_ristretto255* generators);
/* blitzar_api.h:324 (generators: 104-byte stride, see above) */
void sxt_bls12_381_g1_compute_pedersen_commitments_with_generators(
    struct sxt_bls12_381_g1_compressed* commitments, uint32_t num_sequences,
    const struct sxt_sequence_descriptor* descriptors, const struct sxt_bls12_381_g1* generators);
/* blitzar_api.h:364 (affine Montgomery outputs; identity = {0, R mod p, infinity = 1}) */
void sxt_bn254_g1_uncompressed_compute_pedersen_commitments_with_generators(
    struct sxt_bn254_g1* commitments, uint32_t num_sequences,
    const struct sxt_sequence_descriptor* descriptors, const struct sxt_bn254_g1* generators);
/* blitzar_api.h:404 */
void sxt_grumpkin_uncompressed_compute_pedersen_commitments_with_generators(
    struct sxt_grumpkin* commitments, uint32_t num_sequences,
    const struct sxt_sequence_descriptor* descriptors, const struct sxt_grumpkin* generators);

/* blitzar_api.h:440. ABI quirk kept: the second argument is the COUNT and the third the OFFSET,
 * as implemented and tested by the reference (cbindings/get_generators.cc:32-33), although its
 * header names them the other way round. Returns 1 if generators == NULL and count > 0. */
int sxt_ristretto255_get_generators(struct sxt_ristretto255* generators, uint64_t num_generators,
                                    uint64_t offset_generators);
/* blitzar_api.h:477. one_commit = g(0) + ... + g(n-1) (identity for n = 0) */
int sxt_curve25519_get_one_commit(struct sxt_ristretto255* one_commit, uint64_t n);

/* blitzar_api.h:566 / :611. Inner-product argument over g(generators_offset ..) with Q = g[np],
 * np = 2^ceil(log2 n); `transcript` is the caller's Merlin transcript (203 bytes), advanced in
 * place exactly as the reference advances it. verify returns 1 / 0. */
void sxt_curve25519_prove_inner_product(struct sxt_ristretto255_compressed* l_vector,
                                        struct sxt_ristretto255_compressed* r_vector,
                                        struct sxt_curve25519_scalar* ap_value,
                                        struct sxt_transcript* transcript, uint64_t n,
                                        uint64_t generators_offset,
                                        const struct sxt_curve25519_scalar* a_vector,
                                        const struct sxt_curve25519_scalar* b_vector);
int sxt_curve25519_verify_inner_product(struct sxt_transcript* transcript, uint64_t n,
                                        uint64_t generators_offset,
                                        const struct sxt_curve25519_scalar* b_vector,
                                        const struct sxt_curve25519_scalar* product,
                                        const struct sxt_ristretto255* a_commit,
                                        const struct sxt_ristretto255_compressed* l_vector,
                                        const struct sxt_ristretto255_compressed* r_vector,
                                        const struct sxt_curve25519_scalar* ap_value);

/* blitzar_api.h:631-655. generators: sxt_ristretto255 / *_p2 arrays per curve_id; copied to HBM. */
struct sxt_multiexp_handle* sxt_multiexp_handle_new(unsigned curve_id, const void* generators,
                                                    unsigned n);
struct sxt_multiexp_handle* sxt_multiexp_handle_new_from_file(unsigned curve_id,
                                                              const char* filename);
void sxt_multiexp_handle_write_to_file(const struct sxt_multiexp_handle* handle,
                                       const char* filename);
void sxt_multiexp_handle_free(struct sxt_multiexp_handle* handle);

/* blitzar_api.h:685. scalars: n rows, row i = num_outputs x element_num_bytes bytes; res: projective
 * elements (sxt_ristretto255 / *_p2), one per output. */
void sxt_fixed_multiexponentiation(void* res, const struct sxt_multiexp_handle* handle,
                                   unsigned element_num_bytes, unsigned num_outputs, unsigned n,
                                   const uint8_t* scalars);
/* blitzar_api.h:712. bit-packed rows: output j owns output_bit_table[j] consecutive bits */
void sxt_fixed_packed_multiexponentiation(void* res, const struct sxt_multiexp_handle* handle,
                                          const unsigned* output_bit_table, unsigned num_outputs,
                                          unsigned n, const uint8_t* scalars);
/* blitzar_api.h:741. as packed, output j uses only the first output_lengths[j] rows */
void sxt_fixed_vlen_multiexponentiation(void* res, const struct sxt_multiexp_handle* handle,
                                        const unsigned* output_bit_table,
                                        const unsigned* output_lengths, unsigned num_outputs,
                                        const uint8_t* scalars);
/* blitzar_api.h:766. Outside this library's scope (SURVEY §2 #20): aborts with a message. */
void sxt_prove_sumcheck(void* polynomials, void* evaluation_point, unsigned field_id,
                        const struct sumcheck_descriptor* descriptor, void* transcript_callback,
                        void* transcript_context);

/* ---- Part 2: device-resident extension ---- */

/* Bind the calling thread / library to a CUDA device before sxt_init (default: current device). */
void b200_set_device(int device);
/* Number of kernels this library has launched so far in this process. */
unsigned long long b200_launch_count(void);
/* sizeof of the internal accumulator point of a curve (for partial-result buffers). */
unsigned b200_point_bytes(unsigned curve_id);
/* Raw device buffers on the library's stream-ordered pool. */
void* b200_malloc(uint64_t bytes);
void b200_free(void* device_ptr);
void b200_memcpy_h2d(void* device_dst, const void* host_src, uint64_t bytes);
void b200_memcpy_d2h(void* host_dst, const void* device_src, uint64_t bytes);
void b200_synchronize(void);
/* The cudaStream_t every kernel of the engine is launched on (e.g. to wrap it as an external stream
 * of another runtime so that collectives can be ordered against it without host synchronisation). */
void* b200_stream(void);
/* CUDA events on the library's stream (the stream every kernel of the engine is launched on). */
void* b200_event_create(void);
void b200_event_record(void* event);
float b200_event_elapsed_ms(void* start, void* stop); /* synchronises on stop */
void b200_event_destroy(void* event);

/* Variable-base MSM with every input already in HBM, laid out exactly as the host ABI lays it out
 * (descriptors[i].data and generators are DEVICE pointers; generators == NULL selects the built-in
 * ristretto generators at offset_generators). Results:
 *   out_commitments (device or NULL): canonical commitments, as the sxt_*_commitments calls write
 *   out_partials    (device or NULL): internal accumulator points (b200_point_bytes each), to be
 *                                     combined across GPUs with b200_combine_partials_device
 * Enqueued on the library stream; returns without synchronising. */
void b200_commit_device(unsigned curve_id, void* out_commitments, void* out_partials,
                        uint32_t num_sequences, const struct sxt_sequence_descriptor* descriptors,
                        const void* generators, uint64_t offset_generators);
/* The host-pointer commitment call (same copy / compute pipeline as the sxt_*_commitments entry
 * points: descriptors[i].data and generators are HOST pointers) that leaves one internal accumulator
 * point per column in DEVICE memory instead of canonical commitments — the per-rank half of a
 * generator-range-sharded multi-GPU commitment. Synchronises before returning. */
void b200_commit_host_partials(unsigned curve_id, void* out_partials, uint32_t num_sequences,
                               const struct sxt_sequence_descriptor* descriptors,
                               const void* generators, uint64_t offset_generators);
/* commitments[j] = sum_i a_ij * g(offsets[j] + i), all columns in one engine pass. generators ==
 * NULL: built-in ristretto generators (curve 0 only); else the caller's array in the layout / stride
 * of the curve's sxt_*_with_generators call. offsets == NULL: all 0. commitments in the layout of
 * the matching sxt_* call. Host pointers; synchronises. */
void b200_compute_pedersen_commitments_with_offsets(unsigned curve_id, void* commitments,
                                                    uint32_t num_sequences,
                                                    const struct sxt_sequence_descriptor* descriptors,
                                                    const void* generators, const uint64_t* offsets);
/* as b200_commit_device (device descriptors / generators, out_commitments and / or out_partials,
 * no synchronisation); offsets is a HOST array */
void b200_commit_device_with_offsets(unsigned curve_id, void* out_commitments, void* out_partials,
                                     uint32_t num_sequences,
                                     const struct sxt_sequence_descriptor* descriptors,
                                     const void* generators, const uint64_t* offsets);
/* as the three sxt_fixed_* calls (host scalars; mode 0 fixed width, 1 packed, 2 vlen), partial
 * accumulator points to device memory */
void b200_fixed_msm_host_partials(void* out_partials, const struct sxt_multiexp_handle* handle,
                                  int mode, unsigned element_num_bytes,
                                  const unsigned* output_bit_table, const unsigned* output_lengths,
                                  unsigned num_outputs, unsigned n, const uint8_t* scalars);
/* sxt_multiexp_handle_new over generators that already sit in HBM (projective ABI structs) */
struct sxt_multiexp_handle* b200_multiexp_handle_new_device(unsigned curve_id,
                                                            const void* generators_dev,
                                                            unsigned n);
/* out[j] = sum_r partials[r * count + j]; writes canonical commitments (device pointer). */
void b200_combine_partials_device(unsigned curve_id, void* out_commitments, const void* partials,
                                  uint32_t num_parts, uint32_t count);
/* Fixed-base MSM with the scalar table already in HBM (mode 0: fixed width; 1: packed; 2: vlen as
 * in the three sxt_fixed_* calls). out_res / out_partials as above (res = projective ABI structs). */
void b200_fixed_msm_device(void* out_res, void* out_partials,
                           const struct sxt_multiexp_handle* handle, int mode,
                           unsigned element_num_bytes, const unsigned* output_bit_table,
                           const unsigned* output_lengths, unsigned num_outputs, unsigned n,
                           const uint8_t* scalars);
/* as b200_combine_partials_device but writes projective ABI structs */
void b200_combine_partials_projective_device(unsigned curve_id, void* out_res,
                                             const void* partials, uint32_t num_parts,
                                             uint32_t count);
/* Synthetic benchmark / test inputs generated in HBM (device pointer out): the generators the
 * reference's own benchmarks use — ristretto255: built-in g(first + i) as sxt_ristretto255 structs;
 * other curves: generate_random_element with fast_random_number_generator{i + 1, i + 2}
 * (cbindings/pedersen.t.cc:81-123, benchmark/multi_exp_pip/benchmark.m.cc:84-95), as projective
 * *_p2 structs (projective != 0, handle input) or affine structs at the commitment stride. */
void b200_synthetic_generators_device(unsigned curve_id, void* out_generators, uint64_t n,
                                      uint64_t first, int projective);
/* The reference's partition table (2^w compact elements per group of w generators, identity-padded)
 * of n projective ABI generators already in HBM, written to out_table_dev (device, 2^w * ceil(n/w) *
 * compact bytes). window_width 1..24; 0 = the reference's default (BLITZAR_PARTITION_WINDOW_WIDTH,
 * else 16). Enqueued on the library stream; returns without synchronising. */
void b200_partition_table_device(unsigned curve_id, void* out_table_dev, const void* generators_dev,
                                 uint64_t n, unsigned window_width);
/* Writes the handle as the reference's handle file ([u32 window_width][table],
 * in_memory_partition_table_accessor.h:98-105), readable by libblitzar's
 * sxt_multiexp_handle_new_from_file and by this library's. Synchronises before returning. */
void b200_multiexp_handle_write_partition_table(const struct sxt_multiexp_handle* handle,
                                                const char* filename, unsigned window_width);
/* Attaches to the handle the partition table of width window_width (1..24; 0 = the reference's
 * default, BLITZAR_PARTITION_WINDOW_WIDTH, else 16) over its generators, kept in HBM: 2^w subset sums
 * per group of w generators (per shard with BLITZAR_B200_DEVICES). Fixed-base calls over the handle
 * then answer the outputs that are cheaper that way (narrow widths) by table lookups. Replaces a
 * table attached before. Returns the width attached, or 0 when the table would take more than 40 %
 * of the free HBM; the handle then has no table and works as before. Synchronises. */
unsigned b200_multiexp_handle_add_partition_table(struct sxt_multiexp_handle* handle,
                                                  unsigned window_width);
/* Width of the handle's partition table, or 0 when it has none. */
unsigned b200_multiexp_handle_partition_window(const struct sxt_multiexp_handle* handle);
/* Proves num_proofs independent inner-product arguments in one call. Proof p, and transcripts[p], are
 * byte-identical to sxt_curve25519_prove_inner_product(l, r, &ap_values[p], &transcripts[p], n[p],
 * generators_offsets[p], a_p, b_p) called alone. Arrays are flattened in proof order: with
 * k_p = ceil(log2 n_p), proof p's L / R values start at the sum of k_q over the proofs q < p, its a / b
 * scalars at the sum of n_q. Every round of every proof runs in one engine pass per round of the
 * longest proof. Host pointers; synchronises. num_proofs == 0: no-op. */
void b200_curve25519_prove_inner_products(
    uint32_t num_proofs, struct sxt_ristretto255_compressed* l_vectors /* sum k_p */,
    struct sxt_ristretto255_compressed* r_vectors /* sum k_p */,
    struct sxt_curve25519_scalar* ap_values /* num_proofs */,
    struct sxt_transcript* transcripts /* num_proofs, advanced in place */, const uint64_t* n,
    const uint64_t* generators_offsets, const struct sxt_curve25519_scalar* a_vectors /* sum n_p */,
    const struct sxt_curve25519_scalar* b_vectors /* sum n_p */);
/* results[p] = what sxt_curve25519_verify_inner_product returns for proof p alone (1 / 0), transcripts
 * advanced as that call advances them; arrays flattened as for b200_curve25519_prove_inner_products
 * (products, a_commits, ap_values: one per proof). One engine pass for the whole batch. Returns the
 * number of accepted proofs. Host pointers; synchronises. */
uint32_t b200_curve25519_verify_inner_products(
    uint32_t num_proofs, int* results, struct sxt_transcript* transcripts, const uint64_t* n,
    const uint64_t* generators_offsets, const struct sxt_curve25519_scalar* b_vectors /* sum n_p */,
    const struct sxt_curve25519_scalar* products, const struct sxt_ristretto255* a_commits,
    const struct sxt_ristretto255_compressed* l_vectors /* sum k_p */,
    const struct sxt_ristretto255_compressed* r_vectors /* sum k_p */,
    const struct sxt_curve25519_scalar* ap_values);
/* Self-test of the warp-cooperative (lane-sliced) field arithmetic of the tail kernels against the
 * per-thread arithmetic on `warps` warps of pseudo-random and edge-case operands: returns the number
 * of mismatching checks (0 = pass). */
unsigned b200_selftest_lane_arithmetic(unsigned warps, unsigned seed);
/* Test hook: one field operation of the device arithmetic on each of n elements, out[i] = op(a[i],
 * b[i]). Operands and results are little-endian u32 limbs. Fields: 0 curve25519 Fp (8 limbs, loosely
 * reduced: any value below 2^256), 1 bls12-381 Fp (12), 2 bn254 Fp (8), 3 grumpkin Fp (8), 4 the
 * ristretto255 scalars mod l (8), 5 curve25519 Fp lane-sliced over 10 lanes (10 limbs of radix
 * 2^25.5). Fields 1-4 hold Montgomery residues. Ops: 0 add, 1 sub, 2 neg, 3 dbl, 4 mul, 5 mul_ref,
 * 6 sqr (fields 0-4); field 0: 7 mul_lat, 8 canonical, 9 is_negative (1 limb out), 10 invert,
 * 11 pow22523, 12 from_radix51 (10 limbs in: 5 x u64), 13 to_radix51 (10 limbs out),
 * 14 sqrt_ratio_m1 (a = u, b = v; out: x, then the was-square flag); fields 1-4: 10 invert,
 * 15 invert_eea, 16 from_mont, 17 to_mont, 18 lexicographically_largest (1 limb out); field 5:
 * 0 add, 4 mul, 11 pow22523, 19 carry1, 20 sub2p, 21 sub4p, 22 slice (8 limbs in), 23 gather (8
 * limbs out). b is read only by binary ops (add, sub, mul, mul_ref, mul_lat, sqrt_ratio_m1, sub2p,
 * sub4p). Host pointers; synchronises. Returns 0, or ~0u when the field does not offer op. */
unsigned b200_field_op(unsigned field, unsigned op, uint64_t n, const uint32_t* a,
                       const uint32_t* b, uint32_t* out);
/* Self-test of the binned bucket sort: sorts the (term, window) entries of the device-resident
 * columns (window width `window_bits`, 0 = automatic) with the atomic and the binned path and returns
 * the number of buckets whose end offset or entry multiset differs (0 = pass; ~0u when the binned path
 * does not apply to the shape). */
unsigned b200_selftest_sort(const struct sxt_sequence_descriptor* columns, unsigned num,
                            unsigned window_bits);
/* Per-launch CUDA-event timing of the dominant kernel (level-1 bucket accumulation) on the library
 * stream: enable, run, then read the total milliseconds and launch count since the last read. */
void b200_profile_accumulate(int enable);
void b200_profile_read(float* total_ms, unsigned* launches);
/* Engine tuning (0 keeps the default): window bits c, first-level and cascade chunk lengths. */
void b200_set_tuning(unsigned window_bits, unsigned chunk1, unsigned chunkn);
/* Bucket-reduction group sizes (powers of two; 0 keeps the default): first level, later levels. */
void b200_set_reduce_groups(unsigned g1, unsigned gn);

#ifdef __cplusplus
}
#endif
#endif /* BLITZAR_B200_H */
