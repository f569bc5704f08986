// TEST INFRASTRUCTURE — not product code.
//
// Thin C-ABI driver over the UNMODIFIED reference cpu-backend sources (compiled where they lie under
// a reference checkout by oracle/ref_build/Makefile; outputs go to oracle/_ref/ only). It exposes the
// reference's own CPU implementation of the MSM hot path as `ref_*` symbols so tests and
// bench.py's cpu_baseline / `--impl reference` leg can call it through ctypes.
//
// Every function below is a few lines of glue that mirrors what the reference's cbindings +
// cpu_backend do (file:line cited per function); all arithmetic is the reference's.
#include <cstdint>
#include <cstring>
#include <memory>
#include <numeric>
#include <vector>

#include "sxt/base/container/span.h"
#include "sxt/base/num/divide_up.h"
#include "sxt/base/num/fast_random_number_generator.h"
#include "sxt/cbindings/backend/computational_backend_utility.h"
#include "sxt/curve21/operation/add.h"
#include "sxt/curve21/operation/double.h"
#include "sxt/curve21/operation/neg.h"
#include "sxt/curve21/type/element_p3.h"
#include "sxt/curve_bng1/operation/add.h"
#include "sxt/curve_bng1/operation/double.h"
#include "sxt/curve_bng1/operation/neg.h"
#include "sxt/curve_bng1/random/element_p2.h"
#include "sxt/curve_bng1/type/conversion_utility.h"
#include "sxt/curve_bng1/type/element_affine.h"
#include "sxt/curve_bng1/type/element_p2.h"
#include "sxt/curve_g1/operation/add.h"
#include "sxt/curve_g1/operation/compression.h"
#include "sxt/curve_g1/operation/double.h"
#include "sxt/curve_g1/operation/neg.h"
#include "sxt/curve_g1/random/element_p2.h"
#include "sxt/curve_g1/type/compressed_element.h"
#include "sxt/curve_g1/type/conversion_utility.h"
#include "sxt/curve_g1/type/element_affine.h"
#include "sxt/curve_g1/type/element_p2.h"
#include "sxt/curve_gk/operation/add.h"
#include "sxt/curve_gk/operation/double.h"
#include "sxt/curve_gk/operation/neg.h"
#include "sxt/curve_gk/random/element_p2.h"
#include "sxt/curve_gk/type/conversion_utility.h"
#include "sxt/curve_gk/type/element_affine.h"
#include "sxt/curve_gk/type/element_p2.h"
#include "sxt/memory/management/managed_array.h"
#include "sxt/memory/resource/managed_device_resource.h"
#include "sxt/multiexp/base/exponent_sequence.h"
#include "sxt/multiexp/curve/multiexponentiation_cpu_driver.h"
#include "sxt/multiexp/curve/pippenger_multiproduct_solver.h"
#include "sxt/multiexp/pippenger/multiexponentiation.h"
#include "sxt/multiexp/pippenger2/in_memory_partition_table_accessor_utility.h"
#include "sxt/multiexp/pippenger2/multiexponentiation.h"
#include "sxt/multiexp/pippenger2/variable_length_multiexponentiation.h"
#include "sxt/base/num/ceil_log2.h"
#include "sxt/proof/inner_product/cpu_driver.h"
#include "sxt/proof/inner_product/proof_computation.h"
#include "sxt/proof/inner_product/proof_descriptor.h"
#include "sxt/proof/transcript/transcript.h"
#include "sxt/ristretto/base/byte_conversion.h"
#include "sxt/scalar25/type/element.h"
#include "sxt/ristretto/operation/compression.h"
#include "sxt/ristretto/type/compressed_element.h"
#include "sxt/seqcommit/generator/base_element.h"
#include "sxt/seqcommit/generator/cpu_generator.h"

using namespace sxt;

// layout-compatible with sxt_sequence_descriptor (cbindings/blitzar_api.h:115-131)
struct ref_sequence_descriptor {
  uint8_t element_nbytes;
  uint64_t n;
  const uint8_t* data;
  int is_signed;
};

// the body of mtxcrv::compute_multiexponentiation (sxt/multiexp/curve/multiexponentiation.h:128-142);
// that header cannot be included under g++ because it also pulls in the CUDA bucket-method headers.
template <class E>
static memmg::managed_array<E> ref_msm(basct::cspan<E> generators,
                                       basct::cspan<mtxb::exponent_sequence> exponents) {
  mtxcrv::pippenger_multiproduct_solver<E> solver;
  mtxcrv::multiexponentiation_cpu_driver<E> driver{&solver};
  return mtxpi::compute_multiexponentiation(
             driver, {static_cast<const void*>(generators.data()), generators.size(), sizeof(E)},
             exponents)
      .value()
      .template as_array<E>();
}

// cbindings/pedersen.cc:44-68 populate_exponent_sequence
static uint64_t to_sequences(std::vector<mtxb::exponent_sequence>& seqs,
                             const ref_sequence_descriptor* d, uint32_t num) {
  uint64_t longest = 0;
  seqs.resize(num);
  for (uint32_t i = 0; i < num; ++i) {
    longest = std::max(longest, d[i].n);
    seqs[i] = {.element_nbytes = d[i].element_nbytes,
               .n = d[i].n,
               .data = d[i].data,
               .is_signed = d[i].is_signed};
  }
  return longest;
}

extern "C" {

// sqcgn::cpu_get_generators (sxt/seqcommit/generator/cpu_generator.cc) — g(offset+i)
void ref_ristretto255_get_generators(void* generators, uint64_t num, uint64_t offset) {
  sqcgn::cpu_get_generators({static_cast<c21t::element_p3*>(generators), num}, offset);
}

// rstb::to_bytes (sxt/ristretto/base/byte_conversion.cc:74-129)
void ref_ristretto255_compress(uint8_t* out32, const void* p3, uint64_t num) {
  auto p = static_cast<const c21t::element_p3*>(p3);
  for (uint64_t i = 0; i < num; ++i) {
    rstb::to_bytes(out32 + 32 * i, p[i]);
  }
}

// cbindings/pedersen.cc:73-102 + cpu_backend.cc:117-123
void ref_curve25519_commit(uint8_t* commitments, uint32_t num_sequences,
                           const ref_sequence_descriptor* descriptors, const void* generators,
                           uint64_t offset_generators) {
  if (num_sequences == 0) {
    return;
  }
  std::vector<mtxb::exponent_sequence> seqs;
  auto n = to_sequences(seqs, descriptors, num_sequences);
  std::vector<c21t::element_p3> temp;
  basct::cspan<c21t::element_p3> gens;
  if (generators == nullptr) {
    temp.resize(n);
    sqcgn::cpu_get_generators(temp, offset_generators);
    gens = temp;
  } else {
    gens = {static_cast<const c21t::element_p3*>(generators), n};
  }
  auto values = ref_msm<c21t::element_p3>(gens, seqs);
  rsto::batch_compress({reinterpret_cast<rstt::compressed_element*>(commitments), num_sequences},
                       values);
}

// cbindings/pedersen.cc:107-133 + cpu_backend.cc:128-134. generators: 104-byte stride affine.
void ref_bls12_381_g1_commit(uint8_t* commitments48, uint32_t num_sequences,
                             const ref_sequence_descriptor* descriptors, const void* generators) {
  if (num_sequences == 0) {
    return;
  }
  std::vector<mtxb::exponent_sequence> seqs;
  auto n = to_sequences(seqs, descriptors, num_sequences);
  memmg::managed_array<cg1t::element_p2> gp(n);
  cg1t::batch_to_element_p2(
      gp, basct::cspan<cg1t::element_affine>{static_cast<const cg1t::element_affine*>(generators),
                                             n});
  auto values = ref_msm<cg1t::element_p2>(gp, seqs);
  cg1o::batch_compress(
      {reinterpret_cast<cg1t::compressed_element*>(commitments48), num_sequences}, values);
}

// cbindings/pedersen.cc:138-164 + cpu_backend.cc:139-145
void ref_bn254_g1_commit(void* commitments, uint32_t num_sequences,
                         const ref_sequence_descriptor* descriptors, const void* generators) {
  if (num_sequences == 0) {
    return;
  }
  std::vector<mtxb::exponent_sequence> seqs;
  auto n = to_sequences(seqs, descriptors, num_sequences);
  memmg::managed_array<cn1t::element_p2> gp(n);
  cn1t::batch_to_element_p2(
      gp, basct::cspan<cn1t::element_affine>{static_cast<const cn1t::element_affine*>(generators),
                                             n});
  auto values = ref_msm<cn1t::element_p2>(gp, seqs);
  cn1t::batch_to_element_affine(
      {static_cast<cn1t::element_affine*>(commitments), num_sequences}, values);
}

// cbindings/pedersen.cc:169-195 + cpu_backend.cc:150-156
void ref_grumpkin_commit(void* commitments, uint32_t num_sequences,
                         const ref_sequence_descriptor* descriptors, const void* generators) {
  if (num_sequences == 0) {
    return;
  }
  std::vector<mtxb::exponent_sequence> seqs;
  auto n = to_sequences(seqs, descriptors, num_sequences);
  memmg::managed_array<cgkt::element_p2> gp(n);
  cgkt::batch_to_element_p2(
      gp, basct::cspan<cgkt::element_affine>{static_cast<const cgkt::element_affine*>(generators),
                                             n});
  auto values = ref_msm<cgkt::element_p2>(gp, seqs);
  cgkt::batch_to_element_affine(
      {static_cast<cgkt::element_affine*>(commitments), num_sequences}, values);
}

// Test-input generators: fast_random_number_generator{i+1,i+2} -> generate_random_element, the
// scheme of cbindings/pedersen.t.cc:81-123 and benchmark/multi_exp_pip/benchmark.m.cc:89-92.
// curve_id: 1 bls12-381, 2 bn254, 3 grumpkin. out_p2 / out_affine may be null.
void ref_random_elements(unsigned curve_id, void* out_p2, void* out_affine, uint64_t n,
                         uint64_t first) {
  for (uint64_t k = 0; k < n; ++k) {
    auto i = first + k;
    basn::fast_random_number_generator rng{i + 1, i + 2};
    if (curve_id == 1) {
      cg1t::element_p2 e;
      cg1rn::generate_random_element(e, rng);
      if (out_p2)
        static_cast<cg1t::element_p2*>(out_p2)[k] = e;
      if (out_affine)
        cg1t::to_element_affine(static_cast<cg1t::element_affine*>(out_affine)[k], e);
    } else if (curve_id == 2) {
      cn1t::element_p2 e;
      cn1rn::generate_random_element(e, rng);
      if (out_p2)
        static_cast<cn1t::element_p2*>(out_p2)[k] = e;
      if (out_affine)
        cn1t::to_element_affine(static_cast<cn1t::element_affine*>(out_affine)[k], e);
    } else {
      cgkt::element_p2 e;
      cgkrn::generate_random_element(e, rng);
      if (out_p2)
        static_cast<cgkt::element_p2*>(out_p2)[k] = e;
      if (out_affine)
        cgkt::to_element_affine(static_cast<cgkt::element_affine*>(out_affine)[k], e);
    }
  }
}

// Normalise projective results so two engines' fixed-MSM outputs can be compared
// (SURVEY.md §8c parity definition). ristretto -> 32 B; bls -> 48 B compressed; bn254/grumpkin ->
// affine struct (72 B, padding zeroed).
void ref_normalize(unsigned curve_id, uint8_t* out, const void* in_projective, uint64_t n) {
  for (uint64_t k = 0; k < n; ++k) {
    if (curve_id == 0) {
      rstb::to_bytes(out + 32 * k, static_cast<const c21t::element_p3*>(in_projective)[k]);
    } else if (curve_id == 1) {
      cg1t::compressed_element c;
      cg1o::compress(c, static_cast<const cg1t::element_p2*>(in_projective)[k]);
      std::memcpy(out + 48 * k, &c, 48);
    } else if (curve_id == 2) {
      cn1t::element_affine a;
      std::memset(static_cast<void*>(&a), 0, sizeof(a));
      cn1t::to_element_affine(a, static_cast<const cn1t::element_p2*>(in_projective)[k]);
      std::memset(out + 72 * k, 0, 72);
      std::memcpy(out + 72 * k, &a, 65);
    } else {
      cgkt::element_affine a;
      std::memset(static_cast<void*>(&a), 0, sizeof(a));
      cgkt::to_element_affine(a, static_cast<const cgkt::element_p2*>(in_projective)[k]);
      std::memset(out + 72 * k, 0, 72);
      std::memcpy(out + 72 * k, &a, 65);
    }
  }
}

} // extern "C"

// Fixed-base MSM: cpu_backend::make_partition_table_accessor (cpu_backend.cc:203-218) followed by
// cpu_backend::fixed_multiexponentiation (cpu_backend.cc:223-262). mode 0 = fixed width
// (element_num_bytes), 1 = packed (output_bit_table), 2 = vlen (output_bit_table + output_lengths).
template <class U, class T>
static void fixed_impl(void* res, const void* generators, unsigned num_generators,
                       unsigned window_width, int mode, unsigned element_num_bytes,
                       const unsigned* output_bit_table, const unsigned* output_lengths,
                       unsigned num_outputs, unsigned n, const uint8_t* scalars) {
  auto accessor = mtxpp2::make_in_memory_partition_table_accessor<U, T>(
      basct::cspan<T>{static_cast<const T*>(generators), num_generators}, basm::alloc_t{},
      window_width);
  basct::span<T> res_span{static_cast<T*>(res), num_outputs};
  if (mode == 0) {
    basct::cspan<uint8_t> s{scalars, size_t{element_num_bytes} * num_outputs * n};
    mtxpp2::multiexponentiate<T>(res_span, *accessor, element_num_bytes, s);
  } else if (mode == 1) {
    basct::cspan<unsigned> bt{output_bit_table, num_outputs};
    auto nb = basn::divide_up<size_t>(
        std::accumulate(output_bit_table, output_bit_table + num_outputs, 0u), 8);
    basct::cspan<uint8_t> s{scalars, nb * n};
    mtxpp2::multiexponentiate<T>(res_span, *accessor, bt, s);
  } else {
    basct::cspan<unsigned> bt{output_bit_table, num_outputs};
    basct::cspan<unsigned> ol{output_lengths, num_outputs};
    auto s = cbnbck::make_scalars_span(scalars, bt, ol);
    mtxpp2::multiexponentiate<T>(res_span, *accessor, bt, ol, s);
  }
}

// The reference's partition-table file of a handle (sxt_multiexp_handle_write_to_file ->
// in_memory_partition_table_accessor::write_to_file, in_memory_partition_table_accessor.h:98-105):
// [u32 window_width][table of compact elements].
template <class U, class T>
static void write_table_impl(const char* filename, const void* generators, unsigned num_generators,
                             unsigned window_width) {
  auto accessor = mtxpp2::make_in_memory_partition_table_accessor<U, T>(
      basct::cspan<T>{static_cast<const T*>(generators), num_generators}, basm::alloc_t{},
      window_width);
  accessor->write_to_file(filename);
}

extern "C" {
void ref_write_partition_table(unsigned curve_id, const char* filename, const void* generators,
                               unsigned num_generators, unsigned window_width) {
  switch (curve_id) {
  case 0:
    write_table_impl<c21t::compact_element, c21t::element_p3>(filename, generators, num_generators,
                                                              window_width);
    break;
  case 1:
    write_table_impl<cg1t::compact_element, cg1t::element_p2>(filename, generators, num_generators,
                                                              window_width);
    break;
  case 2:
    write_table_impl<cn1t::compact_element, cn1t::element_p2>(filename, generators, num_generators,
                                                              window_width);
    break;
  default:
    write_table_impl<cgkt::compact_element, cgkt::element_p2>(filename, generators, num_generators,
                                                              window_width);
    break;
  }
}
void ref_fixed_msm(unsigned curve_id, void* res, const void* generators, unsigned num_generators,
                   unsigned window_width, int mode, unsigned element_num_bytes,
                   const unsigned* output_bit_table, const unsigned* output_lengths,
                   unsigned num_outputs, unsigned n, const uint8_t* scalars) {
  switch (curve_id) {
  case 0:
    fixed_impl<c21t::compact_element, c21t::element_p3>(res, generators, num_generators,
                                                        window_width, mode, element_num_bytes,
                                                        output_bit_table, output_lengths,
                                                        num_outputs, n, scalars);
    break;
  case 1:
    fixed_impl<cg1t::compact_element, cg1t::element_p2>(res, generators, num_generators,
                                                        window_width, mode, element_num_bytes,
                                                        output_bit_table, output_lengths,
                                                        num_outputs, n, scalars);
    break;
  case 2:
    fixed_impl<cn1t::compact_element, cn1t::element_p2>(res, generators, num_generators,
                                                        window_width, mode, element_num_bytes,
                                                        output_bit_table, output_lengths,
                                                        num_outputs, n, scalars);
    break;
  default:
    fixed_impl<cgkt::compact_element, cgkt::element_p2>(res, generators, num_generators,
                                                        window_width, mode, element_num_bytes,
                                                        output_bit_table, output_lengths,
                                                        num_outputs, n, scalars);
    break;
  }
}

// A fresh Merlin transcript with the given label, as a caller of the proof API creates it
// (sxt/proof/transcript/transcript.cc:41-53); 203 bytes.
void ref_transcript_new(uint8_t* transcript203, const char* label) {
  prft::transcript t{label};
  static_assert(sizeof(prft::transcript) == 203);
  std::memcpy(transcript203, &t, 203);
}
// Draw a 32-byte challenge (used by tests to check that two transcripts are in the same state)
void ref_transcript_challenge(uint8_t* out32, uint8_t* transcript203, const char* label) {
  auto& t = *reinterpret_cast<prft::transcript*>(transcript203);
  t.challenge_bytes({out32, 32}, label);
}

// cbindings/inner_product_proof.cc:101-130 with the cpu backend (cpu_backend.cc:171-181)
void ref_prove_inner_product(uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
                             uint8_t* transcript203, uint64_t n, uint64_t generators_offset,
                             const uint8_t* a_vector, const uint8_t* b_vector) {
  auto n_lg2 = static_cast<size_t>(basn::ceil_log2(n));
  auto np = 1ull << n_lg2;
  std::vector<c21t::element_p3> gens(np + 1);
  sqcgn::cpu_get_generators(gens, generators_offset);
  prfip::proof_descriptor descriptor{
      .b_vector = {reinterpret_cast<const s25t::element*>(b_vector), n},
      .g_vector = {gens.data(), np},
      .q_value = gens.data() + np};
  prfip::cpu_driver drv;
  auto fut = prfip::prove_inner_product(
      {reinterpret_cast<rstt::compressed_element*>(l_vector), n_lg2},
      {reinterpret_cast<rstt::compressed_element*>(r_vector), n_lg2},
      *reinterpret_cast<s25t::element*>(ap_value),
      *reinterpret_cast<prft::transcript*>(transcript203), drv, descriptor,
      {reinterpret_cast<const s25t::element*>(a_vector), n});
  (void)fut;
}

// cbindings/inner_product_proof.cc:135-167 with the cpu backend (cpu_backend.cc:186-198)
int ref_verify_inner_product(uint8_t* transcript203, uint64_t n, uint64_t generators_offset,
                             const uint8_t* b_vector, const uint8_t* product,
                             const uint8_t* a_commit160, const uint8_t* l_vector,
                             const uint8_t* r_vector, const uint8_t* ap_value) {
  auto n_lg2 = static_cast<size_t>(basn::ceil_log2(n));
  auto np = 1ull << n_lg2;
  std::vector<c21t::element_p3> gens(np + 1);
  sqcgn::cpu_get_generators(gens, generators_offset);
  prfip::proof_descriptor descriptor{
      .b_vector = {reinterpret_cast<const s25t::element*>(b_vector), n},
      .g_vector = {gens.data(), np},
      .q_value = gens.data() + np};
  prfip::cpu_driver drv;
  return prfip::verify_inner_product(
             *reinterpret_cast<prft::transcript*>(transcript203), drv, descriptor,
             *reinterpret_cast<const s25t::element*>(product),
             *reinterpret_cast<const c21t::element_p3*>(a_commit160),
             {reinterpret_cast<const rstt::compressed_element*>(l_vector), n_lg2},
             {reinterpret_cast<const rstt::compressed_element*>(r_vector), n_lg2},
             *reinterpret_cast<const s25t::element*>(ap_value))
      .value();
}

// sizes the tests rely on (sizeof of the reference types)
unsigned ref_sizeof(unsigned curve_id, int what) { // what: 0 projective, 1 affine, 2 compact
  switch (curve_id * 4 + what) {
  case 0:
    return sizeof(c21t::element_p3);
  case 2:
    return sizeof(c21t::compact_element);
  case 4:
    return sizeof(cg1t::element_p2);
  case 5:
    return sizeof(cg1t::element_affine);
  case 6:
    return sizeof(cg1t::compact_element);
  case 8:
    return sizeof(cn1t::element_p2);
  case 9:
    return sizeof(cn1t::element_affine);
  case 10:
    return sizeof(cn1t::compact_element);
  case 12:
    return sizeof(cgkt::element_p2);
  case 13:
    return sizeof(cgkt::element_affine);
  case 14:
    return sizeof(cgkt::compact_element);
  }
  return 0;
}
} // extern "C"
