// TEST INFRASTRUCTURE — never linked into the product.
//
// The batched inner-product argument (IpaBatch, blitzar_b200/csrc/ipa.cuh) through the emulated
// kernel bodies, with the same contracts as b200_curve25519_prove_inner_products / _verify_. Each
// entry takes the number of built-in generators first (sxt_config::num_precomputed_generators, no
// fixed-base table), so that a batch can run with its round-0 generators read from the precomputed
// table in place or generated; the engine runs under its default options. The Python side is
// tests/emul/ipa_batch.py.
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine.cuh"

using namespace b200;

static EngineCtx batch_ctx(uint64_t num_builtin) {
  static std::vector<unsigned char> builtin;
  static uint64_t built = 0;
  if (num_builtin != built) {
    builtin.assign((size_t)(num_builtin ? num_builtin : 1) * kVTableEd25519.gen_bytes, 0);
    EngineCtx gen{0, MsmOptions(), nullptr, 0};
    launch_builtin_generators(gen, builtin.data(), 0, num_builtin);
    built = num_builtin;
  }
  EngineCtx ctx{0, MsmOptions(), num_builtin ? builtin.data() : nullptr, num_builtin};
  ctx.builtin_windows = num_builtin ? 1 : 0;
  return ctx;
}

extern "C" {
void emul_prove_inner_products(uint64_t num_builtin, uint32_t num_proofs, uint8_t* l_vectors,
                               uint8_t* r_vectors, uint8_t* ap_values, uint8_t* transcripts,
                               const uint64_t* n, const uint64_t* offsets,
                               const uint8_t* a_vectors, const uint8_t* b_vectors) {
  ipa_prove_batch(batch_ctx(num_builtin), num_proofs, l_vectors, r_vectors, ap_values, transcripts,
                  n, offsets, a_vectors, b_vectors);
}
uint32_t emul_verify_inner_products(uint64_t num_builtin, uint32_t num_proofs, int* results,
                                    uint8_t* transcripts, const uint64_t* n,
                                    const uint64_t* offsets, const uint8_t* b_vectors,
                                    const uint8_t* products, const uint8_t* a_commits,
                                    const uint8_t* l_vectors, const uint8_t* r_vectors,
                                    const uint8_t* ap_values) {
  return ipa_verify_batch(batch_ctx(num_builtin), num_proofs, results, transcripts, n, offsets,
                          b_vectors, products, a_commits, l_vectors, r_vectors, ap_values);
}
}
