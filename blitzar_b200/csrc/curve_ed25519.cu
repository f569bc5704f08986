// Instantiates every kernel of the MSM engine for Ed25519 (one translation unit per curve so the
// four curves compile in parallel) and exports them through the curve's vtable.
#include "engine.cuh"
#include "ipa.cuh"
namespace b200 {
B200_DEFINE_CURVE_VTABLE(kVTableEd25519, Ed25519);
void launch_builtin_generators(const EngineCtx& ctx, void* gens, uint64_t first, uint64_t n) {
  launch(BuiltinGeneratorBody{(Ed25519::Gen*)gens, first}, n, ctx.s);
}
unsigned selftest_lane_arithmetic(const EngineCtx& ctx, unsigned warps, unsigned seed) {
#ifdef B200_LANE_TAIL
  DevBuf<u32> bad(1, ctx.s);
  dev_zero(bad.p, sizeof(u32), ctx.s);
  launch(lane10::SelfTestBody{seed, bad.p}, (u64)warps * 32, ctx.s);
  u32 host = 0;
  copy_d2h(&host, bad.p, sizeof(u32), ctx.s);
  stream_sync(ctx.s);
  return host;
#else
  (void)ctx;
  (void)warps;
  (void)seed;
  return 0;
#endif
}
unsigned selftest_sort(const EngineCtx& ctx, const sxt_sequence_descriptor* d, unsigned num,
                       unsigned window_bits) {
  std::vector<ColumnDesc> cols(num);
  for (unsigned i = 0; i < num; ++i) {
    cols[i] = ColumnDesc{};
    cols[i].base = d[i].data;
    cols[i].row_stride = d[i].element_nbytes;
    cols[i].bit_width = 8u * d[i].element_nbytes;
    cols[i].n = (u32)d[i].n;
    cols[i].is_signed = d[i].is_signed ? 1u : 0u;
  }
  return sort_selftest(ctx.s, std::move(cols), window_bits);
}
void ipa_prove(const EngineCtx& ctx, uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
               uint8_t* transcript203, uint64_t n, uint64_t generators_offset,
               const uint8_t* a_vector, const uint8_t* b_vector) {
  Ipa::prove(ctx, l_vector, r_vector, ap_value, transcript203, n, generators_offset, a_vector,
             b_vector);
}
int ipa_verify(const EngineCtx& ctx, uint8_t* transcript203, uint64_t n,
               uint64_t generators_offset, const uint8_t* b_vector, const uint8_t* product,
               const uint8_t* a_commit160, const uint8_t* l_vector, const uint8_t* r_vector,
               const uint8_t* ap_value) {
  int result = 0;  // a batch of one
  IpaBatch::verify(ctx, 1, &result, transcript203, &n, &generators_offset, b_vector, product,
                   a_commit160, l_vector, r_vector, ap_value);
  return result;
}
void ipa_prove_batch(const EngineCtx& ctx, uint32_t num_proofs, uint8_t* l_vectors,
                     uint8_t* r_vectors, uint8_t* ap_values, uint8_t* transcripts,
                     const uint64_t* n, const uint64_t* generators_offsets,
                     const uint8_t* a_vectors, const uint8_t* b_vectors) {
  IpaBatch::prove(ctx, num_proofs, l_vectors, r_vectors, ap_values, transcripts, n,
                  generators_offsets, a_vectors, b_vectors);
}
uint32_t ipa_verify_batch(const EngineCtx& ctx, uint32_t num_proofs, int* results,
                          uint8_t* transcripts, const uint64_t* n,
                          const uint64_t* generators_offsets, const uint8_t* b_vectors,
                          const uint8_t* products, const uint8_t* a_commits,
                          const uint8_t* l_vectors, const uint8_t* r_vectors,
                          const uint8_t* ap_values) {
  return IpaBatch::verify(ctx, num_proofs, results, transcripts, n, generators_offsets, b_vectors,
                          products, a_commits, l_vectors, r_vectors, ap_values);
}
}  // namespace b200
