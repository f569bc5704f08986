// Instantiates every kernel of the MSM engine for Ed25519 (one translation unit per curve so the
// four curves compile in parallel) and exports them through the curve's vtable.
#include "engine.cuh"
#include "ipa.cuh"
namespace b200 {
B200_DEFINE_CURVE_VTABLE(kVTableEd25519, Ed25519);

// Self-test body (b200_selftest_field_multiply): F25519::mul, the carry-chain schedule the kernels
// run, against the plain 64-bit schedule F25519::mul_ref, limb for limb (both fold the same
// 512-bit product to the same loosely reduced residue). Operand a of thread t is edge case t % 10,
// b is edge case t / 10 % 10 (9 = random), so every pair of edge cases meets; beyond the first
// 100 threads one limb of a or b is also forced to all ones.
struct FieldMulSelfTestBody {
  static constexpr int kBlock = 128;
  u32 seed;
  u32* mismatches;
  static B200_HD u32 rnd(u64& st) {
    st ^= st << 13;
    st ^= st >> 7;
    st ^= st << 17;
    return (u32)(st >> 16);
  }
  static B200_HD void operand(F25519::E& x, u32 k, u64& st) {
    for (int i = 0; i < 8; ++i)
      x.l[i] = rnd(st);
    const u32 ones = 0xffffffffu;
    switch (k) {
    case 0: for (int i = 0; i < 8; ++i) x.l[i] = 0; break;                                 // 0
    case 1: for (int i = 0; i < 8; ++i) x.l[i] = i == 0; break;                            // 1
    case 2: for (int i = 0; i < 8; ++i) x.l[i] = ones; x.l[0] = 0xffffffecu; x.l[7] >>= 1; break;  // p - 1
    case 3: for (int i = 0; i < 8; ++i) x.l[i] = ones; x.l[0] = 0xffffffedu; x.l[7] >>= 1; break;  // p
    case 4: for (int i = 0; i < 8; ++i) x.l[i] = ones; x.l[7] >>= 1; break;                // p + 18
    case 5: for (int i = 0; i < 8; ++i) x.l[i] = 0; x.l[7] = 0x80000000u; break;           // 2^255
    case 6: for (int i = 0; i < 8; ++i) x.l[i] = ones; break;                              // 2^256 - 1
    case 7: for (int i = 0; i < 8; ++i) x.l[i] = ones; x.l[0] = 0xffffffdau; break;        // 2^256 - 38
    case 8: for (int i = 0; i < 8; ++i) x.l[i] = i < 4 ? ones : 0u; break;                 // 2^128 - 1
    default: break;
    }
  }
  B200_HD void operator()(u64 tid) const {
    u64 st = ((u64)seed << 32) ^ (0x9E3779B97F4A7C15ull * (tid + 1));
    F25519::E a, b, got, want;
    operand(a, (u32)(tid % 10), st);
    operand(b, (u32)(tid / 10 % 10), st);
    const u32 f = (u32)(tid / 100);
    if (f % 3 == 1)
      a.l[f / 3 % 8] = 0xffffffffu;
    if (f % 3 == 2)
      b.l[f / 3 % 8] = 0xffffffffu;
    F25519::mul(got, a, b);
    F25519::mul_ref(want, a, b);
    u32 diff = 0;
    for (int i = 0; i < 8; ++i)
      diff |= got.l[i] ^ want.l[i];
    if (diff)
      B200_ATOMIC_ADD(mismatches, 1u);
  }
};
unsigned selftest_field_multiply(const EngineCtx& ctx, unsigned threads, unsigned seed) {
  DevBuf<u32> bad(1, ctx.s);
  dev_zero(bad.p, sizeof(u32), ctx.s);
  launch(FieldMulSelfTestBody{seed, bad.p}, threads, ctx.s);
  u32 host = 0;
  copy_d2h(&host, bad.p, sizeof(u32), ctx.s);
  stream_sync(ctx.s);
  return host;
}
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
