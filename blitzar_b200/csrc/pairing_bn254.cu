// The bn254 pairing (pairing.cuh) in its own translation unit, so that it compiles in parallel with the
// curve units and leaves them untouched.
#include "pairing.cuh"
namespace b200 {
void multi_pairing_bn254(const EngineCtx& ctx, void* out, uint32_t num_products,
                         const uint32_t* lengths, const void* g1, const void* g2) {
  multi_pairing<BnTower>(ctx, out, num_products, lengths, g1, g2);
}
unsigned field_op_bn254_gt(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                           const uint32_t* b, uint32_t* out) {
  return run_fp12_op<BnTower>(ctx, op, n, a, b, out);
}
}  // namespace b200
