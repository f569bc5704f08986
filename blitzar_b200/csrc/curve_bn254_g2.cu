// Instantiates every kernel of the MSM engine for Bn254G2 (one translation unit per curve so the
// curves compile in parallel) and exports them through the curve's vtable.
#include "engine.cuh"
#include "field_op.cuh"
namespace b200 {
B200_DEFINE_CURVE_VTABLE(kVTableBn254G2, Bn254G2);
unsigned field_op_bn254_g2(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                           const uint32_t* b, uint32_t* out) {
  return run_field_op<Fp2Bn>(ctx, op, n, a, b, out);
}
}  // namespace b200
