// Instantiates every kernel of the MSM engine for Bn254G1 (one translation unit per curve so the
// four curves compile in parallel) and exports them through the curve's vtable.
#include "engine.cuh"
#include "field_op.cuh"
namespace b200 {
B200_DEFINE_CURVE_VTABLE(kVTableBn254, Bn254G1);
unsigned field_op_bn254(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                        const uint32_t* b, uint32_t* out) {
  return run_field_op<FBn>(ctx, op, n, a, b, out);
}
}  // namespace b200
