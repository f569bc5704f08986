// Instantiates every kernel of the MSM engine for GrumpkinG (one translation unit per curve so the
// four curves compile in parallel) and exports them through the curve's vtable.
#include "engine.cuh"
#include "field_op.cuh"
namespace b200 {
B200_DEFINE_CURVE_VTABLE(kVTableGrumpkin, GrumpkinG);
unsigned field_op_grumpkin(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                           const uint32_t* b, uint32_t* out) {
  return run_field_op<FGk>(ctx, op, n, a, b, out);
}
}  // namespace b200
