// Point checks and decoding (points.cuh) for bls12-381 G1 and G2 in their own translation unit, so
// that the square roots and subgroup checks compile in parallel with the curve units and leave them
// untouched.
#include "points.cuh"
namespace b200 {
void check_points_bls12381(const EngineCtx& ctx, unsigned curve_id, uint8_t* valid,
                           const void* points, uint64_t n) {
  if (curve_id == kBls12381)
    launch(CheckPointsBody<Bls12381G1>{(const unsigned char*)points, valid}, n, ctx.s);
  else
    launch(CheckPointsBody<Bls12381G2>{(const unsigned char*)points, valid}, n, ctx.s);
}
void decode_points_bls12381(const EngineCtx& ctx, unsigned curve_id, void* out_p2, uint8_t* valid,
                            const void* encoded, uint64_t n) {
  const unsigned char* e = (const unsigned char*)encoded;
  if (curve_id == kBls12381)
    launch(DecodePointsBody<Bls12381G1>{e, (unsigned char*)out_p2, valid}, n, ctx.s);
  else
    launch(DecodePointsBody<Bls12381G2>{e, (unsigned char*)out_p2, valid}, n, ctx.s);
}
unsigned field_op_sqrt_bls12381(const EngineCtx& ctx, unsigned field, uint64_t n, const uint32_t* a,
                                uint32_t* out) {
  return field == 1 ? run_sqrt_op<FBls>(ctx, n, a, out) : run_sqrt_op<Fp2Bls>(ctx, n, a, out);
}
}  // namespace b200
