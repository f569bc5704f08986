// Point checks and decoding (points.cuh) for bn254 G1, Grumpkin and bn254 G2 in their own translation
// unit, so that they compile in parallel with the curve units and leave them untouched.
#include "points.cuh"
namespace b200 {
void check_points_bn254(const EngineCtx& ctx, unsigned curve_id, uint8_t* valid, const void* points,
                        uint64_t n) {
  const unsigned char* p = (const unsigned char*)points;
  if (curve_id == kBn254)
    launch(CheckPointsBody<Bn254G1>{p, valid}, n, ctx.s);
  else if (curve_id == kGrumpkin)
    launch(CheckPointsBody<GrumpkinG>{p, valid}, n, ctx.s);
  else
    launch(CheckPointsBody<Bn254G2>{p, valid}, n, ctx.s);
}
void decode_points_bn254(const EngineCtx& ctx, unsigned curve_id, void* out_p2, uint8_t* valid,
                         const void* encoded, uint64_t n) {
  const unsigned char* e = (const unsigned char*)encoded;
  unsigned char* o = (unsigned char*)out_p2;
  if (curve_id == kBn254)
    launch(DecodePointsBody<Bn254G1>{e, o, valid}, n, ctx.s);
  else if (curve_id == kGrumpkin)
    launch(DecodePointsBody<GrumpkinG>{e, o, valid}, n, ctx.s);
  else
    launch(DecodePointsBody<Bn254G2>{e, o, valid}, n, ctx.s);
}
}  // namespace b200
