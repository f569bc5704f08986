// TEST INFRASTRUCTURE — never linked into the product.
//
// Point checks and decoding (blitzar_b200/csrc/points.cuh) through the emulated kernel bodies, with the
// contracts of b200_check_points and b200_decode_points (host pointers, the number of valid points
// returned). The Python side is tests/emul/points.py.
#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine_api.cuh"

using namespace b200;

namespace {
uint64_t count_valid(const uint8_t* valid, uint64_t n) {
  uint64_t count = 0;
  for (uint64_t i = 0; i < n; ++i)
    count += valid[i] != 0;
  return count;
}
}  // namespace

extern "C" uint64_t emul_check_points(unsigned curve_id, uint8_t* valid, const void* points,
                                      uint64_t n) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  check_points(ctx, curve_id, valid, points, n);
  return count_valid(valid, n);
}

extern "C" uint64_t emul_decode_points(unsigned curve_id, void* out_p2, uint8_t* valid,
                                       const void* encoded, uint64_t n) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  decode_points(ctx, curve_id, out_p2, valid, encoded, n);
  return count_valid(valid, n);
}
