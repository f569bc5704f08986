// TEST INFRASTRUCTURE — never linked into the product.
//
// Pairing products (blitzar_b200/csrc/pairing.cuh) through the emulated kernel bodies, with the contract
// of b200_multi_pairing_device and host pointers standing in for device pointers. The Python side is
// tests/emul/pairing.py.
#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine_api.cuh"

using namespace b200;

extern "C" void emul_multi_pairing(unsigned curve_id, void* out, uint32_t num_products,
                                   const uint32_t* lengths, const void* g1, const void* g2) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  multi_pairing(ctx, curve_id, out, num_products, lengths, g1, g2);
}
