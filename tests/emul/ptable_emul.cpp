// TEST INFRASTRUCTURE — never linked into the product.
//
// The partition-table kernel bodies (blitzar_b200/csrc/ptable.cuh) as serial host loops, reached
// through the same per-curve vtables as api.cu. Compiled into the emulation library next to
// emul.cpp (blitzar_b200/build.py build_emul); Python side in tests/partition_tables.py.
#include <algorithm>
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine_api.cuh"

using namespace b200;

static const CurveVTable& ptable_vt(unsigned curve_id) {
  switch (curve_id) {
  case 0: return kVTableEd25519;
  case 1: return kVTableBls12381;
  case 2: return kVTableBn254;
  default: return kVTableGrumpkin;
  }
}

extern "C" {
// the reference's partition table (without the u32 window-width header) of n projective ABI
// generators, built `chunk_groups` groups at a time (0 = all at once), as b200_partition_table_device
// does on the device
void emul_partition_table(unsigned curve_id, void* out_table, const void* generators_proj,
                          uint64_t n, unsigned window_width, uint64_t chunk_groups) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  const CurveVTable& V = ptable_vt(curve_id);
  std::vector<unsigned char> gens((size_t)(n ? n : 1) * V.gen_bytes);
  V.ingest_projective(ctx, generators_proj, gens.data(), n);
  const uint64_t groups = (n + window_width - 1) / window_width;
  const uint64_t step = chunk_groups ? chunk_groups : (groups ? groups : 1);
  const size_t group_bytes = (size_t)V.abi_compact_bytes << window_width;
  for (uint64_t g = 0; g < groups; g += step)
    V.partition_table(ctx, gens.data(), n, window_width, g, std::min(step, groups - g),
                      (unsigned char*)out_table + g * group_bytes);
}
}
