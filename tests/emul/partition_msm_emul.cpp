// TEST INFRASTRUCTURE — never linked into the product.
//
// Fixed-base MSMs over a handle that carries a partition table (ptable.cuh, partition_msm.cuh,
// CurveOps::fixed_device's routing) as serial host loops, reached through the same per-curve vtables
// as api.cu. Compiled into the emulation library next to emul.cpp (blitzar_b200/build.py build_emul);
// Python side in tests/partition_msm_emul.py.
#include <algorithm>
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine.cuh"

using namespace b200;

static const CurveVTable& pmsm_vt(unsigned curve_id) {
  switch (curve_id) {
  case 0: return kVTableEd25519;
  case 1: return kVTableBls12381;
  case 2: return kVTableBn254;
  default: return kVTableGrumpkin;
  }
}

extern "C" {
// handle_new over num_gens projective ABI generators (no fixed-base table), its partition table of
// width window_width built chunk_groups groups at a time (0 = all at once; window_width 0 = no table),
// and a fixed MSM under the partition policy (mode as in b200_fixed_msm_device). Results as
// projective ABI structs to res.
void emul_partition_fixed_msm(unsigned curve_id, void* res, const void* generators_proj,
                              unsigned num_gens, unsigned window_width, uint64_t chunk_groups,
                              unsigned policy, int mode, unsigned element_num_bytes,
                              const unsigned* bit_table, const unsigned* lengths,
                              unsigned num_outputs, unsigned n, const uint8_t* scalars) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  ctx.partition_policy = policy;
  const CurveVTable& V = pmsm_vt(curve_id);
  std::vector<unsigned char> gens((size_t)(num_gens ? num_gens : 1) * V.gen_bytes);
  V.ingest_projective(ctx, generators_proj, gens.data(), num_gens);
  Handle h{curve_id, num_gens, gens.data()};
  std::vector<unsigned char> table;
  if (window_width) {
    const uint64_t groups = (num_gens + window_width - 1) / window_width;
    const uint64_t step = chunk_groups ? chunk_groups : std::max<uint64_t>(groups, 1);
    table.resize(std::max<size_t>(1, ((size_t)groups << window_width) * V.gen_bytes));
    for (uint64_t g = 0; g < groups; g += step)
      V.partition_gens(ctx, gens.data(), num_gens, window_width, g, std::min(step, groups - g),
                       table.data() + ((size_t)g << window_width) * V.gen_bytes);
    h.ptable = table.data();
    h.ptable_w = window_width;
    h.ptable_groups = groups;
  }
  unsigned rows = n;
  if (mode == 2) {
    rows = 0;
    for (unsigned j = 0; j < num_outputs; ++j) rows = std::max(rows, lengths[j]);
  }
  V.fixed_device(ctx, res, nullptr, &h, mode, element_num_bytes, bit_table, lengths, num_outputs,
                 rows, scalars);
}

// the outputs partition_route sends to a table of width window_width (policy as above) for outputs
// of the given widths and lengths over a handle of num_gens generators without a fixed-base table:
// their indices to routed, their count returned
unsigned emul_partition_route(unsigned curve_id, unsigned num_gens, unsigned window_width,
                              unsigned policy, const unsigned* widths, const unsigned* lengths,
                              unsigned num_outputs, unsigned* routed) {
  EngineCtx ctx{0, MsmOptions(), nullptr, 0};
  ctx.partition_policy = policy;
  unsigned char dummy = 0;
  Handle h{curve_id, num_gens, nullptr};
  h.ptable = &dummy;  // only its presence is read
  h.ptable_w = window_width;
  std::vector<ColumnDesc> cols(num_outputs);
  for (unsigned j = 0; j < num_outputs; ++j) {
    cols[j] = ColumnDesc();
    cols[j].bit_width = widths[j];
    cols[j].n = lengths[j];
  }
  std::vector<u32> r;
  switch (curve_id) {
  case 0: r = CurveOps<Ed25519>::partition_route(ctx, &h, cols); break;
  case 1: r = CurveOps<Bls12381G1>::partition_route(ctx, &h, cols); break;
  case 2: r = CurveOps<Bn254G1>::partition_route(ctx, &h, cols); break;
  default: r = CurveOps<GrumpkinG>::partition_route(ctx, &h, cols); break;
  }
  std::copy(r.begin(), r.end(), routed);
  return (unsigned)r.size();
}
}
