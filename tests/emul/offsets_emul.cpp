// TEST INFRASTRUCTURE — never linked into the product.
//
// Commitments with per-column generator offsets (CurveOps::commit_device_offsets, GenLayout) as
// serial host loops, reached through the same per-curve vtables as api.cu. Compiled into the
// emulation library next to emul.cpp (blitzar_b200/build.py build_emul); Python side in
// tests/commit_offsets_emul.py. The engine options of these calls are set here, independently of
// emul.cpp's.
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine_api.cuh"

using namespace b200;

static const CurveVTable& offsets_vt(unsigned curve_id) {
  switch (curve_id) {
  case 0: return kVTableEd25519;
  case 1: return kVTableBls12381;
  case 2: return kVTableBn254;
  default: return kVTableGrumpkin;
  }
}

static MsmOptions g_offsets_opt;
static unsigned g_offsets_ranges = 1;
static std::vector<unsigned char> g_offsets_builtin;  // built-in generators + their table
static uint64_t g_offsets_num_builtin = 0;
static unsigned g_offsets_builtin_c = 0;

extern "C" {
// upload pieces, sort-pass and column-group entry limits (0 = default), batch-affine pair levels
// (-1 = automatic), fixed-base table policy (0 cost model, 1 always, 2 never), and
// sxt_config::num_precomputed_generators with a table of the given window (0 = none)
void emul_offsets_configure(unsigned num_ranges, unsigned long long range_entries,
                            unsigned long long group_entries, int pair_levels,
                            unsigned table_policy, uint64_t num_builtin, unsigned window_bits) {
  g_offsets_opt = MsmOptions();
  g_offsets_ranges = num_ranges ? num_ranges : 1;
  if (range_entries)
    g_offsets_opt.max_range_entries = range_entries;
  if (group_entries)
    g_offsets_opt.max_group_entries = group_entries;
  g_offsets_opt.pair_levels = pair_levels;
  g_offsets_opt.table_policy = table_policy;
  g_offsets_builtin.clear();
  g_offsets_num_builtin = num_builtin;
  g_offsets_builtin_c = window_bits;
  if (num_builtin == 0)
    return;
  const unsigned windows = window_bits ? 256 / window_bits + 1 : 1;
  g_offsets_builtin.resize((size_t)num_builtin * windows * offsets_vt(0).gen_bytes);
  EngineCtx ctx{0, g_offsets_opt, nullptr, 0};
  launch_builtin_generators(ctx, g_offsets_builtin.data(), 0, num_builtin);
  offsets_vt(0).build_table(ctx, g_offsets_builtin.data(), num_builtin, window_bits, windows);
}

// same contract as b200_commit_device_with_offsets, with host pointers standing in for device
// pointers (offsets null = all 0)
void emul_commit_offsets(unsigned curve_id, void* out_commitments, uint32_t num,
                         const sxt_sequence_descriptor* d, const void* generators,
                         const uint64_t* offsets) {
  if (num == 0) return;
  EngineCtx ctx{0, g_offsets_opt,
                g_offsets_builtin.empty() ? nullptr : g_offsets_builtin.data(),
                g_offsets_num_builtin};
  ctx.builtin_window_bits = g_offsets_builtin_c;
  ctx.builtin_windows =
      g_offsets_builtin_c ? 256 / g_offsets_builtin_c + 1 : (g_offsets_num_builtin ? 1 : 0);
  offsets_vt(curve_id).commit_device_offsets(ctx, out_commitments, nullptr, num, d, generators,
                                             offsets, false, g_offsets_ranges, nullptr, nullptr);
}
}
