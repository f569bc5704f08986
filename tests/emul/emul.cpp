// TEST INFRASTRUCTURE — never linked into the product.
//
// Builds the product's kernel bodies (blitzar_b200/csrc/*.cuh) as SERIAL HOST LOOPS
// (-DB200_EMULATE: launch() iterates the thread index, device memory is malloc) so that the whole
// MSM pipeline — digit recoding, counting sort, chunked accumulation cascade, bucket reduction,
// window combination, canonicalisation — can be checked against the oracle in a container without
// a GPU. The product library (api.cu) has no such path and aborts without a GPU.
//
// The per-curve translation units of the product (csrc/curve_*.cu) are compiled as host C++ with
// emul_prefix.h force-included and reached through the same type-erased vtables api.cu uses. Every
// entry runs under the one set of engine options that emul_configure sets; the Python side is
// tests/emul/harness.py.
#include <algorithm>
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine.cuh"
#include "../../blitzar_b200/csrc/scalar25.h"

using namespace b200;

static MsmOptions g_opt;
static unsigned g_ranges = 1;
static unsigned g_table_c = 0;  // fixed-base table window of emul_fixed handles (0 = no table)
static unsigned g_partition_policy = 0;
static std::vector<unsigned char> g_builtin;  // built-in generators and their fixed-base table
static uint64_t g_num_builtin = 0;
static unsigned g_builtin_c = 0;
static EngineCtx make_ctx() {
  EngineCtx ctx{0, g_opt, g_builtin.empty() ? nullptr : g_builtin.data(), g_num_builtin};
  ctx.builtin_window_bits = g_builtin_c;
  ctx.builtin_windows = g_builtin_c ? 256 / g_builtin_c + 1 : (g_num_builtin ? 1 : 0);
  ctx.partition_policy = g_partition_policy;
  return ctx;
}

// projective ABI generators -> the device generator layout, room for `windows` table windows
static std::vector<unsigned char> ingest(const EngineCtx& ctx, const CurveVTable& V,
                                         const void* generators_proj, uint64_t n,
                                         unsigned windows = 1) {
  std::vector<unsigned char> gens((size_t)(n ? n : 1) * windows * V.gen_bytes);
  V.ingest_projective(ctx, generators_proj, gens.data(), n);
  return gens;
}

// the first group and the group count of each chunk of `chunk_groups` groups (0 = one chunk)
template <class F> static void for_chunks(uint64_t groups, uint64_t chunk_groups, F f) {
  const uint64_t step = chunk_groups ? chunk_groups : std::max<uint64_t>(groups, 1);
  for (uint64_t g = 0; g < groups; g += step)
    f(g, std::min(step, groups - g));
}

extern "C" {
// Every engine option of the entries below; the Python side gives each its default when not set.
// 0 = the product's default for window_bits, chunk1, chunkn, range_entries and group_entries;
// pair_levels -1 = automatic; table_policy and partition_policy 0 = cost model, 1 = always,
// 2 = never; table_window: fixed-base table of emul_fixed handles (0 = none); num_builtin:
// sxt_config::num_precomputed_generators with a fixed-base table of builtin_window (0 = none).
void emul_configure(unsigned num_ranges, unsigned window_bits, unsigned chunk1, unsigned chunkn,
                    unsigned long long range_entries, unsigned long long group_entries,
                    int pair_levels, unsigned pair_batch, unsigned scatter_window_major,
                    unsigned normalize, unsigned table_policy, unsigned table_window,
                    unsigned partition_policy, uint64_t num_builtin, unsigned builtin_window) {
  g_opt = MsmOptions();
  g_opt.window_bits = window_bits;
  g_opt.chunk1 = chunk1;
  if (chunkn)
    g_opt.chunkn = chunkn;
  if (range_entries)
    g_opt.max_range_entries = range_entries;
  if (group_entries)
    g_opt.max_group_entries = group_entries;
  g_opt.pair_levels = pair_levels;
  g_opt.pair_batch = pair_batch;
  g_opt.scatter_window_major = scatter_window_major;
  g_opt.normalize_gens = normalize;
  g_opt.table_policy = table_policy;
  g_ranges = num_ranges ? num_ranges : 1;
  g_table_c = table_window;
  g_partition_policy = partition_policy;
  g_builtin.clear();
  g_num_builtin = num_builtin;
  g_builtin_c = builtin_window;
  if (num_builtin == 0)
    return;
  const CurveVTable& V = curve_vtable(SXT_CURVE_RISTRETTO255);
  const unsigned windows = builtin_window ? 256 / builtin_window + 1 : 1;
  g_builtin.resize((size_t)num_builtin * windows * V.gen_bytes);
  EngineCtx ctx{0, g_opt, nullptr, 0};
  launch_builtin_generators(ctx, g_builtin.data(), 0, num_builtin);
  V.build_table(ctx, g_builtin.data(), num_builtin, builtin_window, windows);
}

// same contract as b200_commit_device, with host pointers standing in for device pointers
void emul_commit(unsigned curve_id, void* out_commitments, void* out_partials, uint32_t num,
                 const sxt_sequence_descriptor* d, const void* generators, uint64_t offset) {
  if (num == 0) return;
  curve_vtable(curve_id).commit_device(make_ctx(), out_commitments, out_partials, num, d,
                                       generators, offset, g_ranges, nullptr, nullptr);
}
// same contract as b200_commit_device_with_offsets, with host pointers standing in for device
// pointers (offsets null = all 0)
void emul_commit_offsets(unsigned curve_id, void* out_commitments, void* out_partials,
                         uint32_t num, const sxt_sequence_descriptor* d, const void* generators,
                         const uint64_t* offsets) {
  if (num == 0) return;
  curve_vtable(curve_id).commit_device_offsets(make_ctx(), out_commitments, out_partials, num, d,
                                               generators, offsets, false, g_ranges, nullptr,
                                               nullptr);
}
void emul_combine_partials(unsigned curve_id, void* out_commitments, const void* partials,
                           uint32_t num_parts, uint32_t count) {
  EngineCtx ctx = make_ctx();
  const CurveVTable& V = curve_vtable(curve_id);
  std::vector<unsigned char> sum((size_t)count * V.point_bytes);
  V.sum_parts(ctx, partials, num_parts, count, sum.data());
  V.store(ctx, sum.data(), out_commitments, count, true);
}
unsigned emul_point_bytes(unsigned curve_id) { return curve_vtable(curve_id).point_bytes; }

// handle_new over num_gens projective ABI generators with the configured fixed-base table window
// and, for partition_window != 0, a partition table of that width built chunk_groups groups at a
// time (0 = all at once); then a fixed MSM (mode as in b200_fixed_msm_device). Results as
// projective ABI structs to res.
void emul_fixed(unsigned curve_id, void* res, const void* generators_proj, unsigned num_gens,
                unsigned partition_window, uint64_t chunk_groups, int mode,
                unsigned element_num_bytes, const unsigned* bit_table, const unsigned* lengths,
                unsigned num_outputs, unsigned n, const uint8_t* scalars) {
  EngineCtx ctx = make_ctx();
  const CurveVTable& V = curve_vtable(curve_id);
  const unsigned windows = g_table_c ? 256 / g_table_c + 1 : 1;
  std::vector<unsigned char> gens = ingest(ctx, V, generators_proj, num_gens, windows);
  V.build_table(ctx, gens.data(), num_gens, g_table_c, windows);
  Handle h{curve_id, num_gens, gens.data()};
  h.window_bits = g_table_c;
  h.windows = windows;
  std::vector<unsigned char> table;
  if (partition_window) {
    const uint64_t groups = (num_gens + partition_window - 1) / partition_window;
    table.resize(std::max<size_t>(1, ((size_t)groups << partition_window) * V.gen_bytes));
    for_chunks(groups, chunk_groups, [&](uint64_t g, uint64_t count) {
      V.partition_gens(ctx, gens.data(), num_gens, partition_window, g, count,
                       table.data() + ((size_t)g << partition_window) * V.gen_bytes);
    });
    h.ptable = table.data();
    h.ptable_w = partition_window;
    h.ptable_groups = groups;
  }
  V.fixed_device(ctx, res, nullptr, &h, mode, element_num_bytes, bit_table, lengths, num_outputs,
                 n, scalars);
}

// the outputs partition_route sends to a table of width window_width for outputs of the given
// widths and lengths over a handle of num_gens generators without a fixed-base table: their
// indices to routed, their count returned
unsigned emul_partition_route(unsigned curve_id, unsigned num_gens, unsigned window_width,
                              const unsigned* widths, const unsigned* lengths,
                              unsigned num_outputs, unsigned* routed) {
  EngineCtx ctx = make_ctx();
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

// the reference's partition table (without the u32 window-width header) of n projective ABI
// generators, built `chunk_groups` groups at a time (0 = all at once), as
// b200_partition_table_device does on the device
void emul_partition_table(unsigned curve_id, void* out_table, const void* generators_proj,
                          uint64_t n, unsigned window_width, uint64_t chunk_groups) {
  EngineCtx ctx = make_ctx();
  const CurveVTable& V = curve_vtable(curve_id);
  std::vector<unsigned char> gens = ingest(ctx, V, generators_proj, n);
  const size_t group_bytes = (size_t)V.abi_compact_bytes << window_width;
  for_chunks((n + window_width - 1) / window_width, chunk_groups, [&](uint64_t g, uint64_t count) {
    V.partition_table(ctx, gens.data(), n, window_width, g, count,
                      (unsigned char*)out_table + g * group_bytes);
  });
}

// n ristretto255 ABI generators -> device generators (Ed25519::Gen, 128 bytes each), normalised
// (normalisation option on) or as IngestBody writes them; returns the Z = 0 flag of the
// normalisation
unsigned emul_ingest_generators(const void* raw, uint64_t n, void* out_gens) {
  if (!g_opt.normalize_gens) {
    launch(IngestBody<Ed25519, false>{(const unsigned char*)raw, (Ed25519::Gen*)out_gens}, n, 0);
    return 0;
  }
  u32 invalid = 0;
  ingest_normalized(0, (const unsigned char*)raw, (Ed25519::Gen*)out_gens, IngestMap{}, n, &invalid);
  return invalid;
}
// generators recovered from a reference partition-table image, as projective ABI structs
void emul_ingest_compact(unsigned curve_id, const void* table, unsigned window_width, uint64_t n,
                         void* out_proj) {
  EngineCtx ctx = make_ctx();
  const CurveVTable& V = curve_vtable(curve_id);
  std::vector<unsigned char> gens((size_t)(n ? n : 1) * V.gen_bytes);
  V.ingest_compact_table(ctx, table, window_width, gens.data(), n);
  V.gens_to_projective(ctx, gens.data(), out_proj, n);
}

void emul_get_generators(void* out160, uint64_t num, uint64_t offset) {
  EngineCtx ctx = make_ctx();
  const CurveVTable& V = curve_vtable(SXT_CURVE_RISTRETTO255);
  std::vector<unsigned char> g((num ? num : 1) * V.gen_bytes);
  launch_builtin_generators(ctx, g.data(), offset, num);
  V.gens_to_projective(ctx, g.data(), out160, num);
}
// same contract as b200_synthetic_generators_device (host memory)
void emul_synth_generators(unsigned curve_id, void* out, uint64_t n, uint64_t first, int projective) {
  curve_vtable(curve_id).synth_generators(make_ctx(), out, n, first, projective != 0);
}

// inner-product argument through the emulated kernels (same contracts as the sxt_* entry points)
void emul_prove_inner_product(uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
                              uint8_t* transcript203, uint64_t n, uint64_t offset,
                              const uint8_t* a_vector, const uint8_t* b_vector) {
  ipa_prove(make_ctx(), l_vector, r_vector, ap_value, transcript203, n, offset, a_vector, b_vector);
}
int emul_verify_inner_product(uint8_t* transcript203, uint64_t n, uint64_t offset,
                              const uint8_t* b_vector, const uint8_t* product,
                              const uint8_t* a_commit160, const uint8_t* l_vector,
                              const uint8_t* r_vector, const uint8_t* ap_value) {
  return ipa_verify(make_ctx(), transcript203, n, offset, b_vector, product, a_commit160, l_vector,
                    r_vector, ap_value);
}
}

// same contract as b200_field_op, run on the CPU (~0u for the lane-sliced field, which is device only)
extern "C" unsigned emul_field_op(unsigned field, unsigned op, uint64_t n, const uint32_t* a,
                                  const uint32_t* b, uint32_t* out) {
  return field_op(make_ctx(), field, op, n, a, b, out);
}

// The host scalar arithmetic of scalar25.h (inner-product challenges and verifier exponents) on n
// elements of 8 little-endian u32 limbs: 0 sc_reduce(a), 1 sc_mul(a, b), 2 sc_mul_mont(sc_to_mont(a),
// b), 3 sc_add, 4 sc_sub, 5 sc_neg(a), 6 sc_inv(a), 7 sc_inner_product of all n pairs (one result).
// Returns 0, or ~0u for an unknown op.
extern "C" unsigned emul_scalar_op(unsigned op, uint64_t n, const uint32_t* a, const uint32_t* b,
                                   uint32_t* out) {
  if (op == 7) {
    sc_store((uint8_t*)out, sc_inner_product((const uint8_t*)a, (const uint8_t*)b, n));
    return 0;
  }
  if (op > 7)
    return ~0u;
  for (uint64_t i = 0; i < n; ++i) {
    const Sc x = sc_load((const uint8_t*)(a + 8 * i));
    const Sc y = b ? sc_load((const uint8_t*)(b + 8 * i)) : sc_zero();
    Sc r;
    switch (op) {
    case 0: r = sc_reduce(x); break;
    case 1: r = sc_mul(x, y); break;
    case 2: r = sc_mul_mont(sc_to_mont(x), y); break;
    case 3: r = sc_add(x, y); break;
    case 4: r = sc_sub(x, y); break;
    case 5: r = sc_neg(x); break;
    default: r = sc_inv(x); break;
    }
    sc_store((uint8_t*)(out + 8 * i), r);
  }
  return 0;
}
