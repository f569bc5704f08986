// Type-erased per-curve entry points of the MSM engine. api.cu sees only this header, so the
// kernels of each curve are compiled exactly once, in that curve's own translation unit.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/blitzar_b200.h"
#include "runtime.cuh"

namespace b200 {

struct MsmOptions {
  u32 window_bits = 0;  // 0 = choose from n
  u32 chunk1 = 0;       // chunk length of the first accumulation level (0 = 32, or 64 for big passes)
  u32 chunkn = 8;       // chunk length of the cascade levels
  u32 reduce_g1 = 16;   // bucket-reduction group size, first level (power of two)
  u32 reduce_gn = 4;    // bucket-reduction group size, later levels (power of two)
  u64 quad_threshold = 32768;  // launches with at most this many logical threads run 4 lanes each
  u64 max_group_entries = 1ull << 30;  // columns are grouped below this many (term, window) entries
  u64 max_range_entries = 1ull << 31;  // one sort pass holds at most this many entries: longer
                                       // columns are processed as several generator ranges
  int pair_levels = -1;  // batch-affine pair levels (Weierstrass): -1 = from the mean bucket load
  u32 pair_batch = 0;    // pairs per thread of a pair level (0 = 32)
  int range_skew = 0;   // piece schedule of a multi-range call (range_begin); set by the host layer
  u32 uniform_add = 2;  // gathering level: runs start from the identity (no divergent start path);
                        // 0 off, 1 on, 2 = ed25519 only
  u32 gens_normalized = 0;  // set per call: the generator array has Z = 1 entries (fixed-base table,
                            // or caller generators normalised at ingestion)
  const u32* unit_veto = nullptr;  // set per call with gens_normalized: device flag, non-zero = the
                                   // ingestion met Z = 0 and left the generators unnormalised
  u32 normalize_gens = 1;  // ed25519 caller generators are normalised to Z = 1 at ingestion
  u32 lane_tail = 1;  // warp-cooperative (lane-sliced) Horner / encoding kernels for ed25519
  u32 scatter_window_major = 0;  // scatter with one thread per (window, term), window-major
  // bucket sort of the entries: 0 = atomic count + scan + scatter; 1 = binned sort (msm.cuh) for
  // unpadded passes of at least kBinnedSortMinEntries entries; 2 = binned whenever it applies
  u32 sort_path = 1;
  u32 table_policy = 0;  // fixed-base tables: 0 = cost model decides, 1 = whenever available, 2 = never
};

struct EngineCtx {
  stream_t s;
  MsmOptions opt;
  const void* builtin;  // device-resident built-in ristretto generators g(0..num_builtin)
  uint64_t num_builtin;
  stream_t tail = stream_t();  // optional second stream: cascade + merge of piece k under piece k+1
  // fixed-base table over the built-in generators (window w of generator i at builtin[w n + i]);
  // builtin_windows <= 1: plain generators only
  u32 builtin_window_bits = 0, builtin_windows = 0;
  // outputs of a fixed-base call over a handle with a partition table: 0 = cost model decides
  // (partition_route), 1 = every non-empty output from the table, 2 = never from the table
  u32 partition_policy = 0;
};

// sxt_multiexp_handle: generators of one curve resident in HBM, plus (when it pays and fits) the
// fixed-base table 2^(c w) G_i, w < windows, laid out window-major: entry w * n + i. Window 0 IS the
// generator array, so `gens` serves both the table mode and the variable-base fallback.
// Optionally (b200_multiexp_handle_add_partition_table) also the reference's partition table of width
// ptable_w over the same generators: 2^w subset sums per group of w generators, normalised device
// generators at entry g * 2^w + k (partition_msm.cuh), the last group padded with the identity.
struct Handle {
  unsigned curve_id;
  unsigned n;
  void* gens;  // device array of the curve's generator layout, windows * n entries
  unsigned window_bits = 0, windows = 1;
  void* ptable = nullptr;  // partition table, ptable_groups << ptable_w entries (null = none)
  unsigned ptable_w = 0;
  uint64_t ptable_groups = 0;
};

// Window width of a fixed-base table over n generators: minimises (digit additions + bucket
// reduction) for one 256-bit output, subject to the table fitting in `budget_bytes` and in the
// 31-bit generator index of a sorted entry. Returns 0 when no table should be built.
inline unsigned table_window_bits(uint64_t n, size_t gen_bytes, double budget_bytes) {
  if (n < 1024)  // tiny handles: the variable-base path with a small window wins anyway
    return 0;
  unsigned best = 0;
  double best_cost = 1e300;
  for (unsigned c = 10; c <= 20; ++c) {
    const double W = 256 / c + 1;
    if (W * (double)n * (double)gen_bytes > budget_bytes || W * (double)n >= 2147483648.0)
      continue;
    const double cost = W * (double)n + 2.5 * (double)(1u << (c - 1));
    if (cost < best_cost) {
      best_cost = cost;
      best = c;
    }
  }
  return best;
}

template <class T> struct DevBuf {
  T* p = nullptr;
  stream_t s;
  DevBuf(size_t count, stream_t s_) : s(s_) { p = (T*)dev_alloc(count * sizeof(T), s); }
  ~DevBuf() { dev_free(p, s); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
};

// generator-range r of `num_ranges` over n terms starts here (shared by the engine and the C-ABI
// layer, which schedules the host-to-device copies of each range)
// skew > 0: pieces shrink towards the end (upload-bound calls: little work is left after the last
// byte has arrived); skew < 0: pieces grow (compute-bound calls: the first kernels start early);
// 0: equal pieces. begin(0) = 0, begin(num_ranges) = n, strictly monotone for n >= num_ranges.
inline uint64_t range_begin(uint64_t n, uint32_t r, uint32_t num_ranges, int skew = 0) {
  if (r == 0)
    return 0;
  if (r >= num_ranges)
    return n;
  if (skew == 0 || n < 64ull * num_ranges)
    return n * r / num_ranges;
  const double t = (double)r / (double)num_ranges;
  const double f = skew > 0 ? 1.0 - (1.0 - t) * std::sqrt(1.0 - t) : t * std::sqrt(t);
  uint64_t b = (uint64_t)((double)n * f);
  const uint64_t lo = r, hi = n - (num_ranges - r);  // keep every piece non-empty
  return b < lo ? lo : (b > hi ? hi : b);
}
// called on the host before the engine touches terms [begin, end) (e.g. make the compute stream wait
// for that range's copies)
typedef void (*range_wait_fn)(void* user, uint64_t begin, uint64_t end);

// validates like cbindings/pedersen.cc:44-68 and returns the longest column
inline uint64_t check_descriptors(const sxt_sequence_descriptor* d, uint32_t num) {
  B200_REQUIRE(d != nullptr, "descriptors == nullptr");
  uint64_t longest = 0;
  for (uint32_t i = 0; i < num; ++i) {
    B200_REQUIRE(d[i].n == 0 || d[i].data != nullptr, "descriptor.n > 0 with data == nullptr");
    B200_REQUIRE(d[i].element_nbytes != 0 && d[i].element_nbytes <= 32,
                 "descriptor.element_nbytes must be in 1..32");
    if (d[i].is_signed)
      B200_REQUIRE(d[i].element_nbytes <= 16 &&
                       (d[i].element_nbytes & (d[i].element_nbytes - 1)) == 0,
                   "signed columns need a power-of-two element_nbytes <= 16");
    B200_REQUIRE(d[i].n < (1ull << 31), "column too long");
    longest = longest < d[i].n ? d[i].n : longest;
  }
  return longest;
}

// Bytes of one scalar row of a fixed-base call (mode 0 fixed width, 1 packed, 2 vlen): the outputs'
// scalars side by side, element_num_bytes bytes each in mode 0, else bit_table[j] bits each.
inline uint64_t fixed_row_bytes(int mode, unsigned element_num_bytes, const unsigned* bit_table,
                                unsigned num_outputs) {
  uint64_t row_bits = 0;
  if (mode == 0) {
    B200_REQUIRE(element_num_bytes >= 1 && element_num_bytes <= 32, "element_num_bytes in 1..32");
    row_bits = 8ull * element_num_bytes * num_outputs;
  } else {
    for (unsigned j = 0; j < num_outputs; ++j) {
      B200_REQUIRE(bit_table[j] > 0 && bit_table[j] <= 256, "output bit width must be in 1..256");
      row_bits += bit_table[j];
    }
  }
  return (row_bits + 7) / 8;
}

// Generator layout of a call whose column j pairs row i with generator offsets[j] + i (offsets null =
// all 0). The intervals [offsets[j], offsets[j] + n_j) of the non-empty columns, merged where they
// overlap or touch, are packed in increasing order into one array; column j's generator of row i
// sits at packed position base[j] + i. The engine (ingestion / generation per range) and the C-ABI
// layer (raw buffer size, upload pieces) both take the layout from here.
struct GenLayout {
  struct Piece {
    uint64_t src, pos, count;  // generators [src, src + count) of the source at packed [pos, pos + count)
  };
  std::vector<Piece> segments;  // the merged intervals
  std::vector<uint32_t> base;   // per column (0 for an empty column)
  uint64_t total = 0;           // packed size
  uint64_t max_n = 0;           // longest column

  GenLayout(const sxt_sequence_descriptor* d, uint32_t num, const uint64_t* offsets)
      : base(num, 0), n_(num, 0) {
    std::vector<uint32_t> order;
    for (uint32_t j = 0; j < num; ++j) {
      n_[j] = d[j].n;
      max_n = std::max<uint64_t>(max_n, d[j].n);
      if (d[j].n) {
        B200_REQUIRE(offset(offsets, j) <= ~0ull - d[j].n, "generator offset + column length overflows");
        order.push_back(j);
      }
    }
    std::stable_sort(order.begin(), order.end(), [offsets](uint32_t a, uint32_t b) {
      return offset(offsets, a) < offset(offsets, b);
    });
    for (uint32_t j : order) {
      const uint64_t lo = offset(offsets, j), hi = lo + n_[j];
      if (segments.empty() || lo > segments.back().src + segments.back().count) {
        const uint64_t pos = segments.empty() ? 0 : segments.back().pos + segments.back().count;
        segments.push_back({lo, pos, 0});
      }
      Piece& s = segments.back();
      s.count = std::max(s.count, hi - s.src);
      B200_REQUIRE(s.pos + s.count < (1ull << 31),
                   "merged generator intervals of 2^31 or more generators");
      base[j] = (uint32_t)(s.pos + (lo - s.src));
    }
    total = segments.empty() ? 0 : segments.back().pos + segments.back().count;
  }
  // every interval ends at or below `limit`
  bool within(uint64_t limit) const {
    return segments.empty() || segments.back().src + segments.back().count <= limit;
  }
  // the generators rows [b, e) of the columns use: U_j [base_j + b, base_j + min(e, n_j)), merged
  // within each segment, in increasing packed order
  std::vector<Piece> needed(uint64_t b, uint64_t e) const {
    std::vector<std::pair<uint64_t, uint64_t>> iv;  // packed [lo, hi)
    for (size_t j = 0; j < base.size(); ++j)
      if (n_[j] > b)
        iv.push_back({base[j] + b, base[j] + std::min(e, n_[j])});
    std::sort(iv.begin(), iv.end());
    std::vector<Piece> out;
    size_t k = 0;  // segment of the current interval (intervals never cross a segment)
    for (auto& v : iv) {
      while (segments[k].pos + segments[k].count <= v.first)
        ++k;
      const Piece& s = segments[k];
      if (!out.empty() && out.back().pos + out.back().count >= v.first && out.back().pos >= s.pos) {
        out.back().count = std::max(out.back().count, v.second - out.back().pos);
        continue;
      }
      out.push_back({s.src + (v.first - s.pos), v.first, v.second - v.first});
    }
    return out;
  }

private:
  std::vector<uint64_t> n_;
  static uint64_t offset(const uint64_t* offsets, uint32_t j) { return offsets ? offsets[j] : 0; }
};

struct CurveVTable {
  unsigned curve_id, point_bytes, gen_bytes, abi_gen_bytes, abi_proj_bytes, abi_commit_bytes;
  void (*commit_device)(const EngineCtx&, void* out_commitments, void* out_partials, uint32_t num,
                        const sxt_sequence_descriptor* d, const void* generators_dev,
                        uint64_t offset_generators, uint32_t num_ranges, range_wait_fn wait,
                        void* wait_user);
  // as commit_device with generator offsets[j] + i for row i of column j (offsets: host array, null
  // = all 0). generators_dev is indexed by offsets[j] + i, or, with `packed`, already holds
  // GenLayout's packed array (host calls upload only the generators the columns use)
  void (*commit_device_offsets)(const EngineCtx&, void* out_commitments, void* out_partials,
                                uint32_t num, const sxt_sequence_descriptor* d,
                                const void* generators_dev, const uint64_t* offsets, bool packed,
                                uint32_t num_ranges, range_wait_fn wait, void* wait_user);
  void (*fixed_device)(const EngineCtx&, void* out_res, void* out_partials, const Handle* h,
                       int mode, unsigned element_num_bytes, const unsigned* bit_table,
                       const unsigned* lengths, unsigned num_outputs, unsigned n,
                       const uint8_t* scalars_dev);
  void (*ingest_projective)(const EngineCtx&, const void* raw_dev, void* gens, uint64_t n);
  void (*gens_to_projective)(const EngineCtx&, const void* gens, void* out_dev, uint64_t n);
  void (*store)(const EngineCtx&, const void* pts, void* out_dev, uint64_t count, bool commit);
  void (*sum_parts)(const EngineCtx&, const void* parts, uint32_t nparts, uint32_t count,
                    void* out_pts);
  // synthetic generators (synth.cuh) in the ABI layout: projective structs or commit-stride affine
  void (*synth_generators)(const EngineCtx&, void* out_dev, uint64_t n, uint64_t first,
                           bool projective);
  unsigned abi_compact_bytes;
  // generators out of a reference partition-table image (device copy of the file's table)
  void (*ingest_compact_table)(const EngineCtx&, const void* table_dev, unsigned window_width,
                               void* gens, uint64_t n);
  // fills windows 1 .. windows-1 of a fixed-base table whose window 0 (n generators) is in place
  void (*build_table)(const EngineCtx&, void* table, uint64_t n, unsigned window_bits,
                      unsigned windows);
  // groups [first_group, first_group + groups) of the reference's partition table of width w over n
  // generators (device generator layout; ptable.cuh) -> compact ABI entries at out_dev
  void (*partition_table)(const EngineCtx&, const void* gens, uint64_t n, unsigned w,
                          uint64_t first_group, uint64_t groups, void* out_dev);
  // the same groups as normalised device generators (C::Gen), the layout of Handle::ptable
  void (*partition_gens)(const EngineCtx&, const void* gens, uint64_t n, unsigned w,
                         uint64_t first_group, uint64_t groups, void* out_gens);
};
extern const CurveVTable kVTableEd25519, kVTableBls12381, kVTableBn254, kVTableGrumpkin;

inline const CurveVTable& curve_vtable(unsigned curve_id) {
  switch (curve_id) {
  case SXT_CURVE_RISTRETTO255:
    return kVTableEd25519;
  case SXT_CURVE_BLS_381:
    return kVTableBls12381;
  case SXT_CURVE_BN_254:
    return kVTableBn254;
  case SXT_CURVE_GRUMPKIN:
    return kVTableGrumpkin;
  default:
    die("unsupported curve id", __FILE__, __LINE__);
  }
}

// inner-product argument over ristretto255 (ipa.cuh); same contracts as the two sxt_* entry points
// (ipa_verify runs a batch of one) and as the two b200_* batch entry points (IpaBatch)
void ipa_prove(const EngineCtx& ctx, uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
               uint8_t* transcript203, uint64_t n, uint64_t generators_offset,
               const uint8_t* a_vector, const uint8_t* b_vector);
int ipa_verify(const EngineCtx& ctx, uint8_t* transcript203, uint64_t n,
               uint64_t generators_offset, const uint8_t* b_vector, const uint8_t* product,
               const uint8_t* a_commit160, const uint8_t* l_vector, const uint8_t* r_vector,
               const uint8_t* ap_value);
void ipa_prove_batch(const EngineCtx& ctx, uint32_t num_proofs, uint8_t* l_vectors,
                     uint8_t* r_vectors, uint8_t* ap_values, uint8_t* transcripts,
                     const uint64_t* n, const uint64_t* generators_offsets,
                     const uint8_t* a_vectors, const uint8_t* b_vectors);
uint32_t ipa_verify_batch(const EngineCtx& ctx, uint32_t num_proofs, int* results,
                          uint8_t* transcripts, const uint64_t* n,
                          const uint64_t* generators_offsets, const uint8_t* b_vectors,
                          const uint8_t* products, const uint8_t* a_commits,
                          const uint8_t* l_vectors, const uint8_t* r_vectors,
                          const uint8_t* ap_values);

// lane-sliced field arithmetic self-test (lanefield.cuh): number of mismatching checks over
// `warps` warps of pseudo-random / edge-case operands
unsigned selftest_lane_arithmetic(const EngineCtx& ctx, unsigned warps, unsigned seed);
// atomic against binned bucket sort of the same device columns (msm.cuh sort_selftest)
unsigned selftest_sort(const EngineCtx& ctx, const sxt_sequence_descriptor* d, unsigned num,
                       unsigned window_bits);

// element-wise field arithmetic (field_op.cuh, b200_field_op): `op` on n elements of host arrays,
// synchronises; ~0u when the field does not offer the operation. Each curve unit runs its own base
// field (field id = curve id); the ed25519 unit also the scalars mod l (4) and the lane-sliced
// F25519 (5, device only).
unsigned field_op_ed25519(const EngineCtx& ctx, unsigned field, unsigned op, uint64_t n,
                          const uint32_t* a, const uint32_t* b, uint32_t* out);
unsigned field_op_bls12381(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                           const uint32_t* b, uint32_t* out);
unsigned field_op_bn254(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                        const uint32_t* b, uint32_t* out);
unsigned field_op_grumpkin(const EngineCtx& ctx, unsigned op, uint64_t n, const uint32_t* a,
                           const uint32_t* b, uint32_t* out);
inline unsigned field_op(const EngineCtx& ctx, unsigned field, unsigned op, uint64_t n,
                         const uint32_t* a, const uint32_t* b, uint32_t* out) {
  switch (field) {
  case 1: return field_op_bls12381(ctx, op, n, a, b, out);
  case 2: return field_op_bn254(ctx, op, n, a, b, out);
  case 3: return field_op_grumpkin(ctx, op, n, a, b, out);
  default: return field_op_ed25519(ctx, field, op, n, a, b, out);
  }
}

// built-in ristretto generators g(first .. first+n) into the device generator layout
void launch_builtin_generators(const EngineCtx& ctx, void* gens, uint64_t first, uint64_t n);

}  // namespace b200
