// Device-level glue between the C ABI and the MSM engine: descriptor validation, column grouping,
// generator ingestion, the choice between a handle's fixed-base table and the variable-base run
// (prefer_table), result canonicalisation. Shared by api.cu (product) and the CPU-side emulation
// harness under tests/emul (test infrastructure), both through the per-curve vtables.
#pragma once
#include <cstdint>
#include <vector>

#include "engine_api.cuh"
#include "msm.cuh"
#include "partition_msm.cuh"
#include "ptable.cuh"
#include "synth.cuh"

namespace b200 {

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

// All kernel launches of one curve live behind CurveOps<C>, so each curve is instantiated in its
// own translation unit (curve_*.cu) and api.cu only sees `extern template` declarations.
template <class C> struct CurveOps {
  typedef typename C::Gen Gen;
  typedef typename C::Point Point;

  // Columns are processed in groups so that (terms x windows) stays below 2^32 entries and the
  // sort scratch stays within a few GB of HBM.
  static void run_columns(const EngineCtx& ctx, const Gen* gens, std::vector<ColumnDesc>& cols,
                          Point* out, u32 num_ranges = 1, RangeHook* hook = nullptr) {
    const uint64_t kMaxEntries = ctx.opt.max_group_entries;
    size_t b = 0;
    while (b < cols.size()) {
      size_t e = b;
      uint64_t entries = 0;
      while (e < cols.size()) {
        uint64_t est = (uint64_t)cols[e].n * (cols[e].bit_width / 10 + 1);
        if (e > b && entries + est > kMaxEntries)
          break;
        entries += est;
        ++e;
      }
      std::vector<ColumnDesc> group(cols.begin() + b, cols.begin() + e);
      const bool whole = b == 0 && e == cols.size();
      // range hooks assume one pass over the generators; several column groups each see all of them
      if (!whole && hook && b == 0) {
        hook->before_range(0, ~0ull);
        hook->before_accumulate();
      }
      msm_run<C>(ctx.s, gens, group, out + b, ctx.opt, whole ? num_ranges : 1,
                 whole ? hook : nullptr, ctx.tail);
      b = e;
    }
  }

  // generator ingestion of one range: ABI layout (device) -> device generator layout
  struct IngestHook : RangeHook {
    const EngineCtx* ctx;
    const unsigned char* raw;  // ABI-layout generators on the device, or null
    Gen* gens;
    uint64_t n, offset_generators;
    bool builtin;  // generate g(offset + i) instead of converting `raw`
    range_wait_fn wait;
    void* wait_user;
    u32* invalid = nullptr;  // non-null: normalise the generators to Z = 1 (ingest_normalized)
    bool pending = false;  // an ingestion is running on the second stream
    void before_range(u64 begin, u64 end) override {
      if (end > n)
        end = n;
      if (begin >= end)
        return;
      if (wait)
        wait(wait_user, begin, end);
      if (raw) {
        // the sort of this range reads only scalars: the ingestion runs beside it on a second
        // stream and is joined right before the first kernel that gathers generators
        stream_t aux = aux_stream();
        stream_follow(aux, ctx->s);
        if constexpr (C::kCurveId == kRistretto255) {
          if (invalid) {
            ingest_normalized(aux, raw + begin * C::kAbiGenBytes, gens + begin, IngestMap{},
                              end - begin, invalid);
            pending = true;
            return;
          }
        }
        launch(IngestBody<C, false>{raw + begin * C::kAbiGenBytes, gens + begin}, end - begin, aux);
        pending = true;
      } else if (builtin) {
        launch_builtin(ctx->s, gens + begin, offset_generators + begin, end - begin);
      }
    }
    void before_accumulate() override {
      if (pending) {
        stream_follow(ctx->s, aux_stream());
        pending = false;
      }
    }
  };
  static void launch_builtin(stream_t s, Gen* gens, uint64_t first, uint64_t count) {
    if constexpr (C::kCurveId == kRistretto255)
      launch(BuiltinGeneratorBody{gens, first}, count, s);
    else
      die("generators == nullptr", __FILE__, __LINE__);
  }

  // generator ingestion / generation of one range with per-column generator starts: every piece of
  // GenLayout::needed in one launch
  struct PiecesHook : RangeHook {
    const EngineCtx* ctx;
    const GenLayout* layout;
    const unsigned char* raw;  // ABI-layout generators on the device, or null
    bool packed;               // raw is in the layout's packed order (else indexed by source index)
    bool generate;             // generate built-in generators instead of converting `raw`
    Gen* gens;                 // the packed device generators
    range_wait_fn wait;
    void* wait_user;
    u32* invalid = nullptr;  // non-null: normalise the generators to Z = 1 (ingest_normalized)
    bool pending = false;  // an ingestion is running on the second stream
    void before_range(u64 begin, u64 end) override {
      end = std::min<u64>(end, layout->max_n);
      if (begin >= end)
        return;
      if (wait)
        wait(wait_user, begin, end);
      if (!raw && !generate)
        return;
      const std::vector<GenLayout::Piece> pieces = layout->needed(begin, end);
      const size_t np = pieces.size();
      std::vector<u64> block(3 * np + 1, 0);  // [start x (np + 1)][from x np][to x np]
      for (size_t k = 0; k < np; ++k) {
        block[k + 1] = block[k] + pieces[k].count;
        block[np + 1 + k] = raw && packed ? pieces[k].pos : pieces[k].src;
        block[2 * np + 1 + k] = pieces[k].pos;
      }
      // as in IngestHook: the ingestion runs under the range's sort on a second stream
      const stream_t on = raw ? aux_stream() : ctx->s;
      if (raw)
        stream_follow(on, ctx->s);
      const u64* staged = (const u64*)stage_to_device(on, block.data(), block.size() * sizeof(u64));
      const GenPieces p{staged, staged + np + 1, staged + 2 * np + 1, (u32)np};
      bool normalized = false;
      if constexpr (C::kCurveId == kRistretto255) {
        if (raw && invalid) {
          ingest_normalized(on, raw, gens, IngestMap{p}, block[np], invalid);
          normalized = true;
        }
      }
      if (raw) {
        if (!normalized)
          launch(IngestPiecesBody<C>{raw, gens, p}, block[np], on);
        pending = true;
      } else if constexpr (C::kCurveId == kRistretto255) {
        launch(BuiltinPiecesBody{gens, p}, block[np], on);
      }
      dev_free((void*)staged, on);
    }
    void before_accumulate() override {
      if (pending) {
        stream_follow(ctx->s, aux_stream());
        pending = false;
      }
    }
  };

  static std::vector<ColumnDesc> columns_of(const sxt_sequence_descriptor* d, uint32_t num) {
    std::vector<ColumnDesc> cols(num);
    for (uint32_t i = 0; i < num; ++i) {
      cols[i].base = d[i].data;
      cols[i].row_stride = d[i].element_nbytes;
      cols[i].bit_offset = 0;
      cols[i].bit_width = 8u * d[i].element_nbytes;
      cols[i].n = (u32)d[i].n;
      cols[i].is_signed = d[i].is_signed ? 1u : 0u;
      cols[i].first_window = cols[i].num_windows = 0;
      cols[i].table_n = 0;
    }
    return cols;
  }

  // the commitments (or partial points) of `cols` over `gens`; builtin_table: gens is the built-in
  // generator array, whose fixed-base table serves the call when it is the cheaper run
  static void commit_columns(const EngineCtx& ctx, void* out_commitments, void* out_partials,
                             std::vector<ColumnDesc>& cols, const Gen* gens, bool builtin_table,
                             uint32_t num_ranges, RangeHook* hook) {
    stream_t s = ctx.s;
    const uint32_t num = (uint32_t)cols.size();
    Point* pts = (Point*)out_partials;
    DevBuf<Point> tmp(out_partials ? 1 : num, s);
    if (!pts)
      pts = tmp.p;
    EngineCtx rctx = ctx;
    if (builtin_table && ctx.builtin_windows > 1)
      rctx.opt.gens_normalized = 1u;  // the built-in table's entries are normalised (Z = 1)
    // built-in generators covered by the precomputed fixed-base table (sxt_config::
    // num_precomputed_generators): shared-bucket table mode when it is the cheaper run
    if (builtin_table &&
        prefer_table(cols, ctx.builtin_window_bits, ctx.builtin_windows, ctx.opt)) {
      rctx.opt.window_bits = ctx.builtin_window_bits;
      for (auto& col : cols)
        col.table_n = (u32)ctx.num_builtin;
    }
    run_columns(rctx, gens, cols, pts, num_ranges ? num_ranges : 1, hook);
    hook->before_accumulate();  // (no-op unless a range was ingested without being accumulated)
    if (out_commitments)
      launch_store_commit<C>(s, pts, (unsigned char*)out_commitments, num, ctx.opt.lane_tail != 0);
  }

  // device-resident variable-base MSM; descriptors[i].data and generators_dev are device pointers.
  // The generator range is processed in num_ranges pieces; `wait` (optional) is called on the host
  // before each piece is touched.
  static void commit_device(const EngineCtx& ctx, void* out_commitments, void* out_partials,
                            uint32_t num, const sxt_sequence_descriptor* d,
                            const void* generators_dev, uint64_t offset_generators,
                            uint32_t num_ranges, range_wait_fn wait, void* wait_user) {
    stream_t s = ctx.s;
    uint64_t n = check_descriptors(d, num);
    DevBuf<Gen> gens(n ? n : 1, s);
    const Gen* gens_ptr = gens.p;
    IngestHook hook;
    hook.ctx = &ctx;
    hook.raw = (const unsigned char*)generators_dev;
    hook.gens = gens.p;
    hook.n = n;
    hook.offset_generators = offset_generators;
    hook.builtin = false;
    hook.wait = wait;
    hook.wait_user = wait_user;
    if (n && !generators_dev) {
      if (C::kCurveId != kRistretto255)
        die("generators == nullptr", __FILE__, __LINE__);
      if (offset_generators + n <= ctx.num_builtin)
        gens_ptr = (const Gen*)ctx.builtin + offset_generators;
      else
        hook.builtin = true;
    }
    std::vector<ColumnDesc> cols = columns_of(d, num);
    const Normalizing norm(ctx, n && generators_dev, &hook.invalid);
    commit_columns(norm.ctx, out_commitments, out_partials, cols, gens_ptr,
                   n && !generators_dev && !hook.builtin, num_ranges, &hook);
  }
  // Caller generators of ed25519 are normalised at ingestion (ingest_normalized) unless
  // opt.normalize_gens is 0. Only then is the call's Z = 0 flag allocated and zeroed (*hook_invalid),
  // and `ctx` runs the gathering level on Z = 1 generators unless that flag gets set.
  struct Normalizing {
    EngineCtx ctx;
    u32* flag = nullptr;
    Normalizing(const EngineCtx& c, bool ingests, u32** hook_invalid) : ctx(c) {
      if (C::kCurveId != kRistretto255 || !ingests || !c.opt.normalize_gens)
        return;
      flag = (u32*)dev_alloc(sizeof(u32), c.s);
      dev_zero(flag, sizeof(u32), c.s);
      *hook_invalid = flag;
      ctx.opt.gens_normalized = 1u;
      ctx.opt.unit_veto = flag;
    }
    ~Normalizing() { dev_free(flag, ctx.s); }
    Normalizing(const Normalizing&) = delete;
    Normalizing& operator=(const Normalizing&) = delete;
  };

  // commit_device with a generator start per column: row i of column j pairs with generator
  // offsets[j] + i (offsets null = all 0). The generators the columns use are laid out by GenLayout;
  // only built-in generators that all lie in the precomputed range are used in place.
  static void commit_device_offsets(const EngineCtx& ctx, void* out_commitments,
                                    void* out_partials, uint32_t num,
                                    const sxt_sequence_descriptor* d, const void* generators_dev,
                                    const uint64_t* offsets, bool packed, uint32_t num_ranges,
                                    range_wait_fn wait, void* wait_user) {
    check_descriptors(d, num);
    const GenLayout layout(d, num, offsets);
    if (layout.total && !generators_dev && C::kCurveId != kRistretto255)
      die("generators == nullptr", __FILE__, __LINE__);
    const bool builtin_table = layout.total && !generators_dev && layout.within(ctx.num_builtin);
    DevBuf<Gen> gens(builtin_table ? 1 : layout.total, ctx.s);
    PiecesHook hook;
    hook.ctx = &ctx;
    hook.layout = &layout;
    hook.raw = (const unsigned char*)generators_dev;
    hook.packed = packed;
    hook.generate = layout.total && !generators_dev && !builtin_table;
    hook.gens = gens.p;
    hook.wait = wait;
    hook.wait_user = wait_user;
    std::vector<ColumnDesc> cols = columns_of(d, num);
    for (uint32_t j = 0; j < num; ++j)  // built-in array: generator g sits at position g
      cols[j].gen_base = builtin_table && d[j].n && offsets ? (u32)offsets[j] : layout.base[j];
    const Normalizing norm(ctx, layout.total && generators_dev, &hook.invalid);
    commit_columns(norm.ctx, out_commitments, out_partials, cols,
                   builtin_table ? (const Gen*)ctx.builtin : gens.p, builtin_table, num_ranges,
                   &hook);
  }

  // fixed-base MSM over a handle's device-resident generators (mode 0 fixed width, 1 packed, 2 vlen)
  static void fixed_device(const EngineCtx& ctx, void* out_res, void* out_partials, const Handle* h,
                           int mode, unsigned element_num_bytes, const unsigned* bit_table,
                           const unsigned* lengths, unsigned num_outputs, unsigned n,
                           const uint8_t* scalars_dev) {
    stream_t s = ctx.s;
    std::vector<ColumnDesc> cols(num_outputs);
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
    const uint64_t row_stride = (row_bits + 7) / 8;
    uint64_t bit_off = 0;
    for (unsigned j = 0; j < num_outputs; ++j) {
      unsigned width = mode == 0 ? 8u * element_num_bytes : bit_table[j];
      unsigned len = mode == 2 ? lengths[j] : n;
      B200_REQUIRE(len <= h->n, "more scalars than generators in the handle");
      cols[j].base = scalars_dev;
      cols[j].row_stride = row_stride;
      cols[j].bit_offset = (u32)bit_off;
      cols[j].bit_width = width;
      cols[j].n = len;
      cols[j].is_signed = 0;
      cols[j].first_window = cols[j].num_windows = 0;
      cols[j].table_n = 0;
      bit_off += width;
    }
    Point* pts = (Point*)out_partials;
    DevBuf<Point> tmp(out_partials ? 1 : (num_outputs ? num_outputs : 1), s);
    if (!pts)
      pts = tmp.p;
    // outputs answered from the handle's partition table run as n = 0 columns of the engine
    const std::vector<u32> routed = partition_route(ctx, h, cols);
    std::vector<ColumnDesc> routed_cols;
    if (!routed.empty()) {
      routed_cols = cols;
      for (u32 j : routed)
        cols[j].n = 0;
    }
    EngineCtx tctx = ctx;
    tctx.opt.gens_normalized = h->windows > 1 ? 1u : 0u;  // build_table normalised every entry
    if (prefer_table(cols, h->window_bits, h->windows, ctx.opt)) {
      tctx.opt.window_bits = h->window_bits;
      for (auto& col : cols)
        col.table_n = h->n;
    }
    run_columns(tctx, (const Gen*)h->gens, cols, pts);
    partition_msm<C>(s, (const Gen*)h->ptable, h->ptable_w, routed_cols, routed, pts);
    if (out_res)
      launch(StoreBody<C, false>{pts, (unsigned char*)out_res}, num_outputs, s);
  }

  // projective ABI structs (device) -> device generator layout
  static void ingest_projective(const EngineCtx& ctx, const void* raw_dev, void* gens, uint64_t n) {
    launch(IngestBody<C, true>{(const unsigned char*)raw_dev, (Gen*)gens}, n, ctx.s);
  }
  static void gens_to_projective(const EngineCtx& ctx, const void* gens, void* out_dev,
                                 uint64_t n) {
    launch(GenToProjBody<C>{(const Gen*)gens, (unsigned char*)out_dev}, n, ctx.s);
  }
  // canonical commitments (commit = true) or projective ABI structs from accumulator points
  static void store(const EngineCtx& ctx, const void* pts, void* out_dev, uint64_t count,
                    bool commit) {
    if (commit)
      launch_store_commit<C>(ctx.s, (const Point*)pts, (unsigned char*)out_dev, count,
                             ctx.opt.lane_tail != 0);
    else
      launch(StoreBody<C, false>{(const Point*)pts, (unsigned char*)out_dev}, count, ctx.s);
  }
  static void sum_parts(const EngineCtx& ctx, const void* parts, uint32_t nparts, uint32_t count,
                        void* out_pts) {
    launch(SumPartsBody<C>{(const Point*)parts, nparts, count, (Point*)out_pts}, count, ctx.s);
  }
  static void ingest_compact_table(const EngineCtx& ctx, const void* table_dev,
                                   unsigned window_width, void* gens, uint64_t n) {
    launch(IngestCompactBody<C>{(const unsigned char*)table_dev, window_width, (Gen*)gens}, n,
           ctx.s);
  }
  static void build_table(const EngineCtx& ctx, void* table, uint64_t n, unsigned window_bits,
                          unsigned windows) {
    B200_REQUIRE(windows <= (unsigned)kMaxTableWindows, "too many table windows");
    if (windows > 1)
      launch(PrecomputeTableBody<C>{(Gen*)table, n, window_bits, windows}, n, ctx.s);
  }
  // Table mode pays when the shared-bucket run (digit additions + ONE bucket reduction per column)
  // is cheaper than the variable-base run at the window width that run would choose; many short
  // columns (bucket_method2-style shapes) stay on the variable-base path.
  static bool prefer_table(const std::vector<ColumnDesc>& cols, unsigned table_c,
                           unsigned table_windows, const MsmOptions& opt) {
    if (table_windows <= 1 || table_c == 0)
      return false;
    u64 max_n = 0;
    u32 max_width = 1, ncols = 0;
    for (auto& col : cols)
      if (col.n) {
        max_n = std::max<u64>(max_n, col.n);
        max_width = std::max(max_width, col.bit_width);
        ++ncols;
      }
    if (ncols == 0 || max_width / table_c + 1 > table_windows || opt.table_policy == 2)
      return false;
    if (opt.table_policy == 1)
      return true;
    const double nb_t = (double)(1u << (table_c - 1));
    if ((double)ncols * nb_t * (double)sizeof(Point) > 3.0e9)
      return false;
    const u32 cv = opt.window_bits ? opt.window_bits
                                   : choose_window_bits(max_n, max_width, ncols, sizeof(Point));
    const double nb_v = (double)(1u << (cv - 1));
    double cost_t = 0, cost_v = 0;
    for (auto& col : cols)
      if (col.n) {
        cost_t += (double)col.n * (col.bit_width / table_c + 1) + 2.5 * nb_t;
        cost_v += (double)(col.bit_width / cv + 1) * ((double)col.n + 2.5 * nb_v);
      }
    return cost_t < cost_v;
  }
  // Outputs of a fixed-base call that the handle's partition table answers (DESIGN §4.4). Policy 0
  // compares, per output of width b and length len, the table path's b ceil(len / w) lookups and b
  // doublings with the engine's estimate as prefer_table makes it (table mode when the call would
  // take it, else the variable-base run at the window width it would choose).
  static std::vector<u32> partition_route(const EngineCtx& ctx, const Handle* h,
                                          const std::vector<ColumnDesc>& cols) {
    std::vector<u32> routed;
    if (!h->ptable || ctx.partition_policy == 2)
      return routed;
    // cost of one table lookup / one bit of the Horner pass, in engine bucket-entry additions, fitted
    // to the H100 timings of tests/partition_msm_timing.py (RESULTS §8): a lookup costs about what a
    // bucket entry does, while the Horner pass is serial (b doublings and additions on one thread),
    // so its latency weighs like 300 entries per bit
    const double kLookup = 1.0, kDouble = 300.0;
    const bool table_mode = prefer_table(cols, h->window_bits, h->windows, ctx.opt);
    u64 max_n = 0;
    u32 max_width = 1, ncols = 0;
    for (auto& col : cols)
      if (col.n) {
        max_n = std::max<u64>(max_n, col.n);
        max_width = std::max(max_width, col.bit_width);
        ++ncols;
      }
    if (ncols == 0)
      return routed;
    const u32 cv = ctx.opt.window_bits ? ctx.opt.window_bits
                                       : choose_window_bits(max_n, max_width, ncols, sizeof(Point));
    const double nb_v = (double)(1u << (cv - 1)), w = h->ptable_w;
    for (u32 j = 0; j < (u32)cols.size(); ++j) {
      const ColumnDesc& col = cols[j];
      if (col.n == 0)
        continue;
      const double n = col.n, b = col.bit_width;
      const double engine =
          table_mode ? n * (double)(col.bit_width / h->window_bits + 1) +
                           2.5 * (double)(1u << (h->window_bits - 1))
                     : (double)(col.bit_width / cv + 1) * (n + 2.5 * nb_v);
      const double table = kLookup * b * std::ceil(n / w) + kDouble * b;
      if (ctx.partition_policy == 1 || table < engine)
        routed.push_back(j);
    }
    return routed;
  }
  static void synth_generators(const EngineCtx& ctx, void* out_dev, uint64_t n, uint64_t first,
                               bool projective) {
    Synth<C>::generators(ctx.s, out_dev, n, first, projective);
  }
  static void partition_table(const EngineCtx& ctx, const void* gens, uint64_t n, unsigned w,
                              uint64_t first_group, uint64_t groups, void* out_dev) {
    build_partition_table<C>(ctx.s, (const Gen*)gens, n, w, first_group, groups,
                             (unsigned char*)out_dev);
  }
  static void partition_gens(const EngineCtx& ctx, const void* gens, uint64_t n, unsigned w,
                             uint64_t first_group, uint64_t groups, void* out_gens) {
    build_partition_table<C>(ctx.s, (const Gen*)gens, n, w, first_group, groups, (Gen*)out_gens);
  }
};

#define B200_DEFINE_CURVE_VTABLE(NAME, C)                                                          \
  const CurveVTable NAME = {C::kCurveId,                                                           \
                            (unsigned)sizeof(typename C::Point),                                   \
                            (unsigned)sizeof(typename C::Gen),                                     \
                            (unsigned)C::kAbiGenBytes,                                             \
                            (unsigned)C::kAbiProjBytes,                                            \
                            (unsigned)C::kAbiCommitBytes,                                          \
                            &CurveOps<C>::commit_device,                                           \
                            &CurveOps<C>::commit_device_offsets,                                   \
                            &CurveOps<C>::fixed_device,                                            \
                            &CurveOps<C>::ingest_projective,                                       \
                            &CurveOps<C>::gens_to_projective,                                      \
                            &CurveOps<C>::store,                                                   \
                            &CurveOps<C>::sum_parts,                                               \
                            &CurveOps<C>::synth_generators,                                        \
                            (unsigned)C::kAbiCompactBytes,                                         \
                            &CurveOps<C>::ingest_compact_table,                                    \
                            &CurveOps<C>::build_table,                                             \
                            &CurveOps<C>::partition_table,                                         \
                            &CurveOps<C>::partition_gens}

}  // namespace b200
