// Pippenger MSM engine: signed-window digit decomposition, counting sort by bucket, chunked
// segmented bucket accumulation, hierarchical bucket reduction and window combination.
//
// Replaces wholesale (SURVEY §8 a5-a8): mtxcrv::async_compute_multiexponentiation
// (sxt/multiexp/curve/multiexponentiation.h:147-200), the bucket method
// (sxt/multiexp/bucket_method/{accumulation,multiexponentiation}.h, kernels accumulation_kernel.h:38-75,
// combination_kernel.h:40-106, fold_kernel.h:38-66, host tail combination.h:28-62), bucket_method2 and
// the per-bit general path (sxt/multiexp/pippenger/multiproduct_decomposition_kernel.cc,
// multiproduct_gpu/kernel.h). One algorithm covers every input shape the ABI admits:
// 1..32-byte unsigned, power-of-two signed, ragged lengths, bit-packed and strided scalar tables.
//
// Design (GPU-first, not the reference's): the reference gives one thread a 1/192 slice of the
// terms and read-modify-writes 255 global-memory buckets per window with c = 8; here every term is
// decomposed into signed c-bit digits (c up to 16, chosen from n), the (window,bucket) keys are
// counting-sorted so each bucket is a contiguous run of generator indices, and the runs are
// summed by a load-balanced chunk walk (every thread sums exactly K consecutive sorted entries,
// whatever the bucket-size distribution) followed by a short cascade over chunk-boundary pieces.
// Bucket arrays live in HBM once per window (no per-block replicas), capped at kMaxBucketBytes.
//
// Round 2: the short Weierstrass curves run the first levels of the bucket sums as batch-affine pair
// additions (batch_affine.cuh) before the chunk walk; fixed-base calls run in table mode (all windows of
// a column share one bucket set over a precomputed table 2^(c w) G_i, PrecomputeTableBody /
// ColumnDesc::table_n — replaces sxt/multiexp/pippenger2/{partition_table,partition_product,
// combine_reduce}.h); the ed25519 tail kernels are warp-cooperative (lanefield.cuh).
#pragma once
#include <algorithm>
#include <vector>

#include "batch_affine.cuh"
#include "curve.cuh"
#include "engine_api.cuh"
#include "lanefield.cuh"

namespace b200 {

// How to read term i of one output column: `bit_width` bits starting `bit_offset` bits into row i.
//   commitments API : base = column data, row_stride = element_nbytes, offset 0, width 8*nbytes
//   fixed MSM       : base = table, row_stride = num_outputs*nbytes, offset = 8*j*nbytes
//   packed / vlen   : base = table, row_stride = ceil(sum bits / 8), offset = prefix bits, n = length
struct ColumnDesc {
  const unsigned char* base;
  u64 row_stride;
  u32 bit_offset;
  u32 bit_width;
  u32 n;
  u32 is_signed;
  u32 first_window;
  u32 num_windows;  // digit windows of the column
  // Fixed-base table mode (generators come from a precomputed table of 2^(c w) G_i, w-major with
  // stride table_n): the digit of window w addresses generator w * table_n + i and ALL windows of the
  // column share ONE bucket set (first_window), so there is no Horner tail. 0 = one bucket set per
  // window (variable-base).
  u32 table_n;
  u32 reserved_;
};
B200_HD u32 bucket_windows(const ColumnDesc& col) { return col.table_n ? (col.num_windows ? 1u : 0u) : col.num_windows; }

B200_HD void load_scalar_bits(u32 v[8], bool& negative, const ColumnDesc& col, u64 i) {
  const unsigned char* row = col.base + i * col.row_stride;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    v[k] = 0;
  const u32 width = col.bit_width;
  const unsigned char* p = row + (col.bit_offset >> 3);
  const u32 sh = col.bit_offset & 7u;
  if (sh == 0 && width == 256 && (((size_t)p) & 15u) == 0) {
    const uint4* q = (const uint4*)p;
    uint4 a = q[0], b = q[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else if (sh == 0 && (width & 31u) == 0 && (((size_t)p) & 3u) == 0) {
    const u32* q = (const u32*)p;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if ((u32)k < (width >> 5))
        v[k] = q[k];
  } else {
    // generic: assemble from bytes
    const u32 nbytes = (sh + width + 7u) >> 3;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      u64 acc = 0;
#pragma unroll
      for (int b = 0; b < 5; ++b) {
        u32 idx = 4u * k + b;
        if (idx < nbytes)
          acc |= (u64)p[idx] << (8 * b);
      }
      v[k] = (u32)(acc >> sh);
    }
    // mask bits beyond width
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int lo = 32 * k;
      if ((int)width <= lo)
        v[k] = 0;
      else if ((int)width < lo + 32)
        v[k] &= (1u << (width - lo)) - 1u;
    }
  }
  negative = false;
  if (col.is_signed) {
    u32 top = width - 1;
    bool neg = false;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if ((top >> 5) == (u32)k)
        neg = (v[k] >> (top & 31u)) & 1u;
    if (neg) {
      // magnitude = 2^width - v : invert within width, add one
      u64 c = 1;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        int lo = 32 * k;
        u32 m = 0;
        if ((int)width >= lo + 32)
          m = 0xffffffffu;
        else if ((int)width > lo)
          m = (1u << (width - lo)) - 1u;
        c += (u64)((~v[k]) & m);
        v[k] = (u32)c & m;
        c = (m == 0xffffffffu) ? (c >> 32) : 0;
      }
      negative = true;
    }
  }
}

// Signed c-bit digit recoding; calls f(key, negate, window) for every non-zero digit.
// only_window != kAllWindows: only that window's digit is reported (the recoding still walks the
// windows below it for the carry).
constexpr u32 kAllWindows = 0xffffffffu;
template <class Fn>
B200_HD void for_each_digit(const u32 v[8], bool negative, const ColumnDesc& col, u32 c,
                            u32 nbuckets, Fn f, u32 only_window = kAllWindows) {
  const u32 half = nbuckets;  // 2^(c-1)
  const u32 mask = (1u << c) - 1u;
  u64 buf = 0;
  u32 nb = 0, w = 0, carry = 0;
  const u32 W = only_window == kAllWindows
                    ? col.num_windows
                    : (only_window < col.num_windows ? only_window + 1 : 0u);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    buf |= (u64)v[k] << nb;
    nb += 32;
    while (nb >= c && w < W) {
      u32 d = ((u32)buf & mask) + carry;
      buf >>= c;
      nb -= c;
      bool dneg = d > half;
      carry = dneg ? 1u : 0u;
      if (dneg)
        d = (1u << c) - d;
      if (d && (only_window == kAllWindows || w == only_window))
        f((col.first_window + (col.table_n ? 0u : w)) * nbuckets + (d - 1u), negative != dneg, w);
      ++w;
    }
  }
  while (w < W) {
    u32 d = ((u32)buf & mask) + carry;
    buf >>= c;
    bool dneg = d > half;
    carry = dneg ? 1u : 0u;
    if (dneg)
      d = (1u << c) - d;
    if (d && (only_window == kAllWindows || w == only_window))
      f((col.first_window + (col.table_n ? 0u : w)) * nbuckets + (d - 1u), negative != dneg, w);
    ++w;
  }
}

// ---- kernels (index-parallel bodies) -------------------------------------------------------------
// column of global term index tid: the last j with col_start[j] <= tid (binary search, so that
// many-output calls — hundreds of narrow columns — do not pay O(columns) loads per term)
B200_HD u32 column_of(const u64* col_start, u32 ncols, u64 tid) {
  u32 lo = 0, hi = ncols;
  while (hi - lo > 1) {
    const u32 mid = (lo + hi) >> 1;
    if (tid >= col_start[mid])
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}
struct CountBody {
  static constexpr int kBlock = 256;
  const ColumnDesc* cols;
  const u64* col_start;  // prefix of n over columns, ncols+1 entries
  u32 ncols, c, nbuckets;
  u32* counts;
  B200_HD void operator()(u64 tid) const {
    const u32 j = column_of(col_start, ncols, tid);
    const ColumnDesc col = cols[j];
    u64 i = tid - col_start[j];
    u32 v[8];
    bool neg;
    load_scalar_bits(v, neg, col, i);
    u32* cnt = counts;
    for_each_digit(v, neg, col, c, nbuckets, [cnt](u32 key, bool, u32) { B200_ATOMIC_ADD(&cnt[key], 1u); });
  }
};

struct ScatterBody {
  static constexpr int kBlock = 256;
  const ColumnDesc* cols;
  const u64* col_start;
  u32 ncols, c, nbuckets;
  u32* cursor;  // exclusive offsets, consumed
  u64* entries;  // (key << 32) | (generator index << 1) | negate
  // window-major order (total_terms != 0): thread = (window, term), all threads of one window run
  // together, so the 8-byte scatter writes of a launch wave land in ONE window's slice of the entry
  // array (n x 8 B) and merge in L2 before they reach HBM, instead of spreading over all windows
  u64 total_terms;
  B200_HD void operator()(u64 tid) const {
    u32 only = kAllWindows;
    if (total_terms) {
      only = (u32)(tid / total_terms);
      tid -= (u64)only * total_terms;
    }
    const u32 j = column_of(col_start, ncols, tid);
    const ColumnDesc col = cols[j];
    if (only != kAllWindows && only >= col.num_windows)
      return;
    u64 i = tid - col_start[j];
    u32 v[8];
    bool neg;
    load_scalar_bits(v, neg, col, i);
    u32* cur = cursor;
    u64* en = entries;
    const u32 ii = (u32)i, tn = col.table_n;
    for_each_digit(v, neg, col, c, nbuckets, [cur, en, ii, tn](u32 key, bool negate, u32 w) {
      u32 pos = B200_ATOMIC_ADD(&cur[key], 1u);
      en[pos] = ((u64)key << 32) | (u64)(((ii + w * tn) << 1) | (negate ? 1u : 0u));
    }, only);
  }
};

// exclusive prefix sum, three index-parallel passes per level. The first level uses short chunks
// (many threads, each walking 256 contiguous bytes); the partial sums above it are few, so they take
// long chunks to keep the recursion at two levels for the usual 2^19 keys.
constexpr u32 kScanChunk = 256, kScanChunkFirst = 64;
struct ScanUpBody {
  static constexpr int kBlock = 128;
  const u32* in;
  u64 n;
  u32* partial;
  u32 chunk;
  B200_HD void operator()(u64 t) const {
    u64 b = t * chunk, e = b + chunk < n ? b + chunk : n;
    u32 s = 0;
    for (u64 i = b; i < e; ++i)
      s += in[i];
    partial[t] = s;
  }
};
struct ScanTopBody {
  static constexpr int kBlock = 32;
  u32* data;
  u64 n;
  B200_HD void operator()(u64) const {
    u32 s = 0;
    for (u64 i = 0; i < n; ++i) {
      u32 v = data[i];
      data[i] = s;
      s += v;
    }
  }
};
struct ScanDownBody {
  static constexpr int kBlock = 128;
  u32* data;  // in: counts, out: exclusive offsets
  u64 n;
  const u32* partial_scanned;
  u32 chunk;
  B200_HD void operator()(u64 t) const {
    u64 b = t * chunk, e = b + chunk < n ? b + chunk : n;
    u32 s = partial_scanned[t];
    for (u64 i = b; i < e; ++i) {
      u32 v = data[i];
      data[i] = s;
      s += v;
    }
  }
};

// in-place exclusive scan of data[0..n); data[n] is included in the scan so that data[n] = total
// when the caller zeroes it beforehand.
inline void exclusive_scan(u32* data, u64 n, stream_t s, u32 chunk = kScanChunkFirst) {
  if (n <= kScanChunk) {
    launch(ScanTopBody{data, n}, 1, s);
    return;
  }
  u64 m = (n + chunk - 1) / chunk;
  u32* partial = (u32*)dev_alloc(m * sizeof(u32), s);
  launch(ScanUpBody{data, n, partial, chunk}, m, s);
  exclusive_scan(partial, m, s, kScanChunk);
  launch(ScanDownBody{data, n, partial, chunk}, m, s);
  dev_free(partial, s);
}

template <class C> struct FillIdentityBody {
  static constexpr int kBlock = 256;
  typename C::Point* p;
  B200_HD void operator()(u64 t) const { p[t] = C::identity(); }
};

// buckets[k] += scratch[k] for every bucket the current generator range touched (bucket_end = the
// range's cursor array after the scatter). A later range accumulates into its own scratch array and
// is merged here: one coalesced pass, instead of a read-add-write at every run boundary of the
// accumulation kernel (about twice as fast per piece at C2 in 4 pieces).
template <class C> struct MergeBucketsBody {
  static constexpr int kBlock = 128;
  const u32* bucket_end;
  const u32* bucket_begin;  // padded layouts: start offset of every bucket; null = dense layout
  const typename C::Point* scratch;
  typename C::Point* buckets;
  B200_HD void operator()(u64 k) const {
    const u32 lo = bucket_begin ? bucket_begin[k] : (k ? bucket_end[k - 1] : 0u);
    if (bucket_end[k] == lo)
      return;
    typename C::Point b = buckets[k];
    C::add(b, b, scratch[k]);
    buckets[k] = b;
  }
};

// Chunk walk. Thread t sums entries [t*K, (t+1)*K) of the sorted list. Segments (runs of one key)
// strictly inside the chunk are complete and go straight to buckets[key]; the first and last
// segment may continue in the neighbouring chunks, so they are emitted as pieces (2 per chunk,
// keys stay sorted) for the next, K/2-times smaller, level. The final level writes everything.
// kUniform (gathering level only): a run starts from the identity and its first generator is ADDED like
// every other one, so that a run boundary costs the lanes that hit it only a bucket store and a reset
// instead of a separate generator-to-point conversion path (one more multiplication by a constant) that
// the rest of the warp waits for; the price is a full addition for the first element of every run.
template <class C, bool kGather, class X = SeqExec, bool kUniform = false> struct AccumulateBody {
  static constexpr int kBlock = 128;
  // register cap: 168 (3 blocks/SM) for 8-limb fields; 12-limb bls12-381 keeps 255 (2 blocks/SM)
  static constexpr int kMinBlocks = !kGather ? 1 : (C::F::N > 8 ? 2 : 3);
  typedef typename C::Point Point;
  const u32* keys;                 // level >= 2
  const u64* entries;              // level 1: (key << 32) | (generator index << 1) | negate
  const typename C::Gen* gens;     // level 1
  const Point* pieces;             // level >= 2
  const u32* m_ptr;                // number of entries at this level (device)
  u32 K;
  u32 final_level;
  Point* buckets;
  u32* out_keys;
  Point* out_pieces;
  u32* out_m_ptr;
  u32 unit_z;  // level 1: every generator is normalised (fixed-base table) — 7M additions on ed25519

  // every bucket is written exactly once per generator range (a run strictly inside a chunk is
  // complete; split runs travel down the cascade and are written by the level that completes them)
  B200_HD void put_bucket(u32 key, const Point& acc, bool writer) const {
    if (writer)
      buckets[key] = acc;
  }
  B200_HD u32 key_at(u64 i) const { return kGather ? (u32)(entries[i] >> 32) : keys[i]; }
  B200_HD void fetch(Point& acc, u64 i, bool first) const {
    if (kGather) {
      u32 e = (u32)entries[i];
      if (first)
        C::gen_to_point(acc, gens[e >> 1], e & 1u);
      else
        C::template add_gen<X>(acc, acc, gens[e >> 1], e & 1u);
    } else {
      if (first)
        acc = pieces[i];
      else
        C::template add<X>(acc, acc, pieces[i]);
    }
  }
  B200_HD void operator()(u64 tid) const {
    const u64 t = tid / X::kLanes;
    const bool writer = (tid % X::kLanes) == 0;
    const u64 M = *m_ptr;
    const u64 T = (M + K - 1) / K;
    if (tid == 0 && out_m_ptr)
      *out_m_ptr = final_level ? 0u : (u32)(2 * T);
    u64 b = t * K;
    if (b >= M)
      return;
    u64 e = b + K < M ? b + K : M;
    u32 cur;
    Point acc;
    bool first_seg = true;
    if (kGather) {
      // software-pipelined gather: the generator of entry i+1 is loaded into registers before the
      // addition of entry i starts, so the random 128-byte read overlaps ~1300 instructions of
      // field arithmetic instead of stalling the warp on the long scoreboard
      u64 ent = entries[b];
      typename C::Gen g = gens[(u32)ent >> 1];
      cur = (u32)(ent >> 32);
      struct {
        Point p;
        bool unit;
        B200_HD void start(const typename C::Gen& g, bool negate) { C::gen_to_point(p, g, negate); }
        B200_HD void add(const typename C::Gen& g, bool negate) {
          C::template add_gen<X>(p, p, g, negate, unit);
        }
        B200_HD void get(Point& out) const { out = p; }
      } ga;
      ga.unit = unit_z != 0;
      for (u64 i = b; i < e; ++i) {
        u64 ent_n = ent;
        typename C::Gen g_n = g;
        if (i + 1 < e) {
          ent_n = entries[i + 1];
          g_n = gens[(u32)ent_n >> 1];
        }
        const u32 k = (u32)(ent >> 32);
        const bool negate = ((u32)ent & 1u) != 0;
        if (kUniform) {
          if (i == b) {
            ga.p = C::identity();
          } else if (k != cur) {
            ga.get(acc);
            if (final_level || !first_seg) {
              put_bucket(cur, acc, writer);
            } else if (writer) {
              out_keys[2 * t] = cur;
              out_pieces[2 * t] = acc;
            }
            first_seg = false;
            cur = k;
            ga.p = C::identity();
          }
          ga.add(g, negate);
        } else if (i == b) {
          ga.start(g, negate);
        } else if (k == cur) {
          ga.add(g, negate);
        } else {
          ga.get(acc);
          if (final_level || !first_seg) {
            put_bucket(cur, acc, writer);
          } else if (writer) {
            out_keys[2 * t] = cur;
            out_pieces[2 * t] = acc;
          }
          first_seg = false;
          cur = k;
          ga.start(g, negate);
        }
        ent = ent_n;
        g = g_n;
      }
      ga.get(acc);
    } else {
      cur = key_at(b);
      fetch(acc, b, true);
      for (u64 i = b + 1; i < e; ++i) {
        u32 k = key_at(i);
        if (k == cur) {
          fetch(acc, i, false);
        } else {
          if (final_level || !first_seg) {
            put_bucket(cur, acc, writer);
          } else if (writer) {
            out_keys[2 * t] = cur;
            out_pieces[2 * t] = acc;
          }
          first_seg = false;
          cur = k;
          fetch(acc, i, true);
        }
      }
    }
    if (final_level) {
      put_bucket(cur, acc, writer);
      return;
    }
    if (!writer)
      return;
    if (first_seg) {  // single-segment chunk: pad the tail slot with the identity
      out_keys[2 * t] = cur;
      out_pieces[2 * t] = acc;
      out_keys[2 * t + 1] = cur;
      out_pieces[2 * t + 1] = C::identity();
    } else {
      out_keys[2 * t + 1] = cur;
      out_pieces[2 * t + 1] = acc;
    }
  }
};

// window_used[w] |= (some entry of this pass landed in window w); bucket_end = cursor array after
// the scatter (end offset of every bucket)
struct WindowUsedBody {
  static constexpr int kBlock = 64;
  const u32* bucket_end;
  u32 nbuckets;
  u32* window_used;
  B200_HD void operator()(u64 w) const {
    u32 lo = w ? bucket_end[w * nbuckets - 1] : 0u;
    u32 hi = bucket_end[(w + 1) * nbuckets - 1];
    if (hi != lo)
      window_used[w] = 1u;
  }
};

// same flag from the per-bucket counts (before they are padded / scanned): thread t looks at 256 buckets
struct WindowUsedFromCountsBody {
  static constexpr int kBlock = 128;
  const u32* counts;
  u64 nkeys;
  u32 nbuckets;
  u32* window_used;
  B200_HD void operator()(u64 t) const {
    const u64 b = t * 256, e = b + 256 < nkeys ? b + 256 : nkeys;
    for (u64 k = b; k < e; ++k)
      if (counts[k])
        window_used[k / nbuckets] = 1u;
  }
};

// Hierarchical bucket reduction. For one window, computes sum_i i*X[i] + sum_i Cin[i] over
// m entries by groups of g: Xout[k] = g * sum_r X[gk+r], Cout[k] = sum_r r*X[gk+r] + sum_r Cin[gk+r]
// (first level: weights r+1, no Cin, because bucket id = index + 1). Repeating until m == 1 leaves
// the window sum in Cout[0].
template <class C, class Ex = SeqExec> struct ReduceBody {
  static constexpr int kBlock = 64;
  typedef typename C::Point Point;
  const Point* X;
  const Point* Cin;  // null on the first level
  u32 m_in, g, log2g;
  Point* Xout;
  Point* Cout;
  const u32* window_used;  // per window: non-zero if any term was scattered into it
  u32 nbuckets;
  B200_HD void operator()(u64 tid) const {
    const u64 t = tid / Ex::kLanes;
    const bool writer = (tid % Ex::kLanes) == 0;
    const u32 m_out = m_in / g;
    const u32 w = (u32)(t / m_out), k = (u32)(t % m_out);
    // empty window: nothing was scattered into any of its buckets
    if (window_used[w] == 0) {
      if (writer) {
        Xout[t] = C::identity();
        Cout[t] = C::identity();
      }
      return;
    }
    const Point* x = X + (u64)w * m_in + (u64)k * g;
    Point run = x[g - 1];
    Point acc = Cin ? C::identity() : run;
    if (Cin) {
      // acc = sum_{r>=1} r*X_r
      acc = run;
      if (g == 1)
        acc = C::identity();
    }
    for (u32 r = g - 1; r-- > 0;) {
      C::template add<Ex>(run, run, x[r]);
      if (r > 0 || !Cin)
        C::template add<Ex>(acc, acc, run);
    }
    if (Cin) {
      const Point* cin = Cin + (u64)w * m_in + (u64)k * g;
      for (u32 r = 0; r < g; ++r)
        C::template add<Ex>(acc, acc, cin[r]);
    }
    for (u32 i = 0; i < log2g; ++i)
      C::template dbl<Ex>(run, run);
    if (writer) {
      Xout[t] = run;
      Cout[t] = acc;
    }
  }
};

// Horner over a column's windows: out = sum_w 2^(c*w) * S[w]
template <class C, class X = SeqExec> struct CombineBody {
  static constexpr int kBlock = 32;
  typedef typename C::Point Point;
  const Point* S;  // one per window (flattened)
  const ColumnDesc* cols;
  u32 c;
  Point* out;
  B200_HD void operator()(u64 tid) const {
    const u64 j = tid / X::kLanes;
    const bool writer = (tid % X::kLanes) == 0;
    const ColumnDesc col = cols[j];
    if (col.num_windows == 0 || col.n == 0) {
      if (writer)
        out[j] = C::identity();
      return;
    }
    const u32 nw = bucket_windows(col);  // table mode: one shared bucket set, no Horner
    Point acc = S[col.first_window + nw - 1];
    for (u32 w = nw - 1; w-- > 0;) {
      for (u32 i = 0; i < c; ++i)
        C::template dbl<X>(acc, acc);
      C::template add<X>(acc, acc, S[col.first_window + w]);
    }
    if (writer)
      out[j] = acc;
  }
};

#if defined(__CUDACC__) && !defined(B200_EMULATE)
#define B200_LANE_TAIL 1
// ---- warp-cooperative tail kernels for ed25519 (lanefield.cuh) -------------------------------------
// Horner over a column's windows, one WARP per column: the c doublings between two windows run on
// lane-sliced coordinates (one coordinate per 8-lane group, limbs across lanes), the window sum is
// added with the quad-lane schedule on the replicated point.
struct CombineLaneBody {
  static constexpr int kBlock = 32;
  typedef Ed25519 C;
  const C::Point* S;
  const ColumnDesc* cols;
  u32 c;
  C::Point* out;
  __device__ void operator()(u64 tid) const {
    const u64 j = tid >> 5;
    const ColumnDesc col = cols[j];
    if (col.num_windows == 0 || col.n == 0) {
      if ((tid & 31u) == 0)
        out[j] = C::identity();
      return;
    }
    const lane10::Lane L = lane10::lane_info();
    const u32 nw = bucket_windows(col);
    C::Point acc = S[col.first_window + nw - 1];
    for (u32 w = nw - 1; w-- > 0;) {
      u32 t;
      const u32 v = lane10::dbl_n(L, lane10::slice_point(L, acc), (int)c, t);
      lane10::gather_point(acc, v, t);
      C::add<QuadExecConv>(acc, acc, S[col.first_window + w]);
    }
    if ((tid & 31u) == 0)
      out[j] = acc;
  }
};
// ristretto255 encoding with the inverse-square-root chain on 10 lanes per output, 3 outputs per warp
struct LanePow {
  static __device__ __forceinline__ void pow22523(F25519::E& r, const F25519::E& a) {
    const lane10::Lane L = lane10::lane_info();
    const u32 g = L.base / 10u;
    lane10::gather(r, lane10::pow22523(L, lane10::slice(L, a)), g < 3 ? g : 0u);
  }
};
struct StoreLaneBody {
  static constexpr int kBlock = 32;
  const Ed25519::Point* pts;
  unsigned char* out;
  u64 count;
  __device__ void operator()(u64 tid) const {
    const u32 lane = (u32)tid & 31u, g = lane / 10u;
    const u64 i = (tid >> 5) * 3 + g;
    const bool live = g < 3 && i < count;  // surplus lanes compute along (warp-wide shuffles)
    unsigned char enc[32];
    Ed25519::encode<LanePow>(enc, pts[live ? i : count - 1]);
    if (live && lane == 10u * g) {
      uint4* d = (uint4*)(out + 32 * i);
      const uint4* e = (const uint4*)enc;
      d[0] = e[0];
      d[1] = e[1];
    }
  }
};
#endif

// canonical commitments of `count` accumulator points
template <class C>
inline void launch_store_commit(stream_t s, const typename C::Point* pts, unsigned char* out,
                                u64 count, bool lane_tail = true);

// generator ingestion (ABI layout -> device layout)
template <class C, bool kProjective> struct IngestBody {
  static constexpr int kBlock = 128;
  const unsigned char* raw;
  typename C::Gen* gens;
  B200_HD void operator()(u64 i) const {
    typename C::Gen g;
    if (kProjective)
      C::load_proj_abi(g, raw + i * C::kAbiProjBytes);
    else
      C::load_gen_abi(g, raw + i * C::kAbiGenBytes);
    gens[i] = g;
  }
};
// Fixed-base precomputation (replaces mtxpp2::compute_partition_table, sxt/multiexp/pippenger2/
// partition_table.h:36-98 — the reference tabulates all 2^w subset sums of w-generator groups; here
// the table holds 2^(c w) G_i for every window w, normalised to Z = 1, so that all windows of a
// fixed-base MSM share one bucket set and the Horner tail disappears). table[0 .. n) holds the
// generators on entry; thread i fills table[w n + i], w = 0 .. W-1 (window 0 = the generator itself,
// normalised too), with one inversion (Montgomery's trick over its W points).
constexpr int kMaxTableWindows = 33;  // c >= 8
template <class C> struct PrecomputeTableBody {
  static constexpr int kBlock = 64;
  typename C::Gen* table;
  u64 n;
  u32 c, W;
  B200_HD void operator()(u64 i) const {
    typedef typename C::F F;
    typename C::Point p, pts[kMaxTableWindows];
    typename F::E prefix[kMaxTableWindows], acc = F::one(), inv;
    C::gen_to_point(p, table[i], false);
    for (u32 w = 0; w < W; ++w) {  // window 0 (the generator itself) is normalised as well
      if (w)
        for (u32 k = 0; k < c; ++k)
          C::dbl(p, p);
      pts[w] = p;
      prefix[w] = acc;
      F::mul(acc, acc, C::denominator(p));
    }
    F::invert(inv, acc);
    for (u32 w = W; w-- > 0;) {
      typename F::E zi;
      F::mul(zi, inv, prefix[w]);
      F::mul(inv, inv, C::denominator(pts[w]));
      typename C::Gen g;
      C::normalized_gen(g, pts[w], zi);
      table[(u64)w * n + i] = g;
    }
  }
};
// generators out of a reference partition-table file: entry (1 << j) of group g is generator
// g * w + j (mtxpp2::in_memory_partition_table_accessor::copy_generators,
// sxt/multiexp/pippenger2/in_memory_partition_table_accessor.h:68-81)
template <class C> struct IngestCompactBody {
  static constexpr int kBlock = 128;
  const unsigned char* table;  // the file's table (device copy)
  u32 window_width;
  typename C::Gen* gens;
  B200_HD void operator()(u64 i) const {
    const u64 group = i / window_width, j = i % window_width;
    const u64 entry = (group << window_width) + (1ull << j);
    typename C::Gen g;
    C::load_compact_abi(g, table + entry * C::kAbiCompactBytes);
    gens[i] = g;
  }
};
struct BuiltinGeneratorBody {
  static constexpr int kBlock = 64;
  Ed25519::Gen* gens;
  u64 first;
  B200_HD void operator()(u64 i) const {
    Ed25519::Point g;
    Ed25519::builtin_generator(g, first + i);
    Ed25519::point_to_gen(gens[i], g);
  }
};
// result canonicalisation
template <class C, bool kCommit> struct StoreBody {
  static constexpr int kBlock = 32;
  const typename C::Point* pts;
  unsigned char* out;
  B200_HD void operator()(u64 i) const {
    if (kCommit)
      C::store_commit_abi(out + i * C::kAbiCommitBytes, pts[i]);
    else
      C::store_proj_abi(out + i * C::kAbiProjBytes, pts[i]);
  }
};
template <class C>
inline void launch_store_commit(stream_t s, const typename C::Point* pts, unsigned char* out,
                                u64 count, bool lane_tail) {
#ifdef B200_LANE_TAIL
  if constexpr (C::kCurveId == kRistretto255) {
    if (lane_tail && count && count <= 4096) {  // latency-bound: 10 lanes per output
      launch(StoreLaneBody{pts, out, count}, (count + 2) / 3 * 32, s);
      return;
    }
  }
#endif
  launch(StoreBody<C, true>{pts, out}, count, s);
}
template <class C> struct GenToProjBody {  // device generators back to the projective ABI layout
  static constexpr int kBlock = 64;
  const typename C::Gen* gens;
  unsigned char* out;
  B200_HD void operator()(u64 i) const {
    typename C::Point p;
    C::gen_to_point(p, gens[i], false);
    C::store_proj_abi(out + i * C::kAbiProjBytes, p);
  }
};
// out[j] = sum_r parts[r*count + j]  (multi-GPU partial combination, prefix sums, ...)
template <class C> struct SumPartsBody {
  static constexpr int kBlock = 32;
  const typename C::Point* parts;
  u32 nparts, count;
  typename C::Point* out;
  B200_HD void operator()(u64 j) const {
    typename C::Point acc = parts[j];
    for (u32 r = 1; r < nparts; ++r)
      C::add(acc, acc, parts[(u64)r * count + j]);
    out[j] = acc;
  }
};

// ---- host orchestration --------------------------------------------------------------------------
// c minimising (windows) x (terms + bucket-reduction work), with the bucket arrays of all columns
// capped at kMaxBucketBytes of HBM. Widths up to 20 are supported (b200_set_tuning) but the automatic
// choice stops at 16: at n = 2^24, c = 20 saves less accumulation than it adds bucket reduction.
inline u32 choose_window_bits(u64 max_n, u32 max_width, u32 ncols, size_t point_bytes) {
  const double kMaxBucketBytes = 3.0e9;
  u32 best = 2;
  double best_cost = 1e300;
  for (u32 c = 2; c <= 16; ++c) {
    double W = (double)(max_width / c + 1);
    if (c > 8 && W * (double)(1u << (c - 1)) * (double)ncols * (double)point_bytes > kMaxBucketBytes)
      break;
    double cost = W * ((double)max_n + 2.5 * (double)(1u << (c - 1)));
    if (cost < best_cost) {
      best_cost = cost;
      best = c;
    }
  }
  return best;
}

// Window / bucket geometry of one pass, fixed from the FULL columns so that generator-range chunks
// of the same pass share one bucket array.
struct MsmPlan {
  u32 c = 0, nbuckets = 0, ncols = 0, total_windows = 0;
  u64 nkeys = 0, max_n = 0, total_terms = 0, total_entries = 0;
  std::vector<ColumnDesc> cols;  // first_window / num_windows filled in
};

inline MsmPlan msm_make_plan(std::vector<ColumnDesc> cols, const MsmOptions& opt,
                             size_t point_bytes) {
  MsmPlan p;
  p.ncols = (u32)cols.size();
  u32 max_width = 1;
  for (auto& col : cols) {
    p.max_n = std::max<u64>(p.max_n, col.n);
    p.total_terms += col.n;
    if (col.n)
      max_width = std::max(max_width, col.bit_width);
  }
  p.c = opt.window_bits ? opt.window_bits
                        : choose_window_bits(p.max_n, max_width, p.ncols, point_bytes);
  p.nbuckets = 1u << (p.c - 1);
  u64 max_entries = 0;
  for (auto& col : cols) {
    col.first_window = p.total_windows;
    col.num_windows = col.n ? col.bit_width / p.c + 1 : 0;
    p.total_windows += bucket_windows(col);
    max_entries += (u64)col.n * col.num_windows;
    if (col.table_n)
      B200_REQUIRE((u64)col.table_n * col.num_windows < (1ull << 31), "generator table too large");
  }
  p.nkeys = (u64)p.total_windows * p.nbuckets;
  p.total_entries = max_entries;
  B200_REQUIRE(p.nkeys < (1ull << 32), "too many buckets for one pass");
  p.cols = std::move(cols);
  return p;
}

// Optional per-range hook: called before the terms [begin, end) are touched (the C-ABI layer uses
// it to wait for that range's host-to-device copies and to ingest its generators).
struct RangeHook {
  virtual void before_range(u64 begin, u64 end) = 0;
  // called right before the first kernel that reads the generators of the current range (the sort
  // does not): lets the hook run generator ingestion on a second stream under the sort
  virtual void before_accumulate() {}
  virtual ~RangeHook() {}
};

// Sort + accumulate the terms [begin, end) of every column into d_buckets (indexed by the plan's
// keys). gens[i] pairs with term i (absolute index). add_into: buckets already hold the sums of
// earlier ranges (this range then goes through a scratch bucket array + MergeBucketsBody). Enqueued on
// s; with tail != s the latency-bound part (cascade levels >= 2, merge) moves to `tail` right after
// the first level, so that it runs under the NEXT range's sort and first level (the caller joins
// `tail` back before the bucket reduction).
template <class C>
void msm_accumulate_range(stream_t s, const MsmPlan& plan, const typename C::Gen* gens, u64 begin,
                          u64 end, bool add_into, typename C::Point* d_buckets,
                          u32* d_window_used, const MsmOptions& opt, stream_t tail,
                          RangeHook* hook = nullptr) {
  typedef typename C::Point Point;
  const u32 ncols = plan.ncols;
  std::vector<ColumnDesc> cols(plan.cols);
  std::vector<u64> col_start(ncols + 1, 0);
  u64 max_entries = 0;
  for (u32 j = 0; j < ncols; ++j) {
    u64 lo = std::min<u64>(begin, cols[j].n), hi = std::min<u64>(end, cols[j].n);
    cols[j].base += lo * cols[j].row_stride;
    cols[j].n = (u32)(hi - lo);
    col_start[j + 1] = col_start[j] + cols[j].n;
    max_entries += (u64)cols[j].n * cols[j].num_windows;
  }
  const u64 total_terms = col_start[ncols];
  if (total_terms == 0)
    return;
  B200_REQUIRE(max_entries < (1ull << 32) && end - begin < (1ull << 31),
               "too many (term, window) entries for one sort pass");
  const u32 c = plan.c, nbuckets = plan.nbuckets;
  const u64 nkeys = plan.nkeys;
  gens += begin;  // entry indices are relative to the range

  // one staging block: [ColumnDesc x ncols][u64 x (ncols+1)], copied with a single H2D
  const size_t desc_bytes = ncols * sizeof(ColumnDesc), start_bytes = (ncols + 1) * sizeof(u64);
  std::vector<unsigned char> stage(desc_bytes + start_bytes);
  std::memcpy(stage.data(), cols.data(), desc_bytes);
  std::memcpy(stage.data() + desc_bytes, col_start.data(), start_bytes);
  unsigned char* d_stage = (unsigned char*)stage_to_device(s, stage.data(), stage.size());
  const ColumnDesc* d_cols = (const ColumnDesc*)d_stage;
  const u64* d_col_start = (const u64*)(d_stage + desc_bytes);

  StageRange nvtx_sort("msm: digit count + scan + scatter");
  u32* d_counts = (u32*)dev_alloc((nkeys + 1) * sizeof(u32), s);
  dev_zero(d_counts, (nkeys + 1) * sizeof(u32), s);
  launch(CountBody{d_cols, d_col_start, ncols, c, nbuckets, d_counts}, total_terms, s);
  // Batch-affine pair levels (short Weierstrass curves, large passes): L levels, buckets padded to
  // multiples of 2^L slots; L from the mean bucket load so that pads stay below ~1/4 of the slots.
  u32 L = 0;
  if constexpr (C::kBatchAffine) {
    const double mean = (double)max_entries / (double)nkeys;
    if (opt.pair_levels >= 0)
      L = (u32)opt.pair_levels;
    else if (max_entries >= (1ull << 23))  // below ~2^19 terms the per-level fixed costs lose (measured)
      while (L < 6 && (double)(32u << L) <= mean)  // 2 levels at a mean load of 64, 3 at 128
        ++L;                                        // (tests/pair_timing.py)
    while (L > 0 && max_entries + nkeys * ((1ull << L) - 1) >= (1ull << 32) - (1ull << L))
      --L;
  }
  const u64 slots_max =
      L ? ((max_entries + nkeys * ((1ull << L) - 1) + (1ull << L) - 1) >> L) << L : max_entries;
  u32* d_starts = nullptr;
  if (L) {
    launch(WindowUsedFromCountsBody{d_counts, nkeys, nbuckets, d_window_used}, (nkeys + 255) / 256, s);
    launch(PadCountsBody{d_counts, (1u << L) - 1u}, nkeys, s);
  }
  exclusive_scan(d_counts, nkeys + 1, s);  // d_counts[nkeys] = number of (padded) entries
  u32* d_m = (u32*)dev_alloc(16 * sizeof(u32), s);
  copy_d2d(d_m, d_counts + nkeys, sizeof(u32), s);
  if (L) {
    d_starts = (u32*)dev_alloc((nkeys + 1) * sizeof(u32), s);
    copy_d2d(d_starts, d_counts, (nkeys + 1) * sizeof(u32), s);
  }
  u64* d_entries = (u64*)dev_alloc(slots_max * sizeof(u64), s);
  u32 max_windows = 0;
  for (u32 j = 0; j < ncols; ++j)
    max_windows = std::max(max_windows, cols[j].n ? cols[j].num_windows : 0u);
  if (opt.scatter_window_major && max_windows > 1)
    launch(ScatterBody{d_cols, d_col_start, ncols, c, nbuckets, d_counts, d_entries, total_terms},
           total_terms * max_windows, s);
  else
    launch(ScatterBody{d_cols, d_col_start, ncols, c, nbuckets, d_counts, d_entries, 0},
           total_terms, s);
  // d_counts[k] is now the END offset of bucket k's real entries
  if (L)
    launch(FillPadsBody{d_starts, d_counts, d_entries}, nkeys, s);
  else
    launch(WindowUsedBody{d_counts, nbuckets, d_window_used}, plan.total_windows, s);

  B200_LOG(3, "range [%llu, %llu): %llu terms, %llu entries max, c=%u, %llu keys, pair levels %u",
           (unsigned long long)begin, (unsigned long long)end, (unsigned long long)total_terms,
           (unsigned long long)max_entries, c, (unsigned long long)nkeys, L);
  std::vector<void*> to_free;
  const typename C::Gen* walk_gens = gens;
  const u64* walk_entries = d_entries;
  u64 m_max = max_entries;
  u32* m_ptr = d_m;
  if (hook)
    hook->before_accumulate();
  KernelTimer::get().begin(s);
  StageRange nvtx_acc("msm: bucket accumulation");
  if constexpr (C::kBatchAffine) {
    if (L) {
      typedef typename C::F F;
      typedef typename F::E fe;
      typedef typename C::Gen Gen;
      // pairs per thread halve from level to level (a thread's sums are its own next-level inputs)
      u32 B = opt.pair_batch ? opt.pair_batch : 32u;
      while (B < (1u << L))
        B *= 2;
      B = (B >> (L - 1)) << (L - 1);
      const u64 T = ((slots_max >> 1) + B - 1) / B;  // the same threads at every level
      // The level is cut in two halves of threads (A, B) on two streams. The heavy passes are chained
      // A, B, A, B, ... by events, so the inversion tree of one half (a chain of small latency-bound
      // kernels ending in one Fermat inversion) runs under the heavy pass of the other half instead
      // of leaving the GPU idle once per level. A thread's next-level inputs are its own outputs, so
      // the halves never read each other's data.
      stream_t s2 = aux_stream();
      const u64 Ta = T / 2, Tb = T - Ta;
      const Gen* in = nullptr;
      fe* pre = (fe*)dev_alloc((slots_max >> 1) * sizeof(fe), s);
      fe* totals = (fe*)dev_alloc(T * sizeof(fe), s);
      std::vector<void*> level_bufs = {pre, totals};
      {
        PairLevel<C> lv0{d_entries, gens, nullptr, d_m, 0, B};
        launch(PairPass1Body<C>{lv0, pre, totals, 0}, Ta, s);
        stream_follow(s2, s);
        launch(PairPass1Body<C>{lv0, pre, totals, Ta}, Tb, s2);
      }
      for (u32 l = 0; l < L; ++l) {
        const u64 npairs = slots_max >> (l + 1);
        const bool last = l + 1 == L;
        // buffers of the next level come from the main stream's pool; the second stream touches
        // them only after following the main stream past this point
        Gen* out = (Gen*)dev_alloc(npairs * sizeof(Gen), s);
        fe* pre_next = last ? nullptr : (fe*)dev_alloc((npairs >> 1) * sizeof(fe), s);
        fe* totals_next = last ? nullptr : (fe*)dev_alloc(T * sizeof(fe), s);
        level_bufs.push_back(out);
        if (!last) {
          level_bufs.push_back(pre_next);
          level_bufs.push_back(totals_next);
        }
        PairLevel<C> lv{l == 0 ? d_entries : nullptr, l == 0 ? gens : nullptr, in, d_m, l, B >> l};
        const u32 desc = (l & 1u) ? 0u : 1u;
        batch_invert<F>(s, totals, Ta);
        stream_follow(s, s2);  // after the other half's previous heavy pass
        launch(PairPass2Body<C>{lv, pre, totals, out, pre_next, totals_next, desc, 0}, Ta, s);
        batch_invert<F>(s2, totals + Ta, Tb);
        stream_follow(s2, s);
        launch(PairPass2Body<C>{lv, pre, totals, out, pre_next, totals_next, desc, Ta}, Tb, s2);
        in = out;
        pre = pre_next;
        totals = totals_next;
      }
      stream_follow(s, s2);
      level_bufs.pop_back();  // the last level's points feed the chunk walk (freed with to_free)
      for (void* ptr : level_bufs)
        if (ptr != (void*)in)
          dev_free(ptr, s);
      m_max = slots_max >> L;
      u64* entries_l = (u64*)dev_alloc(m_max * sizeof(u64), s);
      launch(FinalEntriesBody{d_entries, d_m, L, entries_l, d_m + 9}, m_max, s);
      to_free.push_back((void*)in);
      to_free.push_back(entries_l);
      walk_gens = in;
      walk_entries = entries_l;
      m_ptr = d_m + 9;
    }
  }

  // a chunk of K entries leaves 2 pieces, so K must exceed 2 for the cascade to shrink
  // at C2, K = 64 trims the cascade more than it costs the first level
  const u32 chunk1_auto = m_max >= (1ull << 23) ? 64u : 32u;
  const u32 chunk1 = opt.chunk1 == 0 ? chunk1_auto : (opt.chunk1 < 4 ? 4u : opt.chunk1);
  const u32 chunkn = opt.chunkn < 4 ? 4u : opt.chunkn;
  Point* d_target = d_buckets;
  if (add_into)  // later ranges: own bucket array, merged into the shared one below
    d_target = (Point*)dev_alloc(nkeys * sizeof(Point), s);
  u32 K = chunk1;
  const u32* lvl_keys = nullptr;
  const Point* lvl_pieces = nullptr;
  bool first = true;
  int level = 0;
  stream_t cs = s;  // stream of the current cascade level
  for (;;) {
    bool final_level = m_max <= K;
    u64 T = (m_max + K - 1) / K;
    u32* out_keys = nullptr;
    Point* out_pieces = nullptr;
    u32* out_m = d_m + 1 + (level % 8);
    if (!final_level) {
      out_keys = (u32*)dev_alloc(2 * T * sizeof(u32), cs);
      out_pieces = (Point*)dev_alloc(2 * T * sizeof(Point), cs);
      to_free.push_back(out_keys);
      to_free.push_back(out_pieces);
    }
    const u32 fin = final_level ? 1u : 0u;
    if (first) {
      const u32 unit_z = (walk_gens == gens && opt.gens_normalized) ? 1u : 0u;
      // faster on ed25519 (a run start is a multiplication by a constant there); the Weierstrass
      // start is free, so the extra addition loses
      const bool uniform =
          opt.uniform_add == 2 ? C::kCurveId == kRistretto255 : opt.uniform_add != 0;
      if (uniform)
        launch(AccumulateBody<C, true, SeqExec, true>{nullptr, walk_entries, walk_gens, nullptr,
                                                      m_ptr, K, fin, d_target, out_keys, out_pieces,
                                                      out_m, unit_z},
               T, s);
      else
        launch(AccumulateBody<C, true>{nullptr, walk_entries, walk_gens, nullptr, m_ptr, K, fin,
                                       d_target, out_keys, out_pieces, out_m, unit_z},
               T, s);
      KernelTimer::get().end(s);
      if (tail != s) {
        stream_follow(tail, s);
        cs = tail;
      }
    } else if (T <= opt.quad_threshold) {
      launch(AccumulateBody<C, false, QuadExec>{lvl_keys, nullptr, nullptr, lvl_pieces, m_ptr, K,
                                                fin, d_target, out_keys, out_pieces, out_m, 0u},
             T * QuadExec::kLanes, cs);
    } else {
      launch(AccumulateBody<C, false>{lvl_keys, nullptr, nullptr, lvl_pieces, m_ptr, K, fin,
                                      d_target, out_keys, out_pieces, out_m, 0u},
             T, cs);
    }
    if (final_level)
      break;
    first = false;
    lvl_keys = out_keys;
    lvl_pieces = out_pieces;
    m_ptr = out_m;
    m_max = 2 * T;
    K = chunkn;
    ++level;
  }
  if (add_into) {
    launch(MergeBucketsBody<C>{d_counts, d_starts, d_target, d_buckets}, nkeys, cs);
    dev_free(d_target, cs);
  }
  for (void* ptr : to_free)
    dev_free(ptr, cs);
  dev_free(d_entries, s);
  dev_free(d_m, cs);
  dev_free(d_counts, cs);
  dev_free(d_starts, cs);
  dev_free(d_stage, s);
}

// Bucket reduction + window combination: out[j] for every column of the plan.
template <class C>
void msm_finish(stream_t s, const MsmPlan& plan, const typename C::Point* d_buckets,
                const u32* d_window_used, typename C::Point* out, const MsmOptions& opt) {
  typedef typename C::Point Point;
  StageRange nvtx_fin("msm: bucket reduction + window combination");
  const u32 total_windows = plan.total_windows, nbuckets = plan.nbuckets, ncols = plan.ncols;
  ColumnDesc* d_cols =
      (ColumnDesc*)stage_to_device(s, plan.cols.data(), ncols * sizeof(ColumnDesc));
  Point* d_S = nullptr;
  u32 m = nbuckets;
  const Point* X = d_buckets;
  const Point* Cin = nullptr;
  std::vector<void*> to_free;
  if (m == 1) {  // c == 1 is never chosen, but keep the degenerate case well-defined
    d_S = (Point*)dev_alloc(total_windows * sizeof(Point), s);
    copy_d2d(d_S, d_buckets, total_windows * sizeof(Point), s);
  }
  bool first = true;
  while (m > 1) {
    u32 g = first ? std::min<u32>(opt.reduce_g1, m) : std::min<u32>(opt.reduce_gn, m);
    u32 log2g = 0;
    while ((1u << log2g) < g)
      ++log2g;
    u32 m_out = m / g;
    Point* Xout = (Point*)dev_alloc((u64)total_windows * m_out * sizeof(Point), s);
    Point* Cout = (Point*)dev_alloc((u64)total_windows * m_out * sizeof(Point), s);
    if ((u64)total_windows * m_out <= opt.quad_threshold)  // uniform control flow: full-warp shuffles
      launch(ReduceBody<C, QuadExecConv>{X, Cin, m, g, log2g, Xout, Cout, d_window_used, nbuckets},
             (u64)total_windows * m_out * QuadExec::kLanes, s);
    else
      launch(ReduceBody<C>{X, Cin, m, g, log2g, Xout, Cout, d_window_used, nbuckets},
             (u64)total_windows * m_out, s);
    to_free.push_back(Xout);
    if (m_out > 1)
      to_free.push_back(Cout);
    X = Xout;
    Cin = Cout;
    m = m_out;
    first = false;
    if (m == 1)
      d_S = Cout;
  }
  for (void* ptr : to_free)
    dev_free(ptr, s);
  bool uniform_windows = true;  // same Horner trip count in every quad of a warp
  for (u32 j = 1; j < ncols; ++j)
    uniform_windows = uniform_windows && bucket_windows(plan.cols[j]) == bucket_windows(plan.cols[0]);
#ifdef B200_LANE_TAIL
  bool lane_done = false;
  if constexpr (C::kCurveId == kRistretto255) {
    if (ncols <= 2048 && opt.lane_tail) {  // one warp per column
      launch(CombineLaneBody{d_S, d_cols, plan.c, out}, (u64)ncols * 32, s);
      lane_done = true;
    }
  }
  if (lane_done) {
  } else
#endif
  if (ncols <= opt.quad_threshold && uniform_windows)
    launch(CombineBody<C, QuadExecConv>{d_S, d_cols, plan.c, out}, (u64)ncols * QuadExec::kLanes,
           s);
  else if (ncols <= opt.quad_threshold)
    launch(CombineBody<C, QuadExec>{d_S, d_cols, plan.c, out}, (u64)ncols * QuadExec::kLanes, s);
  else
    launch(CombineBody<C>{d_S, d_cols, plan.c, out}, ncols, s);
  dev_free(d_S, s);
  dev_free(d_cols, s);
}

// Computes out[j] = sum_i scalar(j,i) * G_i for every column j. `cols` are host descriptors whose
// `base` pointers are DEVICE pointers; gens and out are device arrays. The generator range is
// processed in `num_ranges` contiguous pieces that share one bucket array, so that the sort and
// accumulation of one piece overlap the arrival of the next. Everything is enqueued on `s`.
template <class C>
void msm_run(stream_t s, const typename C::Gen* gens, std::vector<ColumnDesc> cols,
             typename C::Point* out, const MsmOptions& opt = MsmOptions(), u32 num_ranges = 1,
             RangeHook* hook = nullptr, stream_t tail = stream_t()) {
  typedef typename C::Point Point;
  if (cols.empty())
    return;
  MsmPlan plan = msm_make_plan(std::move(cols), opt, sizeof(Point));
  B200_LOG(2, "msm: curve %u, %u columns, longest %llu, %llu terms, window %u bits, %u bucket sets%s",
           C::kCurveId, plan.ncols, (unsigned long long)plan.max_n,
           (unsigned long long)plan.total_terms, plan.c, plan.total_windows,
           plan.ncols && plan.cols[0].table_n ? " (fixed-base table)" : "");
  if (plan.total_terms == 0 || plan.total_windows == 0) {
    if (hook)
      hook->before_range(0, plan.max_n);
    launch(FillIdentityBody<C>{out}, plan.ncols, s);
    return;
  }
  Point* d_buckets = (Point*)dev_alloc(plan.nkeys * sizeof(Point), s);
  launch(FillIdentityBody<C>{d_buckets}, plan.nkeys, s);
  u32* d_window_used = (u32*)dev_alloc(plan.total_windows * sizeof(u32), s);
  dev_zero(d_window_used, plan.total_windows * sizeof(u32), s);
  if (num_ranges < 1)
    num_ranges = 1;
  // very long columns: enough ranges that each sort pass stays below the entry limit
  const u64 limit = opt.max_range_entries ? opt.max_range_entries : (1ull << 31);
  const u64 needed = (plan.total_entries + limit - 1) / limit;
  if (needed > num_ranges)
    num_ranges = (u32)std::min<u64>(needed, plan.max_n);
  // several ranges + a second stream: the cascade / merge of range r runs under range r+1
  const bool overlap = num_ranges > 1 && tail != stream_t() && tail != s;
  for (u32 r = 0; r < num_ranges; ++r) {
    u64 begin = range_begin(plan.max_n, r, num_ranges, opt.range_skew),
        end = range_begin(plan.max_n, r + 1, num_ranges, opt.range_skew);
    if (hook)
      hook->before_range(begin, end);
    msm_accumulate_range<C>(s, plan, gens, begin, end, r > 0, d_buckets, d_window_used, opt,
                            overlap ? tail : s, hook);
  }
  if (overlap)
    stream_follow(s, tail);
  msm_finish<C>(s, plan, d_buckets, d_window_used, out, opt);
  dev_free(d_window_used, s);
  dev_free(d_buckets, s);
}

}  // namespace b200
