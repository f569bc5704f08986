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
  // generator of row i (window w) is gens[gen_base + i + w * table_n], gens being the generator
  // pointer of the current range: per-column generator starts (commit_device_offsets); 0 otherwise
  u32 gen_base;
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
  // digit of window w from the low c bits of buf
  const auto step = [&] {
    u32 d = ((u32)buf & mask) + carry;
    buf >>= c;
    bool dneg = d > half;
    carry = dneg ? 1u : 0u;
    if (dneg)
      d = (1u << c) - d;
    if (d && (only_window == kAllWindows || w == only_window))
      f((col.first_window + (col.table_n ? 0u : w)) * nbuckets + (d - 1u), negative != dneg, w);
    ++w;
  };
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    buf |= (u64)v[k] << nb;
    nb += 32;
    for (; nb >= c && w < W; nb -= c)
      step();
  }
  while (w < W)
    step();
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
// f(key, entry) for every non-zero digit of term tid (only_window as for_each_digit)
template <class Fn>
B200_HD void for_each_entry(const ColumnDesc* cols, const u64* col_start, u32 ncols, u32 c,
                            u32 nbuckets, u64 tid, Fn f, u32 only_window = kAllWindows) {
  const u32 j = column_of(col_start, ncols, tid);
  const ColumnDesc col = cols[j];
  if (only_window != kAllWindows && only_window >= col.num_windows)
    return;
  const u64 i = tid - col_start[j];
  u32 v[8];
  bool neg;
  load_scalar_bits(v, neg, col, i);
  const u32 ii = (u32)i + col.gen_base, tn = col.table_n;
  for_each_digit(v, neg, col, c, nbuckets, [&](u32 key, bool negate, u32 w) {
    f(key, make_entry(key, ii + w * tn, negate));
  }, only_window);
}

struct CountBody {
  static constexpr int kBlock = 256;
  const ColumnDesc* cols;
  const u64* col_start;  // prefix of n over columns, ncols+1 entries
  u32 ncols, c, nbuckets;
  u32* counts;
  B200_HD void operator()(u64 tid) const {
    u32* cnt = counts;
    for_each_entry(cols, col_start, ncols, c, nbuckets, tid,
                   [cnt](u32 key, u64) { B200_ATOMIC_ADD(&cnt[key], 1u); });
  }
};

struct ScatterBody {
  static constexpr int kBlock = 256;
  const ColumnDesc* cols;
  const u64* col_start;
  u32 ncols, c, nbuckets;
  u32* cursor;  // exclusive offsets, consumed
  u64* entries;
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
    u32* cur = cursor;
    u64* en = entries;
    for_each_entry(cols, col_start, ncols, c, nbuckets, tid,
                   [cur, en](u32 key, u64 e) { en[B200_ATOMIC_ADD(&cur[key], 1u)] = e; }, only);
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

#if defined(__CUDACC__) && !defined(B200_EMULATE)
#define B200_BINNED_SORT 1
// ---- binned sort of the (term, window) entries (block-cooperative, CUDA only) ----------------------
// The same unpadded SortedLayout as CountBody -> exclusive_scan -> ScatterBody (sort_entries) without a
// global atomic or a scattered 8-byte store per entry:
//   1. MicroCountBody: per tile of terms, a shared-memory histogram of micro-bins (key >> shift),
//      flushed with one global atomic per non-zero counter
//   2. PlanBinsBody: one block scans the micro-bins and groups consecutive ones into bins of at most
//      kBinCap entries and kBinSpan keys; a micro-bin above kBinCap / 2 entries is a bin of its own
//   3. CoarseScatterBody: per tile, ranks its entries by bin in shared memory, reserves the tile's run
//      in every bin with one global atomic, and writes the runs to a temporary array
//   4. BinSortBody: per bin, counting sort by key in shared memory, final positions bin start + local
//      offset, and the bins' bucket end offsets. A bin above kBinCap entries (one micro-bin holding a
//      very dense bucket) is sorted the same way out of global memory.
constexpr u32 kMicroBins = 16384, kBinCap = 16384, kBinSpan = 4096, kMaxBinShift = 12;
// below this many entries the atomic path's fewer launches win (MsmOptions::sort_path = 1)
constexpr u64 kBinnedSortMinEntries = 1ull << 20;

// exclusive prefix of v over the block (kBlock threads, all of them call it); *total = block sum
template <int kBlock> __device__ u32 block_exclusive_scan(u32 v, u32* warp_sums, u32* total) {
  const u32 lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  u32 x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= (u32)d)
      x += y;
  }
  if (lane == 31)
    warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    u32 w = lane < kBlock / 32 ? warp_sums[lane] : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= (u32)d)
        w += y;
    }
    if (lane < kBlock / 32)
      warp_sums[lane] = w;
  }
  __syncthreads();
  const u32 pre = (warp ? warp_sums[warp - 1] : 0u) + x - v;
  *total = warp_sums[kBlock / 32 - 1];
  __syncthreads();  // warp_sums may be reused right away
  return pre;
}

struct MicroCountBody {
  static constexpr int kBlock = 512;
  const ColumnDesc* cols;
  const u64* col_start;
  u32 ncols, c, nbuckets;
  u64 total_terms;
  u32 tile, shift, nmicro;
  u32* micro_counts;  // [nmicro], zeroed
  __device__ void run(u32 b, unsigned char* smem) const {
    u32* h = (u32*)smem;
    for (u32 m = threadIdx.x; m < nmicro; m += kBlock)
      h[m] = 0;
    __syncthreads();
    const u64 lo = (u64)b * tile, hi = lo + tile < total_terms ? lo + tile : total_terms;
    const u32 sh = shift;
    for (u64 t = lo + threadIdx.x; t < hi; t += kBlock)
      for_each_entry(cols, col_start, ncols, c, nbuckets, t,
                     [h, sh](u32 key, u64) { atomicAdd(&h[key >> sh], 1u); });
    __syncthreads();
    for (u32 m = threadIdx.x; m < nmicro; m += kBlock)
      if (h[m])
        atomicAdd(&micro_counts[m], h[m]);
  }
};

struct PlanBinsBody {
  static constexpr int kBlock = 1024;
  const u32* micro_counts;
  u32 nmicro, span_micro;  // a bin never crosses a multiple of span_micro micro-bins
  u64 nkeys;
  u32* bin_of;      // [nmicro]: bin of every micro-bin
  u32* bin_start;   // [nmicro + 1]: first slot of bin b; [nbins] = M
  u32* bin_micro;   // [nmicro + 1]: first micro-bin of bin b; [nbins] = nmicro
  u32* bin_cursor;  // [nmicro]: = bin_start, consumed by the coarse scatter
  u32* nbins_out;
  u32* counts;  // counts[nkeys] = M
  u32* d_m;     // d_m[0] = M
  __device__ bool starts_bin(const u32* st, u32 m) const {
    constexpr u32 H = kBinCap / 2;
    return m == 0 || m % span_micro == 0 || micro_counts[m] > H || micro_counts[m - 1] > H ||
           st[m] / H != st[m - 1] / H;
  }
  __device__ void run(u32, unsigned char* smem) const {
    __shared__ u32 ws[32];
    u32* st = (u32*)smem;  // exclusive prefix of every micro-bin
    const u32 per = (nmicro + kBlock - 1) / kBlock, m0 = min(threadIdx.x * per, nmicro),
              m1 = min(m0 + per, nmicro);
    u32 sum = 0;
    for (u32 m = m0; m < m1; ++m)
      sum += micro_counts[m];
    u32 total;
    u32 run = block_exclusive_scan<kBlock>(sum, ws, &total);
    for (u32 m = m0; m < m1; ++m) {
      st[m] = run;
      run += micro_counts[m];
    }
    __syncthreads();
    u32 nf = 0;
    for (u32 m = m0; m < m1; ++m)
      nf += starts_bin(st, m) ? 1u : 0u;
    u32 nbins;
    u32 id = block_exclusive_scan<kBlock>(nf, ws, &nbins);
    for (u32 m = m0; m < m1; ++m) {
      if (starts_bin(st, m)) {
        bin_start[id] = st[m];
        bin_micro[id] = m;
        bin_cursor[id] = st[m];
        ++id;
      }
      bin_of[m] = id - 1;
    }
    if (threadIdx.x == 0) {
      bin_start[nbins] = total;
      bin_micro[nbins] = nmicro;
      *nbins_out = nbins;
      counts[nkeys] = total;
      d_m[0] = total;
    }
  }
};

// A tile's entries are ordered by bin in shared memory and each bin's run is written in one burst,
// so that a 32-byte sector of the temporary array is complete (or meets its neighbour run) while it
// is still in L2; written entry by entry as the digits are recoded, the runs of all resident tiles
// stay partially written for the whole kernel and the array (M x 8 B) does not fit in L2.
struct CoarseScatterBody {
  static constexpr int kBlock = 1024;
  const ColumnDesc* cols;
  const u64* col_start;
  u32 ncols, c, nbuckets;
  u64 total_terms;
  u32 tile, shift, nmicro;  // tile * (windows of a term) <= the staging capacity
  const u32* bin_of;
  const u32* nbins_ptr;
  u32* bin_cursor;
  u64* tmp;
  __device__ void run(u32 b, unsigned char* smem) const {
    __shared__ u32 ws[32];
    u32* h = (u32*)smem;       // per bin: the tile's count, then its next staging slot
    u32* delta = h + nmicro;   // per bin: global slot - staging slot of the bin's run
    u64* stage = (u64*)(delta + nmicro + (nmicro & 1u));
    const u32 nbins = *nbins_ptr;
    for (u32 k = threadIdx.x; k < nbins; k += kBlock)
      h[k] = 0;
    __syncthreads();
    const u64 lo = (u64)b * tile, hi = lo + tile < total_terms ? lo + tile : total_terms;
    const u32 sh = shift;
    const u32* map = bin_of;
    for (u64 t = lo + threadIdx.x; t < hi; t += kBlock)
      for_each_entry(cols, col_start, ncols, c, nbuckets, t,
                     [h, sh, map](u32 key, u64) { atomicAdd(&h[__ldg(&map[key >> sh])], 1u); });
    __syncthreads();
    const u32 per = (nbins + kBlock - 1) / kBlock, k0 = min(threadIdx.x * per, nbins),
              k1 = min(k0 + per, nbins);
    u32 sum = 0;
    for (u32 k = k0; k < k1; ++k)
      sum += h[k];
    u32 size;
    u32 run = block_exclusive_scan<kBlock>(sum, ws, &size);
    for (u32 k = k0; k < k1; ++k) {
      const u32 n = h[k];
      if (n)
        delta[k] = atomicAdd(&bin_cursor[k], n) - run;
      h[k] = run;
      run += n;
    }
    __syncthreads();
    for (u64 t = lo + threadIdx.x; t < hi; t += kBlock)
      for_each_entry(cols, col_start, ncols, c, nbuckets, t, [h, sh, map, stage](u32 key, u64 e) {
        stage[atomicAdd(&h[__ldg(&map[key >> sh])], 1u)] = e;
      });
    __syncthreads();
    for (u32 i = threadIdx.x; i < size; i += kBlock) {
      const u64 e = stage[i];
      tmp[delta[__ldg(&map[entry_key(e) >> sh])] + i] = e;  // u32 wrap-around: slot < 2^32
    }
  }
};

// A bin's entries are read twice from the temporary array, for the histogram and for the placement;
// the second read finds them in L2. Only the ordered bin is held in shared memory, so a bin can hold
// kBinCap = 16384 entries in 144 KB: twice the entries of a copy-then-order layout, so half as many
// bins for the coarse scatter to count, scan and reserve per tile, and runs per bin twice as long.
struct BinSortBody {
  static constexpr int kBlock = 1024;
  static constexpr size_t kSmem = kBinCap * sizeof(u64) + kBinSpan * sizeof(u32);
  const u64* tmp;
  const u32* bin_start;
  const u32* bin_micro;
  const u32* nbins_ptr;
  u32 shift;
  u64 nkeys;
  u64* entries;
  u32* counts;  // END offset of every bucket
  __device__ void run(u32 b, unsigned char* smem) const {
    __shared__ u32 ws[32];
    if (b >= *nbins_ptr)
      return;
    u64* sorted = (u64*)smem;
    u32* h = (u32*)(smem + kBinCap * sizeof(u64));
    const u32 lo = bin_start[b], size = bin_start[b + 1] - lo;
    const u64 klo = (u64)bin_micro[b] << shift, khi_m = (u64)bin_micro[b + 1] << shift;
    const u32 span = (u32)((khi_m < nkeys ? khi_m : nkeys) - klo);
    const bool local = size <= kBinCap;  // else: a dense micro-bin, placed straight into global memory
    for (u32 k = threadIdx.x; k < span; k += kBlock)
      h[k] = 0;
    __syncthreads();
#pragma unroll 4
    for (u32 i = threadIdx.x; i < size; i += kBlock)
      atomicAdd(&h[entry_key(tmp[(u64)lo + i]) - (u32)klo], 1u);
    __syncthreads();
    const u32 per = (span + kBlock - 1) / kBlock, k0 = min(threadIdx.x * per, span),
              k1 = min(k0 + per, span);
    u32 sum = 0;
    for (u32 k = k0; k < k1; ++k)
      sum += h[k];
    u32 total;
    u32 run = block_exclusive_scan<kBlock>(sum, ws, &total);
    for (u32 k = k0; k < k1; ++k) {
      const u32 n = h[k];
      h[k] = run;
      run += n;
      counts[klo + k] = lo + run;
    }
    __syncthreads();
    if (!local) {
      for (u32 i = threadIdx.x; i < size; i += kBlock) {
        const u64 e = tmp[(u64)lo + i];
        entries[(u64)lo + atomicAdd(&h[entry_key(e) - (u32)klo], 1u)] = e;
      }
      return;
    }
    // ordered in shared memory, then written out contiguously: one store per 32 entries of a warp
    // instead of one 32-byte sector per entry
#pragma unroll 4
    for (u32 i = threadIdx.x; i < size; i += kBlock) {
      const u64 e = tmp[(u64)lo + i];
      sorted[atomicAdd(&h[entry_key(e) - (u32)klo], 1u)] = e;
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < size; i += kBlock)
      entries[(u64)lo + i] = sorted[i];
  }
};

// micro-bin shift for nkeys keys; > kMaxBinShift: too many keys for the binned sort
inline u32 binned_sort_shift(u64 nkeys) {
  u32 shift = 0;
  while ((nkeys + (1ull << shift) - 1) >> shift > kMicroBins)
    ++shift;
  return shift;
}

// Binned sort of the entries of terms [0, total_terms) of d_cols into entries / counts / d_m[0].
inline void binned_sort(stream_t s, const ColumnDesc* d_cols, const u64* d_col_start, u32 ncols,
                        u32 c, u32 nbuckets, u64 total_terms, u64 max_entries, u32 max_windows,
                        u64 nkeys, u64* entries, u32* counts, u32* d_m) {
  const u32 shift = binned_sort_shift(nkeys);
  const u32 nmicro = (u32)((nkeys + (1ull << shift) - 1) >> shift);
  const u32 span_micro = std::max(1u, kBinSpan >> shift);
  // workspace: micro_counts, bin_of, bin_cursor [nmicro]; bin_start, bin_micro [nmicro + 1]; nbins
  u32* ws = (u32*)dev_alloc((5ull * nmicro + 3) * sizeof(u32), s);
  u32 *micro_counts = ws, *bin_of = ws + nmicro, *bin_cursor = ws + 2ull * nmicro,
      *bin_start = ws + 3ull * nmicro, *bin_micro = ws + 4ull * nmicro + 1,
      *nbins = ws + 5ull * nmicro + 2;
  u64* tmp = (u64*)dev_alloc(std::max<u64>(max_entries, 1) * sizeof(u64), s);
  dev_zero(micro_counts, nmicro * sizeof(u32), s);
  const u64 count_tile = 4096;
  launch_blocks(MicroCountBody{d_cols, d_col_start, ncols, c, nbuckets, total_terms,
                               (u32)count_tile, shift, nmicro, micro_counts},
                (total_terms + count_tile - 1) / count_tile, nmicro * sizeof(u32), s);
  launch_blocks(PlanBinsBody{micro_counts, nmicro, span_micro, nkeys, bin_of, bin_start, bin_micro,
                             bin_cursor, nbins, counts, d_m},
                1, nmicro * sizeof(u32), s);
  // scatter tiles: as many terms as the shared memory left by the two per-bin arrays can stage, in
  // whole rounds of the block's threads (a tile of 1.1 rounds recodes twice in a row on a tenth of
  // them while the rest wait at the barrier)
  const size_t scatter_smem = 220 * 1024;
  const size_t bin_bytes = (2ull * nmicro + 2) * sizeof(u32);
  const u64 stage_entries = (scatter_smem - bin_bytes) / sizeof(u64);
  u64 scatter_tile = std::max<u64>(1, stage_entries / max_windows);
  if (scatter_tile > (u64)CoarseScatterBody::kBlock)
    scatter_tile -= scatter_tile % CoarseScatterBody::kBlock;
  launch_blocks(CoarseScatterBody{d_cols, d_col_start, ncols, c, nbuckets, total_terms,
                                  (u32)scatter_tile, shift, nmicro, bin_of, nbins, bin_cursor, tmp},
                (total_terms + scatter_tile - 1) / scatter_tile, scatter_smem, s);
  launch_blocks(BinSortBody{tmp, bin_start, bin_micro, nbins, shift, nkeys, entries, counts}, nmicro,
                BinSortBody::kSmem, s);
  dev_free(tmp, s);
  dev_free(ws, s);
}
#endif

// p[0 .. n) = identity, one 16-byte store per thread: consecutive threads write consecutive 16 bytes,
// so every store instruction of a warp covers 512 contiguous bytes (a thread per point strides the
// warp's stores by the point size and leaves every sector partially written)
template <class C> struct FillIdentityBody {
  static constexpr int kBlock = 256;
  static constexpr u32 kChunks = sizeof(typename C::Point) / 16;
  static_assert(sizeof(typename C::Point) % 16 == 0, "points are made of 16-byte aligned fields");
  uint4* p;
  B200_HD void operator()(u64 t) const {
    const typename C::Point id = C::identity();
    const u32 k = (u32)(t % kChunks);
    uint4 v = ((const uint4*)&id)[0];
#pragma unroll
    for (u32 j = 1; j < kChunks; ++j)  // constant indices: the identity stays in registers
      if (j == k)
        v = ((const uint4*)&id)[j];
    p[t] = v;
  }
};
template <class C> inline void fill_identity(stream_t s, typename C::Point* p, u64 n) {
  launch(FillIdentityBody<C>{(uint4*)p}, n * FillIdentityBody<C>::kChunks, s);
}

// The real entries of bucket k of a sorted range are the slots [begin(k), end(k)). A padded layout
// keeps every bucket's start; in a dense one a bucket starts where the previous one ends.
struct BucketOffsets {
  const u32* ends;    // end offset of every bucket's real entries
  const u32* starts;  // padded layouts: start offset of every bucket, nkeys + 1; null = dense layout
  B200_HD u32 begin(u64 k) const { return starts ? starts[k] : (k ? ends[k - 1] : 0u); }
  B200_HD u32 end(u64 k) const { return ends[k]; }
};

// buckets[k] += scratch[k] for every bucket the current generator range touched. A later range
// accumulates into its own scratch array and is merged here: one coalesced pass, instead of a
// read-add-write at every run boundary of the accumulation kernel (about twice as fast per piece at
// C2 in 4 pieces).
template <class C> struct MergeBucketsBody {
  static constexpr int kBlock = 128;
  BucketOffsets offsets;
  const typename C::Point* scratch;
  typename C::Point* buckets;
  B200_HD void operator()(u64 k) const {
    if (offsets.begin(k) == offsets.end(k))
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
// kUnitZ (gathering level, ed25519 only): every generator is normalised (Z = 1: a fixed-base table, or
// caller generators normalised at ingestion), so an addition takes 7 multiplications and the gather
// never loads Gen::Z2 (96 of the 128 bytes). unit_veto, when set, is a device flag read once at
// entry: non-zero means the ingestion met Z = 0 and left the generators as they came, and the
// 8-multiplication path over the whole Gen runs instead.
template <class C, bool kGather, class X = SeqExec, bool kUniform = false, bool kUnitZ = false>
struct AccumulateBody {
  static constexpr int kBlock = 128;
  // register cap: 168 (3 blocks/SM) for 8-limb fields; 12-limb bls12-381 keeps 255 (2 blocks/SM)
  static constexpr int kMinBlocks = !kGather ? 1 : (C::F::N > 8 ? 2 : 3);
  typedef typename C::Point Point;
  typedef typename C::Gen Gen;
  const u32* keys;                 // level >= 2
  const u64* entries;              // level 1: sorted entries
  const Gen* gens;                 // level 1
  const Point* pieces;             // level >= 2
  const u32* m_ptr;                // number of entries at this level (device)
  u32 K;
  u32 final_level;
  Point* buckets;
  u32* out_keys;
  Point* out_pieces;
  u32* out_m_ptr;
  const u32* unit_veto;  // kUnitZ: device flag, non-zero = run the 8-multiplication path; may be null

  // The run of `key` in chunk t ends with the sum acc. Every bucket is written exactly once per
  // generator range: a run after the chunk's first is complete (it started inside the chunk), and so
  // is every run of the final level; the first run may continue in the previous chunk, so it travels
  // down the cascade as the chunk's first piece and is written by the level that completes it.
  B200_HD void close_run(u64 t, u32 key, const Point& acc, bool writer, bool& first_seg) const {
    if (final_level || !first_seg) {
      if (writer)
        buckets[key] = acc;
    } else if (writer) {
      out_keys[2 * t] = key;
      out_pieces[2 * t] = acc;
    }
    first_seg = false;
  }
  template <bool kUnit> B200_HD Gen load_gen(u32 idx) const {
    if constexpr (kUnit)
      return C::load_unit_gen(gens + idx);
    else
      return gens[idx];
  }
  // level 1: sums entries [b, e) of chunk t
  template <bool kUnit>
  B200_HD void gather_walk(u64 t, u64 b, u64 e, bool writer, u32& cur, Point& acc,
                           bool& first_seg) const {
    // software-pipelined gather: the generator of entry i+1 is loaded into registers before the
    // addition of entry i starts, so the random 128-byte read overlaps ~1300 instructions of
    // field arithmetic instead of stalling the warp on the long scoreboard
    u64 ent = entries[b];
    Gen g = load_gen<kUnit>(entry_gen(ent));
    cur = entry_key(ent);
    for (u64 i = b; i < e; ++i) {
      u64 ent_n = ent;
      Gen g_n = g;
      if (i + 1 < e) {
        ent_n = entries[i + 1];
        g_n = load_gen<kUnit>(entry_gen(ent_n));
      }
      const u32 k = entry_key(ent);
      const bool negate = entry_negate(ent);
      if (kUniform) {
        if (i == b || k != cur) {
          if (i != b) {
            close_run(t, cur, acc, writer, first_seg);
            cur = k;
          }
          acc = C::identity();
        }
        C::template add_gen<X>(acc, acc, g, negate, kUnit);
      } else {
        const bool start = i == b || k != cur;
        if (k != cur) {
          close_run(t, cur, acc, writer, first_seg);
          cur = k;
        }
        if (start)
          C::gen_to_point(acc, g, negate);
        else
          C::template add_gen<X>(acc, acc, g, negate, kUnit);
      }
      ent = ent_n;
      g = g_n;
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
    if constexpr (kGather) {
      if (kUnitZ && unit_veto && *unit_veto)
        gather_walk<false>(t, b, e, writer, cur, acc, first_seg);
      else
        gather_walk<kUnitZ>(t, b, e, writer, cur, acc, first_seg);
    } else {
      cur = keys[b];
      acc = pieces[b];
      for (u64 i = b + 1; i < e; ++i) {
        const u32 k = keys[i];
        if (k == cur) {
          C::template add<X>(acc, acc, pieces[i]);
        } else {
          close_run(t, cur, acc, writer, first_seg);
          cur = k;
          acc = pieces[i];
        }
      }
    }
    if (final_level) {
      close_run(t, cur, acc, writer, first_seg);
      return;
    }
    if (!writer)
      return;
    if (first_seg) {  // single-run chunk: it is the first piece, the identity pads the second
      close_run(t, cur, acc, writer, first_seg);
      acc = C::identity();
    }
    out_keys[2 * t + 1] = cur;
    out_pieces[2 * t + 1] = acc;
  }
};

// window_used[w] |= (some entry of this pass landed in window w). A bucket is padded to zero slots
// exactly when it has no entry, so the padded offsets answer this as well as the dense ones.
struct WindowUsedBody {
  static constexpr int kBlock = 64;
  BucketOffsets offsets;
  u32 nbuckets;
  u32* window_used;
  B200_HD void operator()(u64 w) const {
    if (offsets.begin(w * nbuckets) != offsets.begin((w + 1) * nbuckets))
      window_used[w] = 1u;
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
// Several pieces of generators in one launch (per-column generator starts, GenLayout): piece k moves
// start[k+1] - start[k] generators from source index from[k] to device position to[k]. A thread finds
// its piece by binary search over the prefix `start`, then runs the one-piece body's element code.
struct GenPieces {
  const u64* start;  // [npieces + 1]
  const u64* from;   // [npieces]
  const u64* to;     // [npieces]
  u32 npieces;
};
template <class C> struct IngestPiecesBody {
  static constexpr int kBlock = IngestBody<C, false>::kBlock;
  const unsigned char* raw;  // ABI-layout generators, indexed by `from`
  typename C::Gen* gens;
  GenPieces p;
  B200_HD void operator()(u64 tid) const {
    const u32 k = column_of(p.start, p.npieces, tid);
    IngestBody<C, false>{raw + p.from[k] * C::kAbiGenBytes, gens + p.to[k]}(tid - p.start[k]);
  }
};
struct BuiltinPiecesBody {
  static constexpr int kBlock = BuiltinGeneratorBody::kBlock;
  Ed25519::Gen* gens;
  GenPieces p;  // `from` = index of the built-in generator
  B200_HD void operator()(u64 tid) const {
    const u32 k = column_of(p.start, p.npieces, tid);
    BuiltinGeneratorBody{gens + p.to[k], p.from[k]}(tid - p.start[k]);
  }
};

// ---- normalising ingestion (ed25519) ---------------------------------------------------------------
// Caller generators come with any Z. Scaled by 1/Z (all four coordinates, so the projective point is
// the same whatever its T) they have Z = 1 and 2Z = 2, and every bucket addition over them takes 7
// multiplications instead of 8 (add_gen, unit_z) and gathers 96 bytes instead of 128
// (AccumulateBody kUnitZ). A range of n generators is normalised by Montgomery's trick in two passes
// around the inversion of the group products; thread j owns the generators j, j + T, j + 2T, ...
// (T = ceil(n / kBatchGroup), so that a warp reads and writes consecutive generators):
//   NormalizeUpBody:   reads only Z (40 of the 160 ABI bytes), writes the prefix products and the
//                      group product
//   the T group products are inverted (batch_invert; on CUDA NormalizeUpBlockBody and
//                      NormalizeMidBody below, so that the whole normalisation is three launches)
//   NormalizeDownBody: walks the group backwards, peeling 1/Z off the inverted product, and writes
//                      the scaled generator in the device layout (IngestBody's only write)
// Z = 0 is not a point: it counts as 1 in the products and sets *invalid. The down pass of a range
// that finds *invalid set writes the generators unscaled, exactly as IngestBody, and the gathering
// level, which reads the same flag, runs its 8-multiplication path over them.
struct IngestMap {  // ingestion thread i: ABI generator src of `raw` -> device generator dst
  GenPieces p;      // npieces == 0: src = dst = i
  B200_HD void at(u64 i, u64& src, u64& dst) const {
    if (p.npieces == 0) {
      src = dst = i;
      return;
    }
    const u32 k = column_of(p.start, p.npieces, i);
    src = p.from[k] + (i - p.start[k]);
    dst = p.to[k] + (i - p.start[k]);
  }
};
constexpr u32 kNormBlock = 256;  // groups per block of the CUDA up pass
struct NormalizeUpBody {
  static constexpr int kBlock = 128;
  typedef F25519 F;
  const unsigned char* raw;
  IngestMap map;
  u64 n, T;
  F::E* pre;   // [n]
  F::E* prod;  // [T]
  u32* invalid;
  // prefix products of group j into pre; returns the group product
  B200_HD F::E group(u64 j) const {
    F::E z[kBatchGroup], acc = F::one();
#pragma unroll
    for (u32 k = 0; k < kBatchGroup; ++k) {  // all loads first: 8 reads in flight per thread
      const u64 i = j + k * T;
      z[k] = F::one();
      if (i < n) {
        u64 src, dst;
        map.at(i, src, dst);
        z[k] = Ed25519::load_abi_z(raw + src * Ed25519::kAbiGenBytes);
      }
    }
#pragma unroll
    for (u32 k = 0; k < kBatchGroup; ++k) {
      const u64 i = j + k * T;
      if (i >= n)
        break;
      if (F::is_zero(z[k])) {
        *invalid = 1u;
        z[k] = F::one();
      }
      pre[i] = acc;
      F::mul(acc, acc, z[k]);
    }
    return acc;
  }
  B200_HD void operator()(u64 j) const { prod[j] = group(j); }
};
struct NormalizeDownBody {
  static constexpr int kBlock = 128;
  typedef F25519 F;
  const unsigned char* raw;
  IngestMap map;
  u64 n, T;
  const F::E* pre;
  const F::E* prod;  // inverted: of every group, or (with ps) of every block of kNormBlock groups
  const F::E* ps;    // null, or per group the product of the other groups of its block
  const u32* invalid;
  Ed25519::Gen* gens;
  B200_HD void operator()(u64 j) const {
    const bool scale = *invalid == 0;
    F::E inv = prod[ps ? j / kNormBlock : j];
    if (ps)
      F::mul(inv, inv, ps[j]);
    for (u32 k = kBatchGroup; k-- > 0;) {
      const u64 i = j + k * T;
      if (i >= n)
        continue;
      u64 src, dst;
      map.at(i, src, dst);
      Ed25519::Point p;
      Ed25519::load_point_abi(p, raw + src * Ed25519::kAbiGenBytes);
      if (scale) {  // no Z of the range is 0
        F::E zi;
        F::mul(zi, inv, pre[i]);
        F::mul(inv, inv, p.Z);
        F::mul(p.X, p.X, zi);
        F::mul(p.Y, p.Y, zi);
        F::mul(p.T, p.T, zi);
        p.Z = F::one();
      }
      Ed25519::Gen g;
      Ed25519::point_to_gen(g, p);
      gens[dst] = g;
    }
  }
};
#ifdef B200_BINNED_SORT
// CUDA: the T group products are inverted in two more kernels instead of batch_invert's tree (a
// chain of ~10 small launches that, beside the sort's large blocks, each wait for a free SM):
//   NormalizeUpBlockBody: the up pass, plus per block of kNormBlock groups the exclusive prefix and
//                         suffix products of the group products (warp shuffles): ps[j] = product of
//                         the other groups of the block, prod[b] = the block's product
//   NormalizeMidBody:     one block inverts the blocks' products in place (Montgomery's trick over
//                         chunks, the same scans across the chunks, one inversion)
//   NormalizeDownBody:    1 / (group product) = prod[b] * ps[j]
__device__ __forceinline__ F25519::E shfl_up_fe(const F25519::E& a, u32 d) {
  F25519::E r;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    r.l[k] = __shfl_up_sync(0xffffffffu, a.l[k], d);
  return r;
}
__device__ __forceinline__ F25519::E shfl_down_fe(const F25519::E& a, u32 d) {
  F25519::E r;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    r.l[k] = __shfl_down_sync(0xffffffffu, a.l[k], d);
  return r;
}
// exclusive prefix (P) and suffix (S) products of x over the kBlock threads of the block, and the
// block's product (every thread); ws: kBlock / 32 elements of shared memory
template <int kBlock>
__device__ void block_prefix_suffix(const F25519::E& x, F25519::E& P, F25519::E& S,
                                    F25519::E& total, F25519::E* ws) {
  typedef F25519 F;
  const u32 lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  F::E inc = x, sinc = x;
#pragma unroll
  for (u32 d = 1; d < 32; d <<= 1) {
    const F::E y = shfl_up_fe(inc, d), z = shfl_down_fe(sinc, d);
    if (lane >= d)
      F::mul(inc, inc, y);
    if (lane + d < 32)
      F::mul(sinc, sinc, z);
  }
  F::E pe = shfl_up_fe(inc, 1), se = shfl_down_fe(sinc, 1);
  if (lane == 0)
    pe = F::one();
  if (lane == 31) {
    se = F::one();
    ws[warp] = inc;
  }
  __syncthreads();
  F::E before = F::one(), after = F::one();
  for (u32 w = 0; w < kBlock / 32; ++w) {
    if (w < warp)
      F::mul(before, before, ws[w]);
    else if (w > warp)
      F::mul(after, after, ws[w]);
  }
  F::mul(P, before, pe);
  F::mul(S, se, after);
  F::mul(total, before, ws[warp]);
  F::mul(total, total, after);
  __syncthreads();  // ws may be reused right away
}
struct NormalizeUpBlockBody {
  static constexpr int kBlock = kNormBlock;
  typedef F25519 F;
  NormalizeUpBody up;
  F::E* ps;    // [T]
  F::E* prod;  // [blocks]
  __device__ void run(u32 b, unsigned char*) const {
    __shared__ F::E ws[kBlock / 32];
    const u64 j = (u64)b * kBlock + threadIdx.x;
    const F::E g = j < up.T ? up.group(j) : F::one();
    F::E P, S, total;
    block_prefix_suffix<kBlock>(g, P, S, total, ws);
    if (j < up.T)
      F::mul(ps[j], P, S);
    if (threadIdx.x == 0)
      prod[b] = total;
  }
};
struct NormalizeMidBody {
  static constexpr int kBlock = 1024;
  typedef F25519 F;
  F::E* vals;  // [m], inverted in place
  F::E* pre;   // [m] scratch
  u64 m;
  __device__ void run(u32, unsigned char*) const {
    __shared__ F::E ws[kBlock / 32];
    __shared__ F::E inv_total;
    const u64 per = (m + kBlock - 1) / kBlock, lo = min((u64)threadIdx.x * per, m),
              hi = min(lo + per, m);
    F::E c = F::one();
    for (u64 k = lo; k < hi; ++k) {
      pre[k] = c;
      F::mul(c, c, vals[k]);
    }
    F::E P, S, total;
    block_prefix_suffix<kBlock>(c, P, S, total, ws);
    if (threadIdx.x < 32) {  // 1 / total = total^(p - 2) = (total^(2^252 - 3))^8 * total^3, on 10 lanes
      const lane10::Lane L = lane10::lane_info();
      const u32 z = lane10::slice(L, total);
      const u32 z3 = lane10::mul(L, lane10::mul(L, z, z), z);
      const u32 r = lane10::mul(L, lane10::sqr_n(L, lane10::pow22523(L, z), 3), z3);
      F::E inv;
      lane10::gather(inv, r, 0);
      if (threadIdx.x == 0)
        inv_total = inv;
    }
    __syncthreads();
    F::E inv;  // 1 / c
    F::mul(inv, inv_total, P);
    F::mul(inv, inv, S);
    for (u64 k = hi; k-- > lo;) {
      const F::E v = vals[k];
      F::mul(vals[k], inv, pre[k]);
      F::mul(inv, inv, v);
    }
  }
};
#endif
// IngestBody (map without pieces) / IngestPiecesBody of n generators, normalised; enqueued on s.
// *invalid is zeroed by the caller once per call and set here when a generator has Z = 0.
inline void ingest_normalized(stream_t s, const unsigned char* raw, Ed25519::Gen* gens,
                              const IngestMap& map, u64 n, u32* invalid) {
  typedef F25519::E fe;
  if (n == 0)
    return;
  const u64 T = (n + kBatchGroup - 1) / kBatchGroup;
  fe* pre = (fe*)dev_alloc(n * sizeof(fe), s);
  const NormalizeUpBody up{raw, map, n, T, pre, nullptr, invalid};
#ifdef B200_BINNED_SORT
  const u64 blocks = (T + kNormBlock - 1) / kNormBlock;
  fe* ps = (fe*)dev_alloc((T + 2 * blocks) * sizeof(fe), s);
  fe* prod = ps + T;
  launch_blocks(NormalizeUpBlockBody{up, ps, prod}, blocks, 0, s);
  launch_blocks(NormalizeMidBody{prod, prod + blocks, blocks}, 1, 0, s);
  launch(NormalizeDownBody{raw, map, n, T, pre, prod, ps, invalid, gens}, T, s);
  dev_free(ps, s);
#else
  fe* prod = (fe*)dev_alloc(T * sizeof(fe), s);
  NormalizeUpBody u = up;
  u.prod = prod;
  launch(u, T, s);
  batch_invert<F25519>(s, prod, T);
  launch(NormalizeDownBody{raw, map, n, T, pre, prod, nullptr, invalid, gens}, T, s);
  dev_free(prod, s);
#endif
  dev_free(pre, s);
}
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
    // the largest generator index of the column's entries fits the entry's 31-bit field
    if (col.n)
      B200_REQUIRE((u64)col.gen_base + col.n + (u64)(col.num_windows - 1) * col.table_n < (1ull << 31),
                   "generator index of a column too large");
  }
  p.nkeys = (u64)p.total_windows * p.nbuckets;
  p.total_entries = max_entries;
  B200_REQUIRE(p.nkeys < (1ull << 32), "too many buckets for one pass");
  p.cols = std::move(cols);
  return p;
}

// The columns of a plan restricted to the terms [begin, end), staged with one H2D as a block
// [ColumnDesc x ncols][u64 x (ncols+1)]: descriptors, then the prefix of their lengths.
struct StagedRange {
  const ColumnDesc* d_cols = nullptr;  // the block; null when the range holds no term
  const u64* d_col_start = nullptr;
  u64 total_terms = 0, max_entries = 0;
  u32 max_windows = 0;  // windows of the widest non-empty column
  StagedRange(stream_t s, const MsmPlan& plan, u64 begin, u64 end) {
    const u32 ncols = plan.ncols;
    std::vector<ColumnDesc> cols(plan.cols);
    std::vector<u64> col_start(ncols + 1, 0);
    for (u32 j = 0; j < ncols; ++j) {
      u64 lo = std::min<u64>(begin, cols[j].n), hi = std::min<u64>(end, cols[j].n);
      cols[j].base += lo * cols[j].row_stride;
      cols[j].n = (u32)(hi - lo);
      col_start[j + 1] = col_start[j] + cols[j].n;
      max_entries += (u64)cols[j].n * cols[j].num_windows;
      max_windows = std::max(max_windows, cols[j].n ? cols[j].num_windows : 0u);
    }
    total_terms = col_start[ncols];
    if (total_terms == 0)
      return;
    B200_REQUIRE(max_entries < (1ull << 32) && end - begin < (1ull << 31),
                 "too many (term, window) entries for one sort pass");
    const size_t desc_bytes = ncols * sizeof(ColumnDesc), start_bytes = (ncols + 1) * sizeof(u64);
    std::vector<unsigned char> stage(desc_bytes + start_bytes);
    std::memcpy(stage.data(), cols.data(), desc_bytes);
    std::memcpy(stage.data() + desc_bytes, col_start.data(), start_bytes);
    d_cols = (const ColumnDesc*)stage_to_device(s, stage.data(), stage.size());
    d_col_start = (const u64*)((const unsigned char*)d_cols + desc_bytes);
  }
};

struct SortedLayout {  // the sorted (term, window) entries of one range, read by every later stage
  u64* entries;   // sorted entries; with L > 0 every bucket is followed by pad entries up to a
                  // multiple of 2^L slots
  u32* counts;    // [nkeys + 1]: counts[k] = END offset of bucket k's real entries
  u32* starts;    // [nkeys + 1]: padded start offset of every bucket; null when L = 0
  u32* d_m;       // [16]: d_m[0] = number of slots; the rest is scratch of the later stages
  u64 slots_max;  // slots allocated for `entries` (bound on d_m[0])
  bool binned;    // sorted by the binned path
  BucketOffsets offsets() const { return {counts, starts}; }
};

// Sorts a staged range into a SortedLayout and flags window_used[w] for every window with an entry.
// The binned sort (CUDA build) serves unpadded layouts (L = 0) of at most kMicroBins << kMaxBinShift
// keys: always with opt.sort_path 2, from kBinnedSortMinEntries entries on with 1. The atomic count +
// scan + scatter sorts every other case.
inline SortedLayout sort_entries(stream_t s, const MsmPlan& plan, const StagedRange& r, u32 L,
                                 const MsmOptions& opt, u32* window_used) {
  const u32 ncols = plan.ncols, c = plan.c, nbuckets = plan.nbuckets;
  const u64 nkeys = plan.nkeys, max_entries = r.max_entries, total_terms = r.total_terms;
  SortedLayout out{};
  out.slots_max = L ? ((max_entries + nkeys * ((1ull << L) - 1) + (1ull << L) - 1) >> L) << L : max_entries;
  out.counts = (u32*)dev_alloc((nkeys + 1) * sizeof(u32), s);
  out.d_m = (u32*)dev_alloc(16 * sizeof(u32), s);
  out.entries = (u64*)dev_alloc(out.slots_max * sizeof(u64), s);
#ifdef B200_BINNED_SORT
  out.binned = L == 0 && opt.sort_path != 0 && binned_sort_shift(nkeys) <= kMaxBinShift &&
               (opt.sort_path == 2 || max_entries >= kBinnedSortMinEntries);
  if (out.binned)
    binned_sort(s, r.d_cols, r.d_col_start, ncols, c, nbuckets, total_terms, max_entries,
                r.max_windows, nkeys, out.entries, out.counts, out.d_m);
#endif
  if (!out.binned) {
    dev_zero(out.counts, (nkeys + 1) * sizeof(u32), s);
    launch(CountBody{r.d_cols, r.d_col_start, ncols, c, nbuckets, out.counts}, total_terms, s);
    if (L)
      launch(PadCountsBody{out.counts, (1u << L) - 1u}, nkeys, s);
    exclusive_scan(out.counts, nkeys + 1, s);  // counts[nkeys] = number of (padded) entries
    copy_d2d(out.d_m, out.counts + nkeys, sizeof(u32), s);
    if (L) {
      out.starts = (u32*)dev_alloc((nkeys + 1) * sizeof(u32), s);
      copy_d2d(out.starts, out.counts, (nkeys + 1) * sizeof(u32), s);
    }
    const bool window_major = opt.scatter_window_major && r.max_windows > 1;
    launch(ScatterBody{r.d_cols, r.d_col_start, ncols, c, nbuckets, out.counts, out.entries,
                       window_major ? total_terms : 0},
           window_major ? total_terms * r.max_windows : total_terms, s);
  }
  if (L)
    launch(FillPadsBody{out.starts, out.counts, out.entries}, nkeys, s);
  launch(WindowUsedBody{out.offsets(), nbuckets, window_used}, plan.total_windows, s);
  return out;
}

// Sorts `cols` (host descriptors over device scalars, window width c; 0 = automatic) with sort_entries
// forced to the atomic and to the binned path and returns the number of buckets whose end offset or
// entry multiset differs between the two (0 = agree; ~0u when the binned path does not apply).
inline unsigned sort_selftest(stream_t s, std::vector<ColumnDesc> cols, u32 c) {
  MsmOptions opt;
  opt.window_bits = c;
  const MsmPlan plan = msm_make_plan(std::move(cols), opt, 160);
  const StagedRange r(s, plan, 0, plan.max_n);
  if (r.total_terms == 0)
    return ~0u;
  const u64 nkeys = plan.nkeys, M = r.max_entries;
  DevBuf<u32> window_used(plan.total_windows, s);  // not compared: both paths set it from the counts
  opt.sort_path = 0;
  const SortedLayout a = sort_entries(s, plan, r, 0, opt, window_used.p);
  opt.sort_path = 2;
  const SortedLayout b = sort_entries(s, plan, r, 0, opt, window_used.p);
  std::vector<u32> ca(nkeys + 1), cb(nkeys + 1), m(1);
  std::vector<u64> ea(M), eb(M);
  copy_d2h(ca.data(), a.counts, (nkeys + 1) * sizeof(u32), s);
  copy_d2h(cb.data(), b.counts, (nkeys + 1) * sizeof(u32), s);
  copy_d2h(m.data(), b.d_m, sizeof(u32), s);
  copy_d2h(ea.data(), a.entries, M * sizeof(u64), s);
  copy_d2h(eb.data(), b.entries, M * sizeof(u64), s);
  stream_sync(s);
  for (void* p : {(void*)a.entries, (void*)a.counts, (void*)a.d_m, (void*)b.entries, (void*)b.counts,
                  (void*)b.d_m, (void*)r.d_cols})
    dev_free(p, s);
  if (!b.binned)
    return ~0u;
  unsigned bad = m[0] == ca[nkeys] ? 0u : 1u;  // M: counts[nkeys] of the atomic path
  for (u64 k = 0; k < nkeys; ++k) {
    const u32 lo = k ? ca[k - 1] : 0u, hi = ca[k];
    if (cb[k] != hi || hi < lo || hi > M) {
      ++bad;
      continue;
    }
    std::sort(ea.begin() + lo, ea.begin() + hi);
    std::sort(eb.begin() + lo, eb.begin() + hi);
    if (!std::equal(ea.begin() + lo, ea.begin() + hi, eb.begin() + lo))
      ++bad;
  }
  return bad;
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

// Chunk walk of `walk` into `target`, then the cascade over its pieces (appended to to_free) on `tail`
// when it differs from s. Returns the stream of the last level. unit: walk.gens are normalised
// (Z = 1) unless *unit_veto is set on the device (AccumulateBody kUnitZ).
template <class C>
stream_t chunk_walk(stream_t s, stream_t tail, WalkInput<C> walk, u32* d_m, bool unit,
                    const u32* unit_veto, typename C::Point* target, const MsmOptions& opt,
                    std::vector<void*>& to_free) {
  typedef typename C::Point Point;
  // a chunk of K entries leaves 2 pieces, so K must exceed 2 for the cascade to shrink
  // at C2, K = 64 trims the cascade more than it costs the first level
  u32 K = opt.chunk1 ? std::max(opt.chunk1, 4u) : (walk.m_max >= (1ull << 23) ? 64u : 32u);
  const u32 chunkn = std::max(opt.chunkn, 4u);
  const u32* lvl_keys = nullptr;
  const Point* lvl_pieces = nullptr;
  stream_t cs = s;  // stream of the current cascade level
  for (int level = 0;; ++level) {
    const bool final_level = walk.m_max <= K;
    u64 T = (walk.m_max + K - 1) / K;
    u32* out_keys = final_level ? nullptr : (u32*)dev_alloc(2 * T * sizeof(u32), cs);
    Point* out_pieces = final_level ? nullptr : (Point*)dev_alloc(2 * T * sizeof(Point), cs);
    to_free.insert(to_free.end(), {out_keys, out_pieces});
    u32* out_m = d_m + 1 + (level % 8);
    // `body` only names the AccumulateBody instantiation: every level gets the same fields and reads
    // the ones it needs
    const auto launch_level = [&](auto body, u64 threads, stream_t st) {
      body = {lvl_keys, walk.entries, walk.gens, lvl_pieces, walk.m_ptr, K, final_level, target,
              out_keys, out_pieces, out_m, unit_veto};
      launch(body, threads, st);
    };
    if (level == 0) {
      // faster on ed25519 (a run start is a multiplication by a constant there); the Weierstrass
      // start is free, so the extra addition loses
      const bool uniform =
          opt.uniform_add == 2 ? C::kCurveId == kRistretto255 : opt.uniform_add != 0;
      // normalised generators change the addition on ed25519 only (Weierstrass generators are affine)
      constexpr bool kEd = C::kCurveId == kRistretto255;
      const bool unit_path = kEd && unit;
      if (uniform && unit_path)
        launch_level(AccumulateBody<C, true, SeqExec, true, kEd>{}, T, s);
      else if (uniform)
        launch_level(AccumulateBody<C, true, SeqExec, true>{}, T, s);
      else if (unit_path)
        launch_level(AccumulateBody<C, true, SeqExec, false, kEd>{}, T, s);
      else
        launch_level(AccumulateBody<C, true>{}, T, s);
      KernelTimer::get().end(s);
      if (tail != s)
        stream_follow(tail, s);
      cs = tail;
    } else if (T <= opt.quad_threshold) {
      launch_level(AccumulateBody<C, false, QuadExec>{}, T * QuadExec::kLanes, cs);
    } else {
      launch_level(AccumulateBody<C, false>{}, T, cs);
    }
    if (final_level)
      break;
    lvl_keys = out_keys;
    lvl_pieces = out_pieces;
    walk.m_ptr = out_m;
    walk.m_max = 2 * T;
    K = chunkn;
  }
  return cs;
}

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
  const StagedRange r(s, plan, begin, end);
  if (r.total_terms == 0)
    return;
  gens += begin;  // entry indices are relative to the range
  StageRange nvtx_sort("msm: digit count + scan + scatter");
  const u64 max_entries = r.max_entries, nkeys = plan.nkeys;
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
  const SortedLayout sorted = sort_entries(s, plan, r, L, opt, d_window_used);
  B200_LOG(3, "range [%llu, %llu): %llu terms, %llu entries max, c=%u, %llu keys, pair levels %u",
           (unsigned long long)begin, (unsigned long long)end, (unsigned long long)r.total_terms,
           (unsigned long long)max_entries, plan.c, (unsigned long long)nkeys, L);
  WalkInput<C> walk{gens, sorted.entries, sorted.d_m, max_entries};
  std::vector<void*> to_free;
  if (hook)
    hook->before_accumulate();
  KernelTimer::get().begin(s);
  StageRange nvtx_acc("msm: bucket accumulation");
  if constexpr (C::kBatchAffine) {
    if (L) {
      walk = run_pair_levels<C>(s, L, sorted.entries, gens, sorted.d_m, sorted.slots_max,
                                opt.pair_batch);
      to_free = {(void*)walk.gens, (void*)walk.entries};
    }
  }
  typedef typename C::Point Point;  // later ranges: own bucket array, merged into the shared one below
  Point* target = add_into ? (Point*)dev_alloc(nkeys * sizeof(Point), s) : d_buckets;
  const bool unit = walk.gens == gens && opt.gens_normalized;
  const stream_t cs =
      chunk_walk<C>(s, tail, walk, sorted.d_m, unit, opt.unit_veto, target, opt, to_free);
  // What the later levels and the merge read on cs (pieces, keys, d_m, counts, starts) is freed on cs:
  // freed on s, it could go to the next range's allocations while cs still reads it. So are the last
  // pair level's points and entries. The sorted entries and the staged columns are read on s only.
  if (add_into) {
    launch(MergeBucketsBody<C>{sorted.offsets(), target, d_buckets}, nkeys, cs);
    dev_free(target, cs);
  }
  to_free.insert(to_free.end(), {sorted.d_m, sorted.counts, sorted.starts});
  for (void* ptr : to_free)
    dev_free(ptr, cs);
  dev_free(sorted.entries, s);
  dev_free((void*)r.d_cols, s);
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
    fill_identity<C>(s, out, plan.ncols);
    return;
  }
  Point* d_buckets = (Point*)dev_alloc(plan.nkeys * sizeof(Point), s);
  fill_identity<C>(s, d_buckets, plan.nkeys);
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
