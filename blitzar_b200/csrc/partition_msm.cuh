// Fixed-base MSM outputs answered from a partition table held on the handle (Handle::ptable): for
// every group g of w generators the 2^w subset sums T[g][k] (ptable.cuh, PartitionGenStoreBody), as
// normalised device generators at entry (g << w) + k.
//
// Output j owns bits [bit_offset_j, bit_offset_j + b_j) of every scalar row and spans rows
// [0, len_j). Bit t of the output over group g is one lookup: k collects bit t of the group's w rows,
// and S_{j,t} = sum over the groups of T[g][k]. The output is then R_j = sum_t 2^t S_{j,t}.
//
// Replaces the reference's partition-table product (sxt/multiexp/pippenger2/partition_product.h:47-94,
// one thread per output bit walking every group; variable_length_partition_product.h for vlen) and
// its bit-wise combination (combine_reduce.h). Here:
//   PartitionAccumulateBody: one thread per (routed bit, chunk of groups), bit fastest, so adjacent
//       threads read the same scalar bytes; one mixed addition (add_gen, unit_z) per non-zero k;
//   PartitionFoldBody: the chunk partials of every bit, halved per launch (log-depth);
//   PartitionHornerBody: one thread per routed output, R = 2 R + S_{j,t} from the top bit down.
// The caller (CurveOps::fixed_device) routes outputs here per a cost model and leaves them as n = 0
// columns of the engine run, whose identity points the Horner pass overwrites.
#pragma once
#include <vector>

#include "msm.cuh"

namespace b200 {

struct PartitionBit {
  u32 pos;  // bit position inside a scalar row
  u32 len;  // rows of the bit's output (rows at or past len count as zero)
};
struct PartitionOut {
  u32 dest;       // output index in the call's point array
  u32 first_bit;  // the output's bit 0 among the routed bits
  u32 bits;       // its width b_j
};

template <class C> struct PartitionAccumulateBody {
  static constexpr int kBlock = 128;
  const typename C::Gen* table;  // groups x 2^w normalised entries
  const unsigned char* scalars;
  u64 row_stride;
  const PartitionBit* bits;
  typename C::Point* partial;  // [chunk][bit]
  u32 nbits, w, chunk_groups;
  B200_HD void operator()(u64 t) const {
    const PartitionBit b = bits[t % nbits];
    const unsigned char* col = scalars + (b.pos >> 3);
    const u32 sh = b.pos & 7u;
    typename C::Point acc = C::identity();
    const u64 g0 = t / nbits * chunk_groups;
    for (u64 g = g0; g < g0 + chunk_groups && g * w < b.len; ++g) {
      const u64 r0 = g * w;
      const u32 m = r0 + w <= b.len ? w : (u32)(b.len - r0);
      u32 k = 0;
      for (u32 i = 0; i < m; ++i)
        k |= (u32)((col[(r0 + i) * row_stride] >> sh) & 1u) << i;
      if (k)
        C::add_gen(acc, acc, table[(g << w) + k], false, true);
    }
    partial[t] = acc;
  }
};

// partial[i] += partial[i + off]
template <class C> struct PartitionFoldBody {
  static constexpr int kBlock = 64;
  typename C::Point* partial;
  u64 off;
  B200_HD void operator()(u64 i) const { C::add(partial[i], partial[i], partial[i + off]); }
};

template <class C> struct PartitionHornerBody {
  static constexpr int kBlock = 32;
  const typename C::Point* sums;  // one point per routed bit
  const PartitionOut* outs;
  typename C::Point* pts;
  B200_HD void operator()(u64 r) const {
    const PartitionOut o = outs[r];
    typename C::Point acc = sums[o.first_bit + o.bits - 1];
    for (u32 t = o.bits - 1; t-- > 0;) {
      C::dbl(acc, acc);
      C::add(acc, acc, sums[o.first_bit + t]);
    }
    pts[o.dest] = acc;
  }
};

// Threads of one accumulation launch to aim for: 132 SMs x 2048 resident threads, so that a launch
// covers the GPU for about one wave even when few bits are routed.
constexpr u64 kPartitionTargetThreads = 1ull << 18;

// outputs `routed` of `cols` (n > 0, scalars as in the engine's ColumnDesc) from the partition table
// of width w at `table` -> pts[routed[r]]
template <class C>
inline void partition_msm(stream_t s, const typename C::Gen* table, u32 w,
                          const std::vector<ColumnDesc>& cols, const std::vector<u32>& routed,
                          typename C::Point* pts) {
  typedef typename C::Point Point;
  if (routed.empty())
    return;
  std::vector<PartitionBit> bits;
  std::vector<PartitionOut> outs;
  u64 max_len = 0;
  for (u32 j : routed) {
    const ColumnDesc& col = cols[j];
    outs.push_back({j, (u32)bits.size(), col.bit_width});
    for (u32 t = 0; t < col.bit_width; ++t)
      bits.push_back({col.bit_offset + t, col.n});
    max_len = std::max<u64>(max_len, col.n);
  }
  const u64 nbits = bits.size(), groups = (max_len + w - 1) / w;
  u64 chunks = std::min<u64>(groups, std::max<u64>(1, kPartitionTargetThreads / nbits));
  const u64 chunk_groups = (groups + chunks - 1) / chunks;
  chunks = (groups + chunk_groups - 1) / chunk_groups;
  const size_t bits_bytes = nbits * sizeof(PartitionBit);
  std::vector<unsigned char> block(bits_bytes + outs.size() * sizeof(PartitionOut));
  std::memcpy(block.data(), bits.data(), bits_bytes);
  std::memcpy(block.data() + bits_bytes, outs.data(), outs.size() * sizeof(PartitionOut));
  unsigned char* staged = (unsigned char*)stage_to_device(s, block.data(), block.size());
  Point* partial = (Point*)dev_alloc(chunks * nbits * sizeof(Point), s);
  launch(PartitionAccumulateBody<C>{table, cols[routed[0]].base, cols[routed[0]].row_stride,
                                    (const PartitionBit*)staged, partial, (u32)nbits, w,
                                    (u32)chunk_groups},
         chunks * nbits, s);
  for (u64 m = chunks; m > 1;) {
    const u64 h = (m + 1) / 2;
    launch(PartitionFoldBody<C>{partial, h * nbits}, (m - h) * nbits, s);
    m = h;
  }
  launch(PartitionHornerBody<C>{partial, (const PartitionOut*)(staged + bits_bytes), pts},
         outs.size(), s);
  dev_free(partial, s);
  dev_free(staged, s);
}

}  // namespace b200
