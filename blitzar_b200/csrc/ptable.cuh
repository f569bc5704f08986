// The reference's partition table, built on the device: for every group g of w consecutive
// generators, the 2^w subset sums T[g][k] = sum over the set bits j of k of G[g w + j], as compact
// ABI elements in natural k order (the entry layout of the reference's handle files,
// in_memory_partition_table_accessor.h:98-105; generators past n pad the last group with the
// identity, in_memory_partition_table_accessor_utility.h:45-57).
//
// Replaces the CPU-serial mtxpp2::compute_partition_table_slice (sxt/multiexp/pippenger2/
// partition_table.h:30-75) and its one field inversion per entry in the compact conversion
// (sxt/curve21/type/element_p3.cc:33-41, sxt/curve_bng1/type/element_p2.cc:52-64):
//   rounds j = 0 .. w-1: entries [2^j, 2^(j+1)) of every group are entries [0, 2^j) + G_j — one
//       complete mixed addition per entry, every entry of a round independent (PartitionRoundBody);
//   the projective denominators of the whole chunk are inverted at once by Montgomery's trick over
//       the inversion tree of batch_affine.cuh (denominator 1 for Z = 0, the Weierstrass identity);
//   PartitionStoreBody writes the affine coordinates (ed25519: also T = x y) in the compact layout,
//       the identity encoding for Z = 0.
// PartitionGenStoreBody writes the same entries in the curve's device generator layout (C::Gen, Z = 1)
// instead, for a table kept on a handle and read by partition_msm.cuh.
// The caller splits a table into chunks of whole groups; the scratch lives for one chunk only.
#pragma once
#include <type_traits>

#include "batch_affine.cuh"

namespace b200 {

template <class C> struct PartitionRoundBody {
  static constexpr int kBlock = 128;
  const typename C::Gen* gens;
  typename C::Point* pts;   // the chunk's groups x 2^w entries
  typename C::F::E* den;    // their projective denominators
  u64 n;                    // generators; indices >= n are the identity padding
  u64 first_group;          // group of the chunk's first entry
  u32 w, j;                 // window width, round
  B200_HD void operator()(u64 t) const {
    const u64 g = t >> j, src = (g << w) + (t & ((1ull << j) - 1)), dst = src + (1ull << j);
    typename C::Point p;
    if (j == 0) {
      p = C::identity();
      pts[src] = p;
      den[src] = C::denominator(p);
    } else {
      p = pts[src];
    }
    const u64 gi = (first_group + g) * w + j;
    if (gi < n)
      C::add_gen(p, p, gens[gi], false);
    pts[dst] = p;
    den[dst] = C::denominator(p);
  }
};

template <class C> struct PartitionStoreBody {
  static constexpr int kBlock = 128;
  const typename C::Point* pts;
  const typename C::F::E* zinv;  // inverted denominators
  unsigned char* out;
  B200_HD void operator()(u64 i) const {
    C::store_compact_abi(out + i * C::kAbiCompactBytes, pts[i], zinv[i]);
  }
};

template <class C> struct PartitionGenStoreBody {
  static constexpr int kBlock = 128;
  const typename C::Point* pts;
  const typename C::F::E* zinv;  // inverted denominators
  typename C::Gen* out;
  B200_HD void operator()(u64 i) const { C::normalized_gen(out[i], pts[i], zinv[i]); }
};

// groups [first_group, first_group + groups) of the partition table of width w over n generators
// (device generator layout) -> compact ABI entries (Out = unsigned char) or normalised device
// generators (Out = C::Gen) at `out`
template <class C, class Out>
inline void build_partition_table(stream_t s, const typename C::Gen* gens, u64 n, u32 w,
                                  u64 first_group, u64 groups, Out* out) {
  typedef typename C::Point Point;
  typedef typename C::F::E E;
  const u64 entries = groups << w;
  if (entries == 0)
    return;
  Point* pts = (Point*)dev_alloc(entries * sizeof(Point), s);
  E* den = (E*)dev_alloc(entries * sizeof(E), s);
  for (u32 j = 0; j < w; ++j)
    launch(PartitionRoundBody<C>{gens, pts, den, n, first_group, w, j}, groups << j, s);
  batch_invert<typename C::F>(s, den, entries);
  if constexpr (std::is_same<Out, unsigned char>::value)
    launch(PartitionStoreBody<C>{pts, den, out}, entries, s);
  else
    launch(PartitionGenStoreBody<C>{pts, den, out}, entries, s);
  dev_free(den, s);
  dev_free(pts, s);
}

}  // namespace b200
