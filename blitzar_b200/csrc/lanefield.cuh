// Warp-cooperative ("lane-sliced") arithmetic in GF(2^255 - 19) for the latency-bound tail of an MSM.
//
// The tail kernels (240 Horner doublings over the window sums, the 250-squaring inverse square root
// of the ristretto encoding) are ONE dependent chain per output: a single warp cannot issue a
// 256-bit multiplication faster than its SM sub-partition's multiplier pipe allows (72 IMAD.WIDE at
// ~5.6 cycles each, tests/micro/latency.cu), however few lanes do useful work. Here one field
// element is spread over 10 lanes in the unsaturated radix 2^25.5 (limb i at bit ceil(25.5 i): 26, 25,
// 26, ... bits, so that 2^255 = 19 closes the ring exactly): lane 10g + m of the warp holds limb m of
// the element of group g. A multiplication is then 10 multiply-adds per lane — column m of the
// product, the operands fetched with warp shuffles, wrapped terms times 19, odd-odd terms doubled —
// and the carries travel ACROSS lanes by two shuffle rounds; the spare bits of the radix absorb what
// is left, so additions and subtractions are single instructions without any carry propagation.
// Three elements (groups) are processed per warp: X, Y, Z of a point in the doubling chain.
//
// (A first version kept the saturated 8 x 32-bit limbs of field.cuh across 8 lanes and resolved
// the carries exactly with a ballot-based carry-lookahead; its dependent chain — two ballots and
// two resolutions per operation — made it no faster than the quad-lane schedule for the C2 Horner
// kernel.)
//
// Replaces, for these chains, the per-thread schedules of field.cuh (which replace
// sxt/field51/operation/{mul,sq}.cc). Device only: the CPU emulation harness keeps the scalar path.
#pragma once
#include "curve.cuh"

#if defined(__CUDACC__) && !defined(B200_EMULATE)
namespace b200 {
namespace lane10 {

#define B200_DEV __device__ __forceinline__
constexpr unsigned kFull = 0xffffffffu;

struct Lane {
  u32 base;   // first lane of this lane's group
  u32 m;      // limb index 0..9 (lanes 30, 31 form an idle fourth "group")
  u32 bits;   // 26 for even limbs, 25 for odd ones
  u32 mask;
  u32 prev;   // lane holding limb m - 1 (limb 9 for m = 0)
  u32 twop;   // limb m of 2p
};
B200_DEV Lane lane_info() {
  Lane L;
  const u32 lane = threadIdx.x & 31u;
  const u32 g = lane / 10u;
  L.base = 10u * g;
  L.m = lane - L.base;
  L.bits = (L.m & 1u) ? 25u : 26u;
  L.mask = (1u << L.bits) - 1u;
  L.prev = L.base + (L.m == 0 ? 9u : L.m - 1u);
  L.twop = L.m == 0 ? 0x7ffffdau : ((L.m & 1u) ? 0x3fffffeu : 0x7fffffeu);
  return L;
}

// one carry round: every limb keeps its low bits and hands the rest to the next limb (limb 9 wraps to
// limb 0 times 19). Inputs up to 2^32 - 1 come out below 2^26 + 2^12 (even) / 2^25 + 2^12 (odd).
B200_DEV u32 carry1(const Lane& L, u32 v) {
  u32 c = __shfl_sync(kFull, v >> L.bits, L.prev);
  c = L.m == 0 ? c * 19u : c;
  return (v & L.mask) + c;
}
B200_DEV u32 add(u32 a, u32 b) { return a + b; }                                  // lazy
B200_DEV u32 sub2p(const Lane& L, u32 a, u32 b) { return a + L.twop - b; }        // lazy, b reduced
// lazy; b < 2^27.9 on even limbs, one bit less on odd ones (4p limb-wise: 2^28 - 76, 2^28 - 4 and 2^27 - 4)
B200_DEV u32 sub4p(const Lane& L, u32 a, u32 b) { return a + 2u * L.twop - b; }

// limb m of a * b mod p. Operand bounds: a, b < 2^27.7 on even limbs, one bit less on odd ones
// (19 b and 2 a must fit 32 bits, ten products 64); result below 2^26 + 2^22 (2^25 + 2^22).
B200_DEV u32 mul(const Lane& L, u32 a, u32 b) {
  u64 acc = 0;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    u32 ai = __shfl_sync(kFull, a, L.base + (u32)i);
    const bool wrap = (u32)i > L.m;                       // a_i b_(m - i + 10) carries 2^255 = 19
    const u32 j = wrap ? L.m + 10u - (u32)i : L.m - (u32)i;
    u32 bj = __shfl_sync(kFull, b, L.base + j);
    bj = wrap ? bj * 19u : bj;
    if (i & 1)                                            // both limbs odd: their positions add up
      ai = (L.m & 1u) ? ai : 2u * ai;                     // one bit higher (j odd <=> m even here)
    acc += (u64)ai * bj;
  }
  // two carry rounds across the lanes; the first moves up to 38 bits
  const u64 c = acc >> L.bits;
  const u32 clo = __shfl_sync(kFull, (u32)c, L.prev), chi = __shfl_sync(kFull, (u32)(c >> 32), L.prev);
  u64 cin = ((u64)chi << 32) | clo;
  cin = L.m == 0 ? cin * 19u : cin;
  const u64 v = (acc & L.mask) + cin;                    // < 2^43
  u32 c2 = __shfl_sync(kFull, (u32)(v >> L.bits), L.prev);  // < 2^18
  c2 = L.m == 0 ? c2 * 19u : c2;
  return ((u32)v & L.mask) + c2;
}

// replicated element (8 x 32-bit limbs in every lane, any representative below 2^256) -> this
// lane's radix-2^25.5 limb. Limb 9 keeps bits 230..255 (one bit of slack is used).
B200_DEV u32 slice(const Lane& L, const F25519::E& e) {
  const u32 pos = (51u * L.m + 1u) >> 1, w = pos >> 5, sh = pos & 31u;
  u32 lo = e.l[0], hi = e.l[1];
#pragma unroll
  for (int k = 1; k < 8; ++k) {
    lo = w == (u32)k ? e.l[k] : lo;
    hi = w == (u32)k ? (k < 7 ? e.l[k < 7 ? k + 1 : 7] : 0u) : hi;
  }
  const u32 x = (u32)((((u64)hi << 32) | lo) >> sh);
  return L.m == 9 ? x : (x & L.mask);
}
// lane-sliced element of group g -> replicated 8 x 32-bit limbs in every lane of the warp
B200_DEV void gather(F25519::E& e, u32 v, u32 g) {
  u64 acc[5] = {0, 0, 0, 0, 0};  // 320 bits
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const u64 limb = __shfl_sync(kFull, v, 10u * g + (u32)k);
    const int pos = (51 * k + 1) >> 1, w = pos >> 6, sh = pos & 63;
    // limb << pos into the 64-bit words (limb < 2^32: touches at most two of them)
    const u64 lo = limb << sh, hi = sh > 32 ? (limb >> (64 - sh)) : 0;
    const u64 s = acc[w] + lo;
    acc[w + 1] += hi + (s < lo ? 1u : 0u);  // far below 2^64: limbs arrive in rising position
    acc[w] = s;
  }
  // the few bits above 2^256 fold back with 38
  u64 t = acc[0] + acc[4] * 38u;
  u64 c = t < acc[0] ? 1u : 0u;
  acc[0] = t;
#pragma unroll
  for (int k = 1; k < 4; ++k) {
    t = acc[k] + c;
    c = t < c ? 1u : 0u;
    acc[k] = t;
  }
  acc[0] += c * 38u;  // a second wrap leaves a tiny value: cannot carry
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    e.l[2 * k] = (u32)acc[k];
    e.l[2 * k + 1] = (u32)(acc[k] >> 32);
  }
}
// limb m of the element held by group g, in every group
B200_DEV u32 from_group(const Lane& L, u32 v, u32 g) { return __shfl_sync(kFull, v, 10u * g + L.m); }

B200_DEV u32 sqr_n(const Lane& L, u32 a, int n) {
  for (int i = 0; i < n; ++i)
    a = mul(L, a, a);
  return a;
}
// a^((p-5)/8) = a^(2^252 - 3), the chain of F25519::pow22523
B200_DEV u32 pow22523(const Lane& L, u32 a) {
  u32 t0 = mul(L, a, a);            // 2
  u32 t1 = sqr_n(L, t0, 2);         // 8
  t1 = mul(L, a, t1);               // 9
  t0 = mul(L, t0, t1);              // 11
  u32 t2 = mul(L, t0, t0);          // 22
  t1 = mul(L, t1, t2);              // 2^5 - 1
  t2 = sqr_n(L, t1, 5);
  t1 = mul(L, t2, t1);              // 2^10 - 1
  t2 = sqr_n(L, t1, 10);
  t2 = mul(L, t2, t1);              // 2^20 - 1
  u32 t3 = sqr_n(L, t2, 20);
  t2 = mul(L, t3, t2);              // 2^40 - 1
  t2 = sqr_n(L, t2, 10);
  t1 = mul(L, t2, t1);              // 2^50 - 1
  t2 = sqr_n(L, t1, 50);
  t2 = mul(L, t2, t1);              // 2^100 - 1
  t3 = sqr_n(L, t2, 100);
  t2 = mul(L, t3, t2);              // 2^200 - 1
  t2 = sqr_n(L, t2, 50);
  t1 = mul(L, t2, t1);              // 2^250 - 1
  t1 = sqr_n(L, t1, 2);
  return mul(L, t1, a);
}

// n >= 1 doublings of the point whose X, Y, Z sit in groups 0, 1, 2 (a doubling does not read T,
// dbl-2008-hwcd). Returns X, Y, Z of the result and its T (in every group) in t_out.
//   A = X^2, B = Y^2, ZZ = Z^2 (one round, three groups), XY (all groups),
//   G = A - B, F = G + 2 ZZ, H = A + B, E = -2 XY;   X3 = E F, Y3 = G H, Z3 = F G, T3 = E H
// — the signs of Ed25519::dbl.
B200_DEV u32 dbl_n(const Lane& L, u32 v, int n, u32& t_out) {
  const u32 g = L.base / 10u;
  u32 E = 0, H = 0;
  for (int it = 0; it < n; ++it) {
    const u32 X = from_group(L, v, 0), Y = from_group(L, v, 1);
    const u32 sq = mul(L, v, v);
    const u32 xy = mul(L, X, Y);
    const u32 A = from_group(L, sq, 0), B = from_group(L, sq, 1), ZZ = from_group(L, sq, 2);
    const u32 G = carry1(L, sub2p(L, A, B));          // < 2^26 + 2^12
    const u32 Fv = add(G, add(ZZ, ZZ));               // < 2^27.6
    H = add(A, B);                                    // < 2^27.1
    E = carry1(L, sub4p(L, 0u, add(xy, xy)));         // -2 XY, < 2^26 + 2^12
    const u32 lhs = g == 0 ? E : G;                   // the small operand first
    const u32 rhs = g == 1 ? H : Fv;
    v = mul(L, lhs, rhs);                             // g0: E F, g1: G H, g2: G F
  }
  t_out = mul(L, E, H);
  return v;
}
B200_DEV u32 slice_point(const Lane& L, const Ed25519::Point& p) {
  const u32 g = L.base / 10u;
  const u32 x = slice(L, p.X), y = slice(L, p.Y), z = slice(L, p.Z);
  return g == 0 ? x : (g == 1 ? y : z);
}
B200_DEV void gather_point(Ed25519::Point& p, u32 v, u32 t) {
  gather(p.X, v, 0);
  gather(p.Y, v, 1);
  gather(p.Z, v, 2);
  gather(p.T, t, 0);
}
#undef B200_DEV

// Self-test body (b200_selftest_lane_arithmetic): every group of 10 lanes checks the lane-sliced
// operations against the per-thread schedules of field.cuh / curve.cuh on pseudo-random and edge-case
// operands; mismatches are counted. All collectives are reached warp-uniformly.
struct SelfTestBody {
  static constexpr int kBlock = 32;
  u32 seed;
  u32* mismatches;
  static __device__ u32 rnd(u64& st) {
    st ^= st << 13;
    st ^= st >> 7;
    st ^= st << 17;
    return (u32)(st >> 16);
  }
  static __device__ bool same(const F25519::E& x, const F25519::E& y) {
    F25519::E a, b;
    F25519::canonical(a, x);
    F25519::canonical(b, y);
    bool ok = true;
    for (int i = 0; i < 8; ++i)
      ok = ok && a.l[i] == b.l[i];
    return ok;
  }
  __device__ void operator()(u64 tid) const {
    typedef F25519 F;
    const Lane L = lane_info();
    const u32 g = L.base / 10u;  // 0..2 (3 = the two idle lanes)
    const u32 gg = g < 3 ? g : 0u;
    const u32 group = (u32)(tid >> 5) * 3u + gg;
    u64 st = ((u64)seed << 32) ^ (0x9E3779B97F4A7C15ull * (group + 1));
    F::E a, b, want, got;
    for (int i = 0; i < 8; ++i) {
      a.l[i] = rnd(st);
      b.l[i] = rnd(st);
    }
    switch (group % 9) {  // edge cases: all-ones limbs, zero, p - 1, tiny, top bits
    case 1: for (int i = 0; i < 8; ++i) a.l[i] = 0xffffffffu; break;
    case 2: for (int i = 0; i < 8; ++i) a.l[i] = b.l[i] = 0xffffffffu; break;
    case 3: for (int i = 0; i < 8; ++i) b.l[i] = 0; break;
    case 4: for (int i = 0; i < 8; ++i) a.l[i] = 0xffffffffu; a.l[0] = 0xffffffecu; a.l[7] = 0x7fffffffu; break;
    case 5: for (int i = 1; i < 8; ++i) a.l[i] = 0; a.l[0] = 37; break;
    case 6: for (int i = 0; i < 7; ++i) b.l[i] = 0xffffffffu; break;
    case 7: for (int i = 0; i < 8; ++i) a.l[i] = 0; for (int i = 0; i < 8; ++i) b.l[i] = 0xffffffffu; break;
    default: break;
    }
    u32 bad = 0;
    const u32 la = slice(L, a), lb = slice(L, b);
    gather(got, la, gg);  // round trip
    bad += same(got, a) ? 0 : 1;
    gather(got, mul(L, la, lb), gg);
    F::mul(want, a, b);
    bad += same(got, want) ? 0 : 1;
    gather(got, add(la, lb), gg);
    F::add(want, a, b);
    bad += same(got, want) ? 0 : 1;
    // the subtrahend of sub2p must be a reduced element (a product), as in the kernels
    const u32 lbr = mul(L, lb, slice(L, F::one()));
    gather(got, carry1(L, sub2p(L, la, lbr)), gg);
    F::sub(want, a, b);
    bad += same(got, want) ? 0 : 1;
    {  // lazy operands into the multiplier: (a - b) (a + a), and -(2 a b)
      const u32 d = carry1(L, sub2p(L, la, lbr)), s2 = add(la, la);
      gather(got, mul(L, d, s2), gg);
      F::E d_, s_;
      F::sub(d_, a, b);
      F::add(s_, a, a);
      F::mul(want, d_, s_);
      bad += same(got, want) ? 0 : 1;
      const u32 ab = mul(L, la, lb);
      gather(got, carry1(L, sub4p(L, 0u, add(ab, ab))), gg);
      F::mul(want, a, b);
      F::add(want, want, want);
      F::neg(want, want);
      bad += same(got, want) ? 0 : 1;
    }
    if ((tid >> 5) % 4 == 0) {  // the long chain, on a quarter of the warps (warp-uniform)
      gather(got, pow22523(L, la), gg);
      F::pow22523(want, a);
      bad += same(got, want) ? 0 : 1;
    }
    // point doubling: the whole warp holds ONE point (a built-in generator)
    Ed25519::Point p, q, r;
    Ed25519::builtin_generator(p, (u64)seed * 1000u + (tid >> 5));
    q = p;
    for (int i = 0; i < 5; ++i)
      Ed25519::dbl(q, q);
    u32 t;
    const u32 v = dbl_n(L, slice_point(L, p), 5, t);
    gather_point(r, v, t);
    bad += (same(r.X, q.X) && same(r.Y, q.Y) && same(r.Z, q.Z) && same(r.T, q.T)) ? 0 : 1;
    if (bad && L.m == 0 && g < 3)
      atomicAdd(mismatches, bad);
  }
};

}  // namespace lane10
}  // namespace b200
#endif
