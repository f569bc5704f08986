// Group law for the curves of the MSM hot path, as device functions over field.cuh.
//
// Replaces (re-derived): sxt/curve21 (+ sxt/ristretto compress / elligator), sxt/curve_g1,
// sxt/curve_bng1, sxt/curve_gk — the `add / double / neg / identity` concept of
// sxt/base/curve/element.h:26-35 — and the canonicalisation done on the host by the reference
// (rsto::batch_compress, cg1o::batch_compress, batch_to_element_affine; SURVEY §8 a14).
//
// Each curve is a traits struct:
//   Point   bucket accumulator (extended / homogeneous projective coordinates)
//   Gen     ingested generator as kept in HBM for the gather (ed25519: extended; Weierstrass:
//           affine Montgomery x,y with (0,0) standing for the point at infinity)
// Formulas: ed25519 unified extended addition (Hisil-Wong-Carter-Dawson 2008, complete for a=-1,
// d non-square); short Weierstrass a=0 complete formulas (Renes-Costello-Batina 2016, Alg. 7/8/9).
#pragma once
#include "field.cuh"

namespace b200 {

enum CurveId : unsigned {
  kRistretto255 = 0,
  kBls12381 = 1,
  kBn254 = 2,
  kGrumpkin = 3,
  kBls12381G2 = 4,  // no counterpart in the reference, which defines ids 0-3
  kBn254G2 = 5,     // nor this one
};

// ---- execution policies for the independent field multiplications inside a point operation -------
// SeqExec : one thread computes every product (throughput-bound kernels).
// QuadExec: four adjacent lanes hold identical operands; each lane computes one product of a batch
//           and the results are broadcast with warp shuffles, so a point operation costs 2-4
//           multiplication latencies instead of 8-12 (latency-bound tail kernels). All four lanes
//           execute the same instruction stream on lane-selected operands (no divergence). On the
//           host (emulation) both policies compute every product.
struct SeqExec {
  static constexpr int kLanes = 1;
  template <class F>
  static B200_HD void mul4(typename F::E& o0, typename F::E& o1, typename F::E& o2,
                           typename F::E& o3, const typename F::E& a0, const typename F::E& b0,
                           const typename F::E& a1, const typename F::E& b1,
                           const typename F::E& a2, const typename F::E& b2,
                           const typename F::E& a3, const typename F::E& b3) {
    F::mul(o0, a0, b0);
    F::mul(o1, a1, b1);
    F::mul(o2, a2, b2);
    F::mul(o3, a3, b3);
  }
  template <class F>
  static B200_HD void mul2(typename F::E& o0, typename F::E& o1, const typename F::E& a0,
                           const typename F::E& b0, const typename F::E& a1,
                           const typename F::E& b1) {
    F::mul(o0, a0, b0);
    F::mul(o1, a1, b1);
  }
};
// kFullMask = true: shuffles name the whole warp (fast path; every non-exited lane of the warp must
// reach the call convergently). kFullMask = false: shuffles name only the quad (safe when quads of
// one warp diverge, but a run-time partial mask costs tens of cycles per shuffle).
template <bool kFullMask> struct QuadExecT {
  static constexpr int kLanes = 4;
  template <class F>
  static B200_HD void mul4(typename F::E& o0, typename F::E& o1, typename F::E& o2,
                           typename F::E& o3, const typename F::E& a0, const typename F::E& b0,
                           const typename F::E& a1, const typename F::E& b1,
                           const typename F::E& a2, const typename F::E& b2,
                           const typename F::E& a3, const typename F::E& b3) {
#ifdef __CUDA_ARCH__
    const unsigned lane = threadIdx.x & 3u;
    const unsigned mask = kFullMask ? 0xffffffffu : (0xFu << (threadIdx.x & 28u));
    typename F::E x, y, r;
    // mask-and-or operand selection: guaranteed branch-free (ternaries compile to divergent code)
    const u32 m0 = lane == 0 ? ~0u : 0u, m1 = lane == 1 ? ~0u : 0u, m2 = lane == 2 ? ~0u : 0u,
              m3 = lane == 3 ? ~0u : 0u;
#pragma unroll
    for (int k = 0; k < F::N; ++k) {
      x.l[k] = (a0.l[k] & m0) | (a1.l[k] & m1) | (a2.l[k] & m2) | (a3.l[k] & m3);
      y.l[k] = (b0.l[k] & m0) | (b1.l[k] & m1) | (b2.l[k] & m2) | (b3.l[k] & m3);
    }
    F::mul(r, x, y);
#pragma unroll
    for (int k = 0; k < F::N; ++k) {
      o0.l[k] = __shfl_sync(mask, r.l[k], 0, 4);
      o1.l[k] = __shfl_sync(mask, r.l[k], 1, 4);
      o2.l[k] = __shfl_sync(mask, r.l[k], 2, 4);
      o3.l[k] = __shfl_sync(mask, r.l[k], 3, 4);
    }
#else
    SeqExec::mul4<F>(o0, o1, o2, o3, a0, b0, a1, b1, a2, b2, a3, b3);
#endif
  }
  template <class F>
  static B200_HD void mul2(typename F::E& o0, typename F::E& o1, const typename F::E& a0,
                           const typename F::E& b0, const typename F::E& a1,
                           const typename F::E& b1) {
#ifdef __CUDA_ARCH__
    const unsigned lane = threadIdx.x & 1u;
    const unsigned mask = kFullMask ? 0xffffffffu : (0xFu << (threadIdx.x & 28u));
    typename F::E x, y, r;
    const u32 m1 = lane ? ~0u : 0u, m0 = ~m1;
#pragma unroll
    for (int k = 0; k < F::N; ++k) {
      x.l[k] = (a0.l[k] & m0) | (a1.l[k] & m1);
      y.l[k] = (b0.l[k] & m0) | (b1.l[k] & m1);
    }
    F::mul(r, x, y);
#pragma unroll
    for (int k = 0; k < F::N; ++k) {
      o0.l[k] = __shfl_sync(mask, r.l[k], 0, 4);
      o1.l[k] = __shfl_sync(mask, r.l[k], 1, 4);
    }
#else
    SeqExec::mul2<F>(o0, o1, a0, b0, a1, b1);
#endif
  }
};
typedef QuadExecT<false> QuadExec;
typedef QuadExecT<true> QuadExecConv;

// ================================================================================================
// ed25519 / ristretto255
// ================================================================================================
struct Ed25519 {
  typedef F25519 F;
  typedef F::E fe;
  static constexpr unsigned kCurveId = kRistretto255;
  static constexpr int kAbiGenBytes = 160;     // sxt_ristretto255 (commit generators)
  static constexpr int kAbiProjBytes = 160;    // sxt_ristretto255 (handle generators, fixed res)
  static constexpr int kAbiCommitBytes = 32;   // sxt_ristretto255_compressed
  static constexpr int kScalarBitsHint = 253;
  static constexpr bool kBatchAffine = false;  // extended coordinates: 8M per addition already

  struct Point {
    fe X, Y, Z, T;
  };
  // generator as kept in HBM: "cached" form (Y+X, Y-X, 2Z, 2dT) so that a bucket add costs 8
  // field multiplications (the 2d*T product is paid once per generator at ingestion)
  struct Gen {
    fe YpX, YmX, Z2, T2d;
  };

  static B200_HD Point identity() {
    Point p;
    p.X = F::zero();
    p.Y = F::one();
    p.Z = F::one();
    p.T = F::zero();
    return p;
  }
  static B200_HD void neg(Point& r, const Point& a) {
    F::neg(r.X, a.X);
    r.Y = a.Y;
    r.Z = a.Z;
    F::neg(r.T, a.T);
  }
  // r = a + b (unified; valid for doubling and identity operands); 4 + 1 + 4 multiplications
  template <class X = SeqExec> static B200_HD void add(Point& r, const Point& a, const Point& b) {
    fe A, B, C, D, E, Fv, G, H, t0, t1, t2, t3;
    F::sub(t0, a.Y, a.X);
    F::sub(t1, b.Y, b.X);
    F::add(t2, a.Y, a.X);
    F::add(t3, b.Y, b.X);
    X::template mul4<F>(A, B, C, D, t0, t1, t2, t3, a.T, b.T, a.Z, b.Z);
    F::mul(C, C, F::constant([](int i) { return F25_D2(i); }));
    F::dbl(D, D);
    F::sub(E, B, A);
    F::sub(Fv, D, C);
    F::add(G, D, C);
    F::add(H, B, A);
    Point o;
    X::template mul4<F>(o.X, o.Y, o.T, o.Z, E, Fv, G, H, E, H, Fv, G);
    r = o;
  }
  // coordinates are stored canonical (< p)
  static B200_HD void point_to_gen(Gen& g, const Point& p) {
    F::add(g.YpX, p.Y, p.X);
    F::sub(g.YmX, p.Y, p.X);
    F::dbl(g.Z2, p.Z);
    F::mul(g.T2d, p.T, F::constant([](int i) { return F25_D2(i); }));
    F::canonical(g.YpX, g.YpX);
    F::canonical(g.YmX, g.YmX);
    F::canonical(g.Z2, g.Z2);
    F::canonical(g.T2d, g.T2d);
  }

  // projective denominator of a point / generator form of the affine point (X zi, Y zi)
  static B200_HD fe denominator(const Point& p) { return p.Z; }
  static B200_HD void normalized_gen(Gen& g, const Point& p, const fe& zi) {
    Point a;
    F::mul(a.X, p.X, zi);
    F::mul(a.Y, p.Y, zi);
    a.Z = F::one();
    F::mul(a.T, a.X, a.Y);
    point_to_gen(g, a);
  }
  // (2X : 2Y : 2Z : 2T) — the same point; one multiplication by the constant 1/d
  static B200_HD void gen_to_point(Point& r, const Gen& g, bool negate) {
    fe x2, t2, nx, nt;
    F::sub(x2, g.YpX, g.YmX);
    F::add(r.Y, g.YpX, g.YmX);
    r.Z = g.Z2;
    F::mul(t2, g.T2d, F::constant([](int i) { return F25_INVD(i); }));
    F::neg(nx, x2);
    F::neg(nt, t2);
    F::select(r.X, x2, nx, negate);
    F::select(r.T, t2, nt, negate);
  }
  // r = a +/- g in 8 multiplications; branch-free in `negate` (-g swaps Y+X / Y-X and negates 2dT)
  // so the lanes of a warp add generators of either sign in one pass
  // unit_z: the generator is normalised (Z = 1, so 2Z = 2 — every entry of a fixed-base table): the
  // product Z1 * 2Z2 becomes a doubling, 7 multiplications instead of 8
  template <class X = SeqExec>
  static B200_HD void add_gen(Point& r, const Point& a, const Gen& g, bool negate,
                              bool unit_z = false) {
    // -g negates C = T1 2dT2, which swaps D - C and D + C: selected after the sums rather than
    // negating 2dT2 before the product
    fe A, B, C, D, E, Fv, G, H, t0, t1, qp, qm, dmc, dpc;
    F::select(qp, g.YpX, g.YmX, negate);
    F::select(qm, g.YmX, g.YpX, negate);
    F::sub(t0, a.Y, a.X);
    F::add(t1, a.Y, a.X);
    if (unit_z) {
      F::mul(A, t0, qm);
      F::mul(B, t1, qp);
      F::mul(C, a.T, g.T2d);
      F::dbl(D, a.Z);
    } else {
      X::template mul4<F>(A, B, C, D, t0, qm, t1, qp, a.T, g.T2d, a.Z, g.Z2);
    }
    F::sub(E, B, A);
    F::sub(dmc, D, C);
    F::add(dpc, D, C);
    F::select(Fv, dmc, dpc, negate);
    F::select(G, dpc, dmc, negate);
    F::add(H, B, A);
    Point o;
    X::template mul4<F>(o.X, o.Y, o.T, o.Z, E, Fv, G, H, E, H, Fv, G);
    r = o;
  }
  template <class X = SeqExec> static B200_HD void dbl(Point& r, const Point& a) {
    fe A, B, C, E, Fv, G, H, t0, t1;
    F::add(t0, a.X, a.Y);
    X::template mul4<F>(A, B, C, t1, a.X, a.X, a.Y, a.Y, a.Z, a.Z, t0, t0);
    F::dbl(C, C);
    F::add(H, A, B);
    F::sub(E, H, t1);
    F::sub(G, A, B);
    F::add(Fv, C, G);
    Point o;
    X::template mul4<F>(o.X, o.Y, o.T, o.Z, E, Fv, G, H, E, H, Fv, G);
    r = o;
  }

  // a normalised generator (Z = 1) without a load of its Z2 field, which is the constant 2
  static B200_HD Gen load_unit_gen(const Gen* src) {
    Gen g;
    g.YpX = src->YpX;
    g.YmX = src->YmX;
    g.T2d = src->T2d;
    g.Z2 = F::zero();
    g.Z2.l[0] = 2;
    return g;
  }

  // sxt_ristretto255 { u64 X[5], Y[5], Z[5], T[5] }
  static B200_HD void load_point_abi(Point& p, const void* src) {
    const u64* s = (const u64*)src;
    F::from_radix51(p.X, s);
    F::from_radix51(p.Y, s + 5);
    F::from_radix51(p.Z, s + 10);
    F::from_radix51(p.T, s + 15);
  }
  static B200_HD fe load_abi_z(const void* src) {
    fe z;
    F::from_radix51(z, (const u64*)src + 10);
    return z;
  }
  static B200_HD void load_gen_abi(Gen& g, const void* src) {
    Point p;
    load_point_abi(p, src);
    point_to_gen(g, p);
  }
  static B200_HD void load_proj_abi(Gen& g, const void* src) { load_gen_abi(g, src); }
  // c21t::compact_element {X, Y, T = XY} with Z = 1 (sxt/curve21/type/compact_element.h:30-38),
  // the entry type of the reference's partition-table files
  static constexpr int kAbiCompactBytes = 120;
  static B200_HD void load_compact_abi(Gen& g, const void* src) {
    const u64* s = (const u64*)src;
    Point p;
    F::from_radix51(p.X, s);
    F::from_radix51(p.Y, s + 5);
    p.Z = F::one();
    F::from_radix51(p.T, s + 10);
    point_to_gen(g, p);
  }
  // the inverse of load_compact_abi for the point p with zi = 1 / Z: canonical radix-2^51 limbs
  // (each < 2^51, value < p) of x = X zi, y = Y zi and T = x y
  static B200_HD void store_compact_abi(void* dst, const Point& p, const fe& zi) {
    u64* d = (u64*)dst;
    fe x, y, t;
    F::mul(x, p.X, zi);
    F::mul(y, p.Y, zi);
    F::mul(t, x, y);
    F::to_radix51(d, x);
    F::to_radix51(d + 5, y);
    F::to_radix51(d + 10, t);
  }
  static B200_HD void store_proj_abi(void* dst, const Point& p) {
    u64* d = (u64*)dst;
    F::to_radix51(d, p.X);
    F::to_radix51(d + 5, p.Y);
    F::to_radix51(d + 10, p.Z);
    F::to_radix51(d + 15, p.T);
  }

  // x = sqrt(u/v) helper of RFC 9496 §4.2 (SQRT_RATIO_M1); same contract as
  // rstb::compute_sqrt_ratio_m1 (sxt/ristretto/base/sqrt_ratio_m1.cc:33-67).
  struct ScalarPow {  // the per-thread chain; LanePow (lanefield.cuh) spreads it over 8 lanes
    static B200_HD void pow22523(fe& r, const fe& a) { F::pow22523(r, a); }
  };
  template <class Pow = ScalarPow> static B200_HD int sqrt_ratio_m1(fe& x, const fe& u, const fe& v) {
    fe v3, vxx, t, chk;
    const fe sqrtm1 = F::constant([](int i) { return F25_SQRTM1(i); });
    F::sqr(v3, v);
    F::mul(v3, v3, v);
    F::sqr(x, v3);
    F::mul(x, x, u);
    F::mul(x, x, v);  // u v^7
    Pow::pow22523(x, x);
    F::mul(x, x, v3);
    F::mul(x, x, u);  // u v^3 (u v^7)^((p-5)/8)
    F::sqr(vxx, x);
    F::mul(vxx, vxx, v);
    F::sub(chk, vxx, u);
    int has_m_root = F::is_zero(chk);
    F::add(chk, vxx, u);
    int has_p_root = F::is_zero(chk);
    F::mul(t, u, sqrtm1);
    F::add(chk, vxx, t);
    int has_f_root = F::is_zero(chk);
    fe xs;
    F::mul(xs, x, sqrtm1);
    F::select(x, x, xs, (has_p_root | has_f_root) != 0);
    F::abs(x, x);
    return has_m_root | has_p_root;
  }

  // ristretto255 encoding (RFC 9496 §4.3.2); same result as rstb::to_bytes
  // (sxt/ristretto/base/byte_conversion.cc:74-129).
  static B200_HD void store_commit_abi(void* dst, const Point& p) {
    encode<ScalarPow>((unsigned char*)dst, p);
  }
  template <class Pow> static B200_HD void encode(unsigned char* dst, const Point& p) {
    fe u1, u2, zmy, u1u2u2, inv_sqrt, den1, den2, z_inv, ix, iy, eden, t_z_inv, x_, y_, den_inv,
        x_z_inv, s_, ny;
    const fe one = F::one();
    const fe sqrtm1 = F::constant([](int i) { return F25_SQRTM1(i); });
    F::add(u1, p.Z, p.Y);
    F::sub(zmy, p.Z, p.Y);
    F::mul(u1, u1, zmy);
    F::mul(u2, p.X, p.Y);
    F::sqr(u1u2u2, u2);
    F::mul(u1u2u2, u1, u1u2u2);
    (void)sqrt_ratio_m1<Pow>(inv_sqrt, one, u1u2u2);
    F::mul(den1, inv_sqrt, u1);
    F::mul(den2, inv_sqrt, u2);
    F::mul(z_inv, den1, den2);
    F::mul(z_inv, z_inv, p.T);
    F::mul(ix, p.X, sqrtm1);
    F::mul(iy, p.Y, sqrtm1);
    F::mul(eden, den1, F::constant([](int i) { return F25_INVSQRTAMD(i); }));
    F::mul(t_z_inv, p.T, z_inv);
    bool rotate = F::is_negative(t_z_inv);
    F::select(x_, p.X, iy, rotate);
    F::select(y_, p.Y, ix, rotate);
    F::select(den_inv, den2, eden, rotate);
    F::mul(x_z_inv, x_, z_inv);
    F::neg(ny, y_);
    F::select(y_, y_, ny, F::is_negative(x_z_inv));
    F::sub(s_, p.Z, y_);
    F::mul(s_, den_inv, s_);
    F::abs(s_, s_);
    F::to_bytes(dst, s_);
  }

  // ristretto255 decoding (RFC 9496 §4.3.1); same contract as rstb::from_bytes
  // (sxt/ristretto/base/byte_conversion.cc:135-). Returns false for a non-canonical / invalid
  // encoding (p is then unspecified).
  static B200_HD bool decode(Point& p, const unsigned char* bytes) {
    fe s, ss, u1, u2, u2sq, v, t, inv_sqrt, den_x, den_y, chk;
    const fe one = F::one();
    F::from_bytes(s, bytes);
    // canonical (re-encoding reproduces the bytes, top bit clear) and non-negative
    unsigned char back[32];
    F::to_bytes(back, s);
    bool canonical = true;
    for (int i = 0; i < 32; ++i)
      canonical = canonical && (back[i] == bytes[i]);
    if (!canonical || (bytes[0] & 1))
      return false;
    F::sqr(ss, s);
    F::sub(u1, one, ss);
    F::add(u2, one, ss);
    F::sqr(u2sq, u2);
    F::sqr(t, u1);
    F::mul(t, t, F::constant([](int i) { return F25_D(i); }));
    F::neg(v, t);
    F::sub(v, v, u2sq);
    F::mul(t, v, u2sq);
    int was_square = sqrt_ratio_m1(inv_sqrt, one, t);
    F::mul(den_x, inv_sqrt, u2);
    F::mul(den_y, inv_sqrt, den_x);
    F::mul(den_y, den_y, v);
    F::mul(p.X, s, den_x);
    F::dbl(p.X, p.X);
    F::abs(p.X, p.X);
    F::mul(p.Y, u1, den_y);
    p.Z = one;
    F::mul(p.T, p.X, p.Y);
    chk = p.Y;
    return was_square && !F::is_negative(p.T) && !F::is_zero(chk);
  }

  // ristretto255 one-way map half (RFC 9496 §4.3.4 MAP); same as rstb::apply_elligator
  // (sxt/ristretto/base/elligator.cc:47-93).
  static B200_HD void elligator(Point& p, const fe& t) {
    fe r, u, c, rpd, v, s, s_prime, n, w0, w1, w2, w3, ss;
    const fe one = F::one();
    const fe d = F::constant([](int i) { return F25_D(i); });
    F::sqr(r, t);
    F::mul(r, F::constant([](int i) { return F25_SQRTM1(i); }), r);
    F::add(u, r, one);
    F::mul(u, u, F::constant([](int i) { return F25_ONEMSQD(i); }));
    F::neg(c, one);
    F::add(rpd, r, d);
    F::mul(v, r, d);
    F::sub(v, c, v);
    F::mul(v, v, rpd);
    int wasnt_square = 1 - sqrt_ratio_m1(s, u, v);
    F::mul(s_prime, s, t);
    F::abs(s_prime, s_prime);
    F::neg(s_prime, s_prime);
    F::select(s, s, s_prime, wasnt_square != 0);
    F::select(c, c, r, wasnt_square != 0);
    F::sub(n, r, one);
    F::mul(n, n, c);
    F::mul(n, n, F::constant([](int i) { return F25_SQDMONE(i); }));
    F::sub(n, n, v);
    F::add(w0, s, s);
    F::mul(w0, w0, v);
    F::mul(w1, n, F::constant([](int i) { return F25_SQRTADM1(i); }));
    F::sqr(ss, s);
    F::sub(w2, one, ss);
    F::add(w3, one, ss);
    F::mul(p.X, w0, w3);
    F::mul(p.Y, w2, w1);
    F::mul(p.Z, w1, w3);
    F::mul(p.T, w0, w2);
  }

  // Built-in generator g(index): xorshift128+ seeded (index+1, index+2) -> two field elements ->
  // elligator each -> add. Same derivation as sqcgn::compute_base_element
  // (sxt/seqcommit/generator/base_element.cc:30-35; base/num/fast_random_number_generator.h:27-50;
  //  ristretto/base/point_formation.cc:29-35).
  static B200_HD void builtin_generator(Point& g, u64 index) {
    u64 sa = index + 1, sb = index + 2;
    fe r[2];
    for (int k = 0; k < 2; ++k) {
      u64 w[4];
      for (int j = 0; j < 4; ++j) {
        u64 t = sa, s = sb;
        sa = s;
        t ^= t << 23;
        t ^= t >> 17;
        t ^= s ^ (s >> 26);
        sb = t;
        w[j] = t + s;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        r[k].l[2 * j] = (u32)w[j];
        r[k].l[2 * j + 1] = (u32)(w[j] >> 32);
      }
      r[k].l[7] &= 0x7fffffffu;
    }
    Point p0, p1;
    elligator(p0, r[0]);
    elligator(p1, r[1]);
    add(g, p1, p0);
  }
};

// ================================================================================================
// short Weierstrass y^2 = x^3 + b over a Montgomery field
// ================================================================================================
template <class FieldT, class CP> struct Weierstrass {
  typedef FieldT F;
  typedef typename F::E fe;
  static constexpr int N = F::N;
  static constexpr unsigned kCurveId = CP::kCurveId;
  static constexpr int kAbiGenBytes = CP::kAbiAffineStride;  // affine {X,Y,infinity} stride
  static constexpr int kAbiProjBytes = 3 * 4 * N;            // {X,Y,Z}
  static constexpr int kAbiCommitBytes = CP::kAbiCommitBytes;

  static constexpr bool kBatchAffine = true;  // batch_affine.cuh
  struct Point {
    fe X, Y, Z;
  };
  struct Gen {
    fe x, y;
  };

  static B200_HD Point identity() {
    Point p;
    p.X = F::zero();
    p.Y = F::one();
    p.Z = F::zero();
    return p;
  }
  static B200_HD bool gen_is_identity(const Gen& g) { return F::is_zero(g.y) && F::is_zero(g.x); }
  // the subgroup generator the reference derives its random test / benchmark points from
  // (curve_g1/constant/generator.h:34-66, curve_bng1/..., curve_gk/...)
  static B200_HD Gen subgroup_generator() {
    Gen g;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      g.x.l[i] = F::Params::gx(i);
      g.y.l[i] = F::Params::gy(i);
    }
    return g;
  }
  static B200_HD void neg(Point& r, const Point& a) {
    r.X = a.X;
    F::neg(r.Y, a.Y);
    r.Z = a.Z;
  }
  static B200_HD void mul_by_3b(fe& r, const fe& a) { CP::template mul_by_3b<F>(r, a); }

  // second half shared by Algorithms 7 and 8: six independent products
  template <class X>
  static B200_HD void finish_add(Point& r, const fe& t0, const fe& t1, const fe& t3, const fe& t4,
                                 const fe& y3, const fe& z3) {
    fe x3a, t2a, y3a, t1a, t0a, z3a;
    X::template mul4<F>(x3a, t2a, y3a, t1a, t4, y3, t3, t1, y3, t0, t1, z3);
    X::template mul2<F>(t0a, z3a, t0, t3, z3, t4);
    F::sub(r.X, t2a, x3a);
    F::add(r.Y, t1a, y3a);
    F::add(r.Z, z3a, t0a);
  }
  // RCB16 Algorithm 7 (a = 0), 6 + 6 independent products
  template <class X = SeqExec> static B200_HD void add(Point& r, const Point& p, const Point& q) {
    fe t0, t1, t2, t3, t4, m3, m4, m5, u0, u1, v0, v1, x3, y3, z3;
    F::add(t3, p.X, p.Y);
    F::add(t4, q.X, q.Y);
    F::add(u0, p.Y, p.Z);
    F::add(u1, q.Y, q.Z);
    F::add(v0, p.X, p.Z);
    F::add(v1, q.X, q.Z);
    X::template mul4<F>(t0, t1, t2, m3, p.X, q.X, p.Y, q.Y, p.Z, q.Z, t3, t4);
    X::template mul2<F>(m4, m5, u0, u1, v0, v1);
    F::add(t4, t0, t1);
    F::sub(t3, m3, t4);
    F::add(x3, t1, t2);
    F::sub(t4, m4, x3);
    F::add(y3, t0, t2);
    F::sub(y3, m5, y3);
    F::add(x3, t0, t0);
    F::add(t0, x3, t0);
    mul_by_3b(t2, t2);
    F::add(z3, t1, t2);
    F::sub(t1, t1, t2);
    mul_by_3b(y3, y3);
    Point o;
    finish_add<X>(o, t0, t1, t3, t4, y3, z3);
    r = o;
  }
  // RCB16 Algorithm 8 (a = 0): projective + affine; (0,0) generator = identity = no-op
  template <class X = SeqExec>
  static B200_HD void add_gen(Point& r, const Point& p, const Gen& g, bool negate,
                              bool /*unit_z: generators are always affine here*/ = false) {
    if (gen_is_identity(g)) {
      r = p;
      return;
    }
    fe qy, ny;
    F::neg(ny, g.y);
    F::select(qy, g.y, ny, negate);
    fe t0, t1, t2, t3, t4, m3, x3, y3, z3;
    F::add(t3, g.x, qy);
    F::add(t4, p.X, p.Y);
    X::template mul4<F>(t0, t1, m3, t2, p.X, g.x, p.Y, qy, t3, t4, qy, p.Z);
    F::mul(y3, g.x, p.Z);
    F::add(t4, t0, t1);
    F::sub(t3, m3, t4);
    F::add(t4, t2, p.Y);
    F::add(y3, y3, p.X);
    F::add(x3, t0, t0);
    F::add(t0, x3, t0);
    mul_by_3b(t2, p.Z);
    F::add(z3, t1, t2);
    F::sub(t1, t1, t2);
    mul_by_3b(y3, y3);
    Point o;
    finish_add<X>(o, t0, t1, t3, t4, y3, z3);
    r = o;
  }
  // projective denominator (1 for the identity, whose normalised form is the (0,0) generator)
  static B200_HD fe denominator(const Point& p) { return F::is_zero(p.Z) ? F::one() : p.Z; }
  static B200_HD void normalized_gen(Gen& g, const Point& p, const fe& zi) {
    if (F::is_zero(p.Z)) {
      g.x = F::zero();
      g.y = F::zero();
      return;
    }
    F::mul(g.x, p.X, zi);
    F::mul(g.y, p.Y, zi);
  }
  static B200_HD void gen_to_point(Point& r, const Gen& g, bool negate) {
    if (gen_is_identity(g)) {
      r = identity();
      return;
    }
    fe ny;
    F::neg(ny, g.y);
    r.X = g.x;
    F::select(r.Y, g.y, ny, negate);
    r.Z = F::one();
  }
  // RCB16 Algorithm 9 (a = 0), 4 + 4 independent products
  template <class X = SeqExec> static B200_HD void dbl(Point& r, const Point& p) {
    fe t0, t1, t2, txy, x3, y3, z3, xa, xb;
    X::template mul4<F>(t0, t1, t2, txy, p.Y, p.Y, p.Y, p.Z, p.Z, p.Z, p.X, p.Y);
    F::add(z3, t0, t0);
    F::add(z3, z3, z3);
    F::add(z3, z3, z3);
    mul_by_3b(t2, t2);
    F::add(y3, t0, t2);
    fe t22, t23;
    F::add(t22, t2, t2);
    F::add(t23, t22, t2);
    F::sub(t0, t0, t23);
    Point o;
    X::template mul4<F>(xa, o.Z, y3, xb, t2, z3, t1, z3, t0, y3, t0, txy);
    F::add(o.Y, xa, y3);
    F::add(o.X, xb, xb);
    r = o;
  }

  // affine ABI struct {u64 X[N/2]; u64 Y[N/2]; u8 infinity} (cg1t/cn1t/cgkt::element_affine)
  static B200_HD void load_gen_abi(Gen& g, const void* src) {
    const unsigned char* s = (const unsigned char*)src;
    if (s[8 * N]) {  // infinity flag
      g.x = F::zero();
      g.y = F::zero();
      return;
    }
    F::load(g.x, s);
    F::load(g.y, s + 4 * N);
  }
  // cg1t / cn1t / cgkt::compact_element {X, Y}; identity marked by an all-ones top limb of X
  // (sxt/curve_g1/type/compact_element.h:31, curve_bng1/..., curve_gk/...). Over Fp2 the top limbs are
  // those of c1, which is below p: no coordinate of any curve here has its top 64 bits all ones.
  static constexpr int kAbiCompactBytes = 8 * N;
  static B200_HD void load_compact_abi(Gen& g, const void* src) {
    const u32* s = (const u32*)src;
    if ((s[N - 1] & s[N - 2]) == 0xffffffffu) {
      g.x = F::zero();
      g.y = F::zero();
      return;
    }
    F::load(g.x, s);
    F::load(g.y, s + N);
  }
  // the inverse of load_compact_abi for the point p with zi = 1 / Z (anything when Z = 0): the
  // affine Montgomery limbs, or the identity {X = {0, .., 0, ~0}, Y = R mod p}
  // (compact_element::identity(), sxt/curve_bng1/type/compact_element.h:32-37)
  static B200_HD void store_compact_abi(void* dst, const Point& p, const fe& zi) {
    u32* d = (u32*)dst;
    fe x, y;
    if (F::is_zero(p.Z)) {
      x = F::zero();
      x.l[N - 2] = x.l[N - 1] = 0xffffffffu;
      y = F::one();
    } else {
      F::mul(x, p.X, zi);
      F::mul(y, p.Y, zi);
    }
    F::store(d, x);
    F::store(d + N, y);
  }
  // projective ABI struct {X,Y,Z} -> affine generator (one field inversion)
  static B200_HD void load_proj_abi(Gen& g, const void* src) {
    const unsigned char* s = (const unsigned char*)src;
    fe X, Y, Z, zi;
    F::load(X, s);
    F::load(Y, s + 4 * N);
    F::load(Z, s + 8 * N);
    if (F::is_zero(Z)) {
      g.x = F::zero();
      g.y = F::zero();
      return;
    }
    F::invert(zi, Z);
    F::mul(g.x, X, zi);
    F::mul(g.y, Y, zi);
  }
  static B200_HD void store_proj_abi(void* dst, const Point& p) {
    unsigned char* d = (unsigned char*)dst;
    F::store(d, p.X);
    F::store(d + 4 * N, p.Y);
    F::store(d + 8 * N, p.Z);
  }
  // projective -> affine {x, y, infinity}; identity -> {0, R, 1} (element_affine::identity())
  static B200_HD bool to_affine(fe& x, fe& y, const Point& p) {
    if (F::is_zero(p.Z)) {
      x = F::zero();
      y = F::one();
      return true;
    }
    fe zi;
    F::invert_eea(zi, p.Z);  // one dependent inversion per output: latency matters, not throughput
    F::mul(x, p.X, zi);
    F::mul(y, p.Y, zi);
    return false;
  }
  static B200_HD void store_commit_abi(void* dst, const Point& p) { CP::template store_commit<Weierstrass>(dst, p); }
};

// ---- per-curve parameters ----------------------------------------------------------------------
// affine commitment output {X, Y, infinity, 7 pad bytes (zeroed)} — cn1t/cgkt::element_affine
template <class W> B200_HD void store_affine_commit(void* dst, const typename W::Point& p) {
  typename W::fe x, y;
  bool inf = W::to_affine(x, y, p);
  unsigned char* d = (unsigned char*)dst;
  W::F::store(d, x);
  W::F::store(d + 4 * W::N, y);
  u32* tail = (u32*)(d + 8 * W::N);
  tail[0] = inf ? 1u : 0u;
  tail[1] = 0u;
}

struct BnCurveParams {
  static constexpr unsigned kCurveId = kBn254;
  static constexpr int kAbiAffineStride = 72;
  static constexpr int kAbiCommitBytes = 72;
  // 3b = 9
  template <class F> static B200_HD void mul_by_3b(typename F::E& r, const typename F::E& a) {
    typename F::E t;
    F::dbl(t, a);
    F::dbl(t, t);
    F::dbl(t, t);
    F::add(r, t, a);
  }
  template <class W> static B200_HD void store_commit(void* dst, const typename W::Point& p) {
    store_affine_commit<W>(dst, p);
  }
};
struct GkCurveParams {
  static constexpr unsigned kCurveId = kGrumpkin;
  static constexpr int kAbiAffineStride = 72;
  static constexpr int kAbiCommitBytes = 72;
  // 3b = -51 = -(32 + 16 + 2 + 1)
  template <class F> static B200_HD void mul_by_3b(typename F::E& r, const typename F::E& a) {
    typename F::E t2, t3, t16, t32;
    F::dbl(t2, a);
    F::add(t3, t2, a);
    F::dbl(t16, t2);
    F::dbl(t16, t16);
    F::dbl(t16, t16);
    F::dbl(t32, t16);
    F::add(t32, t32, t16);
    F::add(t32, t32, t3);
    F::neg(r, t32);
  }
  template <class W> static B200_HD void store_commit(void* dst, const typename W::Point& p) {
    store_affine_commit<W>(dst, p);
  }
};
struct BlsCurveParams {
  static constexpr unsigned kCurveId = kBls12381;
  static constexpr int kAbiAffineStride = 104;  // ABI quirk: reference reads 104-byte stride
  static constexpr int kAbiCommitBytes = 48;
  // 3b = 12
  template <class F> static B200_HD void mul_by_3b(typename F::E& r, const typename F::E& a) {
    typename F::E t;
    F::dbl(t, a);
    F::add(t, t, a);
    F::dbl(t, t);
    F::dbl(r, t);
  }
  // zcash-style 48-byte compressed encoding; same result as cg1o::compress
  // (sxt/curve_g1/operation/compression.cc:34-62)
  template <class W> static B200_HD void store_commit(void* dst, const typename W::Point& p) {
    typename W::fe x, y, xp;
    bool inf = W::to_affine(x, y, p);
    if (inf)
      x = W::F::zero();
    W::F::from_mont(xp, x);
    unsigned char* d = (unsigned char*)dst;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      u32 w = xp.l[11 - i];
      d[4 * i] = (unsigned char)(w >> 24);
      d[4 * i + 1] = (unsigned char)(w >> 16);
      d[4 * i + 2] = (unsigned char)(w >> 8);
      d[4 * i + 3] = (unsigned char)w;
    }
    d[0] |= 0x80;
    if (inf)
      d[0] |= 0x40;
    else if (W::F::lexicographically_largest(y))
      d[0] |= 0x20;
  }
};

// bls12-381 G2: y^2 = x^3 + 4 (1 + u) over Fp2Bls
struct Bls2CurveParams {
  static constexpr unsigned kCurveId = kBls12381G2;
  static constexpr int kAbiAffineStride = 200;  // {X[12], Y[12], u8 infinity}, padded to 8 bytes
  static constexpr int kAbiCommitBytes = 96;
  // 3b = 12 (1 + u)
  template <class F> static B200_HD void mul_by_3b(typename F::E& r, const typename F::E& a) {
    typename F::E t;
    F::mul_by_1pu(t, a);
    BlsCurveParams::mul_by_3b<F>(r, t);
  }
  // zcash-style 96-byte compressed encoding (what blst, arkworks and zkcrypto read): x.c1 then x.c0,
  // 48 bytes each, big-endian; flags in the top bits of byte 0 as for G1
  template <class W> static B200_HD void store_commit(void* dst, const typename W::Point& p) {
    typename W::fe x, y, xp;
    bool inf = W::to_affine(x, y, p);
    if (inf)
      x = W::F::zero();
    W::F::from_mont(xp, x);
    unsigned char* d = (unsigned char*)dst;
#pragma unroll
    for (int i = 0; i < 24; ++i) {  // c1 in limbs 12..23 above c0: the 768-bit value c0 + 2^384 c1
      u32 w = xp.l[23 - i];
      d[4 * i] = (unsigned char)(w >> 24);
      d[4 * i + 1] = (unsigned char)(w >> 16);
      d[4 * i + 2] = (unsigned char)(w >> 8);
      d[4 * i + 3] = (unsigned char)w;
    }
    d[0] |= 0x80;
    if (inf)
      d[0] |= 0x40;
    else if (W::F::lexicographically_largest(y))
      d[0] |= 0x20;
  }
};

// bn254 G2: y^2 = x^3 + b' over Fp2Bn, b' = 3 / (9 + u) (the twist of EIP-197)
struct Bn2CurveParams {
  static constexpr unsigned kCurveId = kBn254G2;
  static constexpr int kAbiAffineStride = 136;  // {X[8], Y[8], u8 infinity}, padded to 8 bytes
  static constexpr int kAbiCommitBytes = 136;   // the same struct: uncompressed affine Montgomery
  // 3b' has no form in additions: one Fp2 product by the constant (projective formulas only; the
  // batch-affine pair levels never use b)
  template <class F> static B200_HD void mul_by_3b(typename F::E& r, const typename F::E& a) {
    typename F::E b3;
#pragma unroll
    for (int i = 0; i < F::N; ++i)
      b3.l[i] = BN2_B3(i);
    F::mul(r, a, b3);
  }
  // {X, Y, infinity} as for bn254 G1; the identity is {0, R mod p, 1}
  template <class W> static B200_HD void store_commit(void* dst, const typename W::Point& p) {
    store_affine_commit<W>(dst, p);
  }
};

typedef Weierstrass<FBls, BlsCurveParams> Bls12381G1;
typedef Weierstrass<Fp2Bls, Bls2CurveParams> Bls12381G2;
typedef Weierstrass<FBn, BnCurveParams> Bn254G1;
typedef Weierstrass<Fp2Bn, Bn2CurveParams> Bn254G2;
typedef Weierstrass<FGk, GkCurveParams> GrumpkinG;

}  // namespace b200
