// Pairing products prod_i e(P_i, Q_i) over bls12-381 and bn254 (b200_multi_pairing), on the device.
//
// GT is the order-r subgroup of Fp12*, built as Fp6 = Fp2[v] / (v^3 - xi), Fp12 = Fp6[w] / (w^2 - v)
// over the Fp2 of the G2 curves (xi = 1 + u for bls12-381, 9 + u for bn254). An Fp12 element is
// c0 + c1 w, each an Fp6 b0 + b1 v + b2 v^2, each an Fp2; its memory layout, c0.b0 (a0, a1) first and
// c1.b2 last, is the ABI's b200_*_gt layout, so an element is stored by copying its limbs.
//
// e(P, Q) = f^((p^12 - 1) / r) with
//   bls12-381: f = conj(f_{|x|,Q}(P)), the ate Miller function, conjugated because x < 0;
//   bn254:     f = f_{6x+2,Q}(P) l_{T,pi(Q)}(P) l_{T+pi(Q),-pi^2(Q)}(P), T = [6x+2] Q, the optimal ate.
// The Miller loop keeps T on the twist in homogeneous projective coordinates and evaluates the lines
// (Costello-Lange-Naehrig doubling and addition steps) at the affine P. Those lines differ from the
// affine chord-and-tangent lines of E(Fp12) by factors in Fp2 and, on the M-type twist, by w^3; the
// final exponentiation maps every such factor to 1, so the result is the exact power above.
//
// Kernels, one launch each per call whatever the number of products (the product tree takes one
// launch per level of the longest product): ingestion (projective ABI structs -> affine P, Q and an
// identity flag), the Miller loop (one thread per run of consecutive pairs of one product, one Fp12
// accumulator squared once per bit for all of them), a segmented tree product of those accumulators,
// and the final exponentiation, which writes the GT ABI layout (one for an empty product).
#pragma once
#include <vector>

#include "field_op.cuh"

namespace b200 {

#define B200_NOINLINE __host__ __device__ __attribute__((noinline))

// ---- the two towers ------------------------------------------------------------------------------
// kXi0: xi = kXi0 + u. kMType: the twist of G2 is an M-type (bls12-381: psi(x', y') = (x' w^-2,
// y' w^-3)) rather than a D-type one (bn254: psi(x', y') = (x' w^2, y' w^3)); the line of a Miller step
// is then sparse at Fp2 positions 0, 1, 4 (c0.b0, c0.b1, c1.b1) instead of 0, 3, 4 (c0.b0, c1.b0,
// c1.b1).
struct BlsTower {
  typedef FBls B;
  typedef Fp2Bls F2;
  typedef Bls2CurveParams Twist;
  static constexpr unsigned kCurveId = SXT_CURVE_BLS_381;
  static constexpr u32 kXi0 = BLS12_XI0;
  static constexpr bool kMType = true;
  static constexpr u64 kLoopLo = BLS12_LOOP_LO, kLoopHi = BLS12_LOOP_HI;
  static constexpr int kLoopBits = BLS12_LOOP_BITS;
  static constexpr u64 kXAbs = BLS12_X_ABS;
  static constexpr bool kXNeg = BLS12_X_NEG;
  static constexpr u64 kLambda3Lo = BLS12_LAMBDA3_LO, kLambda3Hi = BLS12_LAMBDA3_HI;
  static B200_HD u32 frob(int i) { return BLS12_FROB(i); }
  static B200_HD u32 two_inv(int i) { return BLS12_TWO_INV(i); }
  static B200_HD u32 twist_frob_x(int) { return 0u; }
  static B200_HD u32 twist_frob_y(int) { return 0u; }
};
struct BnTower {
  typedef FBn B;
  typedef Fp2Bn F2;
  typedef Bn2CurveParams Twist;
  static constexpr unsigned kCurveId = SXT_CURVE_BN_254;
  static constexpr u32 kXi0 = BN12_XI0;
  static constexpr bool kMType = false;
  static constexpr u64 kLoopLo = BN12_LOOP_LO, kLoopHi = BN12_LOOP_HI;
  static constexpr int kLoopBits = BN12_LOOP_BITS;
  static constexpr u64 kXAbs = BN12_X_ABS;
  static constexpr bool kXNeg = BN12_X_NEG;
  static constexpr u64 kLambda3Lo = BN12_LAMBDA3_LO, kLambda3Hi = BN12_LAMBDA3_HI;
  static B200_HD u32 frob(int i) { return BN12_FROB(i); }
  static B200_HD u32 two_inv(int i) { return BN12_TWO_INV(i); }
  static B200_HD u32 twist_frob_x(int i) { return BN12_TWIST_FROB_X(i); }
  static B200_HD u32 twist_frob_y(int i) { return BN12_TWIST_FROB_Y(i); }
};

// ---- Fp2 helpers over the tower --------------------------------------------------------------------
template <class T> struct Fp2Ops {
  typedef typename T::B B;
  typedef typename T::F2 F2;
  typedef typename B::E Be;
  typedef typename F2::E E2;
  static constexpr int H = B::N;

  // r = a (kXi0 + u) = (kXi0 a0 - a1) + (a0 + kXi0 a1) u, kXi0 a by doublings and additions
  static B200_HD void mul_by_xi(E2& r, const E2& a) {
    const Be a0 = F2::part(a, 0), a1 = F2::part(a, 1);
    Be s0 = a0, s1 = a1;
#pragma unroll
    for (int bit = 30; bit >= 0; --bit) {
      if ((T::kXi0 >> (bit + 1)) == 0)
        continue;
      B::dbl(s0, s0);
      B::dbl(s1, s1);
      if ((T::kXi0 >> bit) & 1u) {
        B::add(s0, s0, a0);
        B::add(s1, s1, a1);
      }
    }
    Be c0, c1;
    B::sub(c0, s0, a1);
    B::add(c1, a0, s1);
    F2::join(r, c0, c1);
  }
  static B200_HD void conj(E2& r, const E2& a) {
    Be c1;
    B::neg(c1, F2::part(a, 1));
    F2::join(r, F2::part(a, 0), c1);
  }
  static B200_HD void mul_by_fp(E2& r, const E2& a, const Be& s) {
    Be c0, c1;
    B::mul(c0, F2::part(a, 0), s);
    B::mul(c1, F2::part(a, 1), s);
    F2::join(r, c0, c1);
  }
  template <class C> static B200_HD E2 constant(C c) {
    E2 r;
#pragma unroll
    for (int i = 0; i < 2 * H; ++i)
      r.l[i] = c(i);
    return r;
  }
};

// ---- Fp6 = Fp2[v] / (v^3 - xi) ---------------------------------------------------------------------
template <class T> struct Fp6 {
  typedef typename T::F2 F2;
  typedef typename F2::E E2;
  typedef Fp2Ops<T> O;
  struct E {
    E2 c[3];
  };

  static B200_HD E zero() {
    E r;
    r.c[0] = r.c[1] = r.c[2] = F2::zero();
    return r;
  }
  static B200_HD void add(E& r, const E& a, const E& b) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
      F2::add(r.c[k], a.c[k], b.c[k]);
  }
  static B200_HD void sub(E& r, const E& a, const E& b) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
      F2::sub(r.c[k], a.c[k], b.c[k]);
  }
  static B200_HD void neg(E& r, const E& a) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
      F2::neg(r.c[k], a.c[k]);
  }
  // r = a v = (xi a2, a0, a1)
  static B200_HD void mul_by_v(E& r, const E& a) {
    E2 t;
    O::mul_by_xi(t, a.c[2]);
    const E2 a0 = a.c[0], a1 = a.c[1];
    r.c[0] = t;
    r.c[1] = a0;
    r.c[2] = a1;
  }
  // Karatsuba over three Fp2 products and three of sums
  static B200_NOINLINE void mul(E& r, const E& a, const E& b) {
    E2 v0, v1, v2, s, t, c0, c1, c2;
    F2::mul(v0, a.c[0], b.c[0]);
    F2::mul(v1, a.c[1], b.c[1]);
    F2::mul(v2, a.c[2], b.c[2]);
    F2::add(s, a.c[1], a.c[2]);  // c0 = v0 + xi ((a1 + a2)(b1 + b2) - v1 - v2)
    F2::add(t, b.c[1], b.c[2]);
    F2::mul(c0, s, t);
    F2::sub(c0, c0, v1);
    F2::sub(c0, c0, v2);
    O::mul_by_xi(c0, c0);
    F2::add(c0, c0, v0);
    F2::add(s, a.c[0], a.c[1]);  // c1 = (a0 + a1)(b0 + b1) - v0 - v1 + xi v2
    F2::add(t, b.c[0], b.c[1]);
    F2::mul(c1, s, t);
    F2::sub(c1, c1, v0);
    F2::sub(c1, c1, v1);
    O::mul_by_xi(s, v2);
    F2::add(c1, c1, s);
    F2::add(s, a.c[0], a.c[2]);  // c2 = (a0 + a2)(b0 + b2) - v0 - v2 + v1
    F2::add(t, b.c[0], b.c[2]);
    F2::mul(c2, s, t);
    F2::sub(c2, c2, v0);
    F2::sub(c2, c2, v2);
    F2::add(c2, c2, v1);
    r.c[0] = c0;
    r.c[1] = c1;
    r.c[2] = c2;
  }
  static B200_HD void sqr(E& r, const E& a) { mul(r, a, a); }
  // r = a (b0 + b1 v)
  static B200_HD void mul_by_01(E& r, const E& a, const E2& b0, const E2& b1) {
    E2 aa, bb, t0, t1, t2, s;
    F2::mul(aa, a.c[0], b0);
    F2::mul(bb, a.c[1], b1);
    F2::mul(t0, a.c[2], b1);  // c0 = a0 b0 + xi a2 b1
    O::mul_by_xi(t0, t0);
    F2::add(t0, t0, aa);
    F2::add(s, a.c[0], a.c[2]);  // c2 = (a0 + a2) b0 - a0 b0 + a1 b1
    F2::mul(t2, s, b0);
    F2::sub(t2, t2, aa);
    F2::add(t2, t2, bb);
    F2::add(s, a.c[0], a.c[1]);  // c1 = (a0 + a1)(b0 + b1) - a0 b0 - a1 b1
    E2 u;
    F2::add(u, b0, b1);
    F2::mul(t1, s, u);
    F2::sub(t1, t1, aa);
    F2::sub(t1, t1, bb);
    r.c[0] = t0;
    r.c[1] = t1;
    r.c[2] = t2;
  }
  // r = a b1 v = (xi a2 b1, a0 b1, a1 b1)
  static B200_HD void mul_by_1(E& r, const E& a, const E2& b1) {
    E2 t0, t1, t2;
    F2::mul(t0, a.c[2], b1);
    O::mul_by_xi(t0, t0);
    F2::mul(t1, a.c[0], b1);
    F2::mul(t2, a.c[1], b1);
    r.c[0] = t0;
    r.c[1] = t1;
    r.c[2] = t2;
  }
  // 1 / a = (t0 + t1 v + t2 v^2) / (a0 t0 + xi (a2 t1 + a1 t2)), t0 = a0^2 - xi a1 a2,
  // t1 = xi a2^2 - a0 a1, t2 = a1^2 - a0 a2 (0 -> 0)
  static B200_NOINLINE void invert(E& r, const E& a) {
    E2 t0, t1, t2, s, d;
    F2::sqr(t0, a.c[0]);
    F2::mul(s, a.c[1], a.c[2]);
    O::mul_by_xi(s, s);
    F2::sub(t0, t0, s);
    F2::sqr(t1, a.c[2]);
    O::mul_by_xi(t1, t1);
    F2::mul(s, a.c[0], a.c[1]);
    F2::sub(t1, t1, s);
    F2::sqr(t2, a.c[1]);
    F2::mul(s, a.c[0], a.c[2]);
    F2::sub(t2, t2, s);
    F2::mul(d, a.c[2], t1);
    F2::mul(s, a.c[1], t2);
    F2::add(d, d, s);
    O::mul_by_xi(d, d);
    F2::mul(s, a.c[0], t0);
    F2::add(d, d, s);
    F2::invert_eea(d, d);
    F2::mul(r.c[0], t0, d);
    F2::mul(r.c[1], t1, d);
    F2::mul(r.c[2], t2, d);
  }
};

// ---- Fp12 = Fp6[w] / (w^2 - v) -------------------------------------------------------------------------
template <class T> struct Fp12 {
  typedef typename T::F2 F2;
  typedef typename F2::E E2;
  typedef Fp6<T> F6;
  typedef typename F6::E E6;
  typedef Fp2Ops<T> O;
  static constexpr int H = T::B::N;
  static constexpr int N = 12 * H;  // u32 limbs of one element
  struct E {
    E6 c[2];
  };

  static B200_HD E one() {
    E r;
    r.c[0] = r.c[1] = F6::zero();
    r.c[0].c[0] = F2::one();
    return r;
  }
  static B200_HD void load(E& r, const u32* src) {
    u32* d = reinterpret_cast<u32*>(&r);
    for (int i = 0; i < N; ++i)
      d[i] = src[i];
  }
  static B200_HD void store(u32* dst, const E& a) {
    const u32* s = reinterpret_cast<const u32*>(&a);
    for (int i = 0; i < N; ++i)
      dst[i] = s[i];
  }
  static B200_HD void add(E& r, const E& a, const E& b) {
    F6::add(r.c[0], a.c[0], b.c[0]);
    F6::add(r.c[1], a.c[1], b.c[1]);
  }
  static B200_HD void sub(E& r, const E& a, const E& b) {
    F6::sub(r.c[0], a.c[0], b.c[0]);
    F6::sub(r.c[1], a.c[1], b.c[1]);
  }
  static B200_HD void neg(E& r, const E& a) {
    F6::neg(r.c[0], a.c[0]);
    F6::neg(r.c[1], a.c[1]);
  }
  // a^(p^6)
  static B200_HD void conj(E& r, const E& a) {
    r.c[0] = a.c[0];
    F6::neg(r.c[1], a.c[1]);
  }
  // Karatsuba: c0 = a0 b0 + v a1 b1, c1 = (a0 + a1)(b0 + b1) - a0 b0 - a1 b1
  static B200_NOINLINE void mul(E& r, const E& a, const E& b) {
    E6 v0, v1, s, t;
    F6::mul(v0, a.c[0], b.c[0]);
    F6::mul(v1, a.c[1], b.c[1]);
    F6::add(s, a.c[0], a.c[1]);
    F6::add(t, b.c[0], b.c[1]);
    F6::mul(s, s, t);
    F6::sub(s, s, v0);
    F6::sub(r.c[1], s, v1);
    F6::mul_by_v(v1, v1);
    F6::add(r.c[0], v0, v1);
  }
  // complex squaring: t = a0 a1, c0 = (a0 + a1)(a0 + v a1) - t - v t, c1 = 2 t
  static B200_NOINLINE void sqr(E& r, const E& a) {
    E6 t, s, u;
    F6::mul(t, a.c[0], a.c[1]);
    F6::add(s, a.c[0], a.c[1]);
    F6::mul_by_v(u, a.c[1]);
    F6::add(u, u, a.c[0]);
    F6::mul(s, s, u);
    F6::sub(s, s, t);
    F6::mul_by_v(u, t);
    F6::sub(r.c[0], s, u);
    F6::add(r.c[1], t, t);
  }
  // 1 / a = (a0 - a1 w) / (a0^2 - v a1^2) (0 -> 0)
  static B200_NOINLINE void invert(E& r, const E& a) {
    E6 t0, t1;
    F6::sqr(t0, a.c[0]);
    F6::sqr(t1, a.c[1]);
    F6::mul_by_v(t1, t1);
    F6::sub(t0, t0, t1);
    F6::invert(t0, t0);
    F6::mul(t1, a.c[1], t0);
    F6::mul(r.c[0], a.c[0], t0);
    F6::neg(r.c[1], t1);
  }
  // a^(p^K): the coefficient g_i of w^i becomes conj^K(g_i) gamma_{K,i}, gamma_{K,i} = xi^(i (p^K - 1) / 6)
  // (c0.b_j is the coefficient of w^(2j), c1.b_j that of w^(2j+1))
  template <int K> static B200_HD void frobenius(E& r, const E& a) {
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int i = 2 * j + c;
        E2 g = a.c[c].c[j];
        if (K & 1)
          O::conj(g, g);
        if (i > 0) {
          const int base = ((K - 1) * 5 + i - 1) * 2 * H;
          const E2 gamma = O::constant([base](int l) { return T::frob(base + l); });
          F2::mul(g, g, gamma);
        }
        r.c[c].c[j] = g;
      }
  }
  // Granger-Scott squaring of an element of the cyclotomic subgroup (a^(p^6 + 1) = 1): Fp12 as
  // Fp4^3 over Fp4 = Fp2[s] / (s^2 - xi), s = w^3, with the pairs (c0.b0, c1.b1), (c1.b0, c0.b2),
  // (c0.b1, c1.b2); three Fp4 squarings and additions
  static B200_NOINLINE void cyclotomic_sqr(E& r, const E& a) {
    E2 z0 = a.c[0].c[0], z4 = a.c[0].c[1], z3 = a.c[0].c[2];
    E2 z2 = a.c[1].c[0], z1 = a.c[1].c[1], z5 = a.c[1].c[2];
    E2 t0, t1, t2, t3, t4, t5;
    fp4_sqr(t0, t1, z0, z1);
    fp4_sqr(t2, t3, z2, z3);
    fp4_sqr(t4, t5, z4, z5);
    E2 x;
    triple_minus_double(z0, t0, z0);  // z0 = 3 t0 - 2 z0
    triple_plus_double(z1, t1, z1);   // z1 = 3 t1 + 2 z1
    O::mul_by_xi(x, t5);
    triple_plus_double(z2, x, z2);    // z2 = 3 xi t5 + 2 z2
    triple_minus_double(z3, t4, z3);  // z3 = 3 t4 - 2 z3
    triple_minus_double(z4, t2, z4);  // z4 = 3 t2 - 2 z4
    triple_plus_double(z5, t3, z5);   // z5 = 3 t3 + 2 z5
    r.c[0].c[0] = z0;
    r.c[0].c[1] = z4;
    r.c[0].c[2] = z3;
    r.c[1].c[0] = z2;
    r.c[1].c[1] = z1;
    r.c[1].c[2] = z5;
  }
  // (a + b s)^2 = (a^2 + xi b^2) + 2 a b s, as (a + b)(a + xi b) - t - xi t, 2 t with t = a b
  static B200_HD void fp4_sqr(E2& r0, E2& r1, const E2& a, const E2& b) {
    E2 t, s, u;
    F2::mul(t, a, b);
    F2::add(s, a, b);
    O::mul_by_xi(u, b);
    F2::add(u, u, a);
    F2::mul(s, s, u);
    F2::sub(s, s, t);
    O::mul_by_xi(u, t);
    F2::sub(r0, s, u);
    F2::dbl(r1, t);
  }
  static B200_HD void triple_minus_double(E2& r, const E2& t, const E2& z) {
    E2 d;
    F2::sub(d, t, z);
    F2::dbl(d, d);
    F2::add(r, d, t);
  }
  static B200_HD void triple_plus_double(E2& r, const E2& t, const E2& z) {
    E2 d;
    F2::add(d, t, z);
    F2::dbl(d, d);
    F2::add(r, d, t);
  }
  // f *= l0 + l1 v + l4 v w (positions 0, 1, 4: the M-type line)
  static B200_NOINLINE void mul_by_014(E& f, const E2& l0, const E2& l1, const E2& l4) {
    E6 aa, bb, s;
    F6::mul_by_01(aa, f.c[0], l0, l1);
    F6::mul_by_1(bb, f.c[1], l4);
    E2 o;
    F2::add(o, l1, l4);
    F6::add(s, f.c[0], f.c[1]);
    F6::mul_by_01(s, s, l0, o);
    F6::sub(s, s, aa);
    F6::sub(f.c[1], s, bb);
    F6::mul_by_v(bb, bb);
    F6::add(f.c[0], bb, aa);
  }
  // f *= l0 + (l3 + l4 v) w (positions 0, 3, 4: the D-type line)
  static B200_NOINLINE void mul_by_034(E& f, const E2& l0, const E2& l3, const E2& l4) {
    E6 aa, bb, s;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      F2::mul(aa.c[k], f.c[0].c[k], l0);
    F6::mul_by_01(bb, f.c[1], l3, l4);
    E2 o;
    F2::add(o, l0, l3);
    F6::add(s, f.c[0], f.c[1]);
    F6::mul_by_01(s, s, o, l4);
    F6::sub(s, s, aa);
    F6::sub(f.c[1], s, bb);
    F6::mul_by_v(bb, bb);
    F6::add(f.c[0], bb, aa);
  }
};

// ---- the pairing ---------------------------------------------------------------------------------------
template <class T> struct Pairing {
  typedef typename T::B B;
  typedef typename T::F2 F2;
  typedef typename B::E Be;
  typedef typename F2::E E2;
  typedef Fp2Ops<T> O;
  typedef Fp12<T> F12;
  typedef typename F12::E E;
  static constexpr int H = B::N;

  struct G2Proj {  // homogeneous projective: (x, y) = (X / Z, Y / Z)
    E2 x, y, z;
  };
  struct Line {  // the three non-zero Fp2 coefficients, at positions 0, 1, 4 (M) or 0, 3, 4 (D)
    E2 a, b, c;
  };
  // one pair after ingestion: affine P and Q, or identity != 0 when either side is the identity
  struct Pair {
    Be px, py;
    E2 qx, qy;
    u32 identity;
  };

  static B200_HD void mul_by_line(E& f, const Line& l) {
    if (T::kMType)
      F12::mul_by_014(f, l.a, l.b, l.c);
    else
      F12::mul_by_034(f, l.a, l.b, l.c);
  }

  // T = 2T and the tangent at T evaluated at P, scaled by -Z^2 (and by w^3 on the M-type twist):
  // (3b' Z^2 - Y^2) + 3 X^2 x_P w^2 - 2 Y Z y_P w^3 (M), -2 Y Z y_P + 3 X^2 x_P w + (3b' Z^2 - Y^2) w^3 (D)
  static B200_HD void dbl_step(Line& l, G2Proj& t, const Be& px, const Be& py) {
    const Be half = B::constant([](int i) { return T::two_inv(i); });
    E2 a, b, c, e, f, g, h, i, j, s;
    F2::mul(a, t.x, t.y);
    O::mul_by_fp(a, a, half);  // X Y / 2
    F2::sqr(b, t.y);
    F2::sqr(c, t.z);
    T::Twist::template mul_by_3b<F2>(e, c);  // 3 b' Z^2
    F2::dbl(f, e);
    F2::add(f, f, e);  // 3 e
    F2::add(g, b, f);
    O::mul_by_fp(g, g, half);
    F2::add(h, t.y, t.z);
    F2::sqr(h, h);
    F2::add(s, b, c);
    F2::sub(h, h, s);  // 2 Y Z
    F2::sub(i, e, b);
    F2::sqr(j, t.x);
    F2::sub(s, b, f);
    F2::mul(t.x, a, s);
    F2::sqr(s, e);
    E2 e3;
    F2::dbl(e3, s);
    F2::add(e3, e3, s);
    F2::sqr(s, g);
    F2::sub(t.y, s, e3);
    F2::mul(t.z, b, h);
    E2 jx, hy;
    F2::dbl(jx, j);
    F2::add(jx, jx, j);
    O::mul_by_fp(jx, jx, px);
    O::mul_by_fp(hy, h, py);
    F2::neg(hy, hy);
    if (T::kMType) {
      l.a = i;
      l.b = jx;
      l.c = hy;
    } else {
      l.a = hy;
      l.b = jx;
      l.c = i;
    }
  }
  // T = T + Q (Q affine) and the chord through T and Q evaluated at P, with theta = Y - y_Q Z,
  // lambda = X - x_Q Z, j = theta x_Q - lambda y_Q: j - theta x_P w^2 + lambda y_P w^3 (M),
  // lambda y_P - theta x_P w + j w^3 (D)
  static B200_HD void add_step(Line& l, G2Proj& t, const E2& qx, const E2& qy, const Be& px,
                               const Be& py) {
    E2 theta, lambda, c, d, e, f, g, h, s;
    F2::mul(s, qy, t.z);
    F2::sub(theta, t.y, s);
    F2::mul(s, qx, t.z);
    F2::sub(lambda, t.x, s);
    F2::sqr(c, theta);
    F2::sqr(d, lambda);
    F2::mul(e, lambda, d);
    F2::mul(f, t.z, c);
    F2::mul(g, t.x, d);
    F2::add(h, e, f);
    F2::dbl(s, g);
    F2::sub(h, h, s);
    F2::mul(t.x, lambda, h);
    F2::mul(s, e, t.y);
    F2::sub(g, g, h);
    F2::mul(t.y, theta, g);
    F2::sub(t.y, t.y, s);
    F2::mul(t.z, t.z, e);
    E2 j, tx, ly;
    F2::mul(j, theta, qx);
    F2::mul(s, lambda, qy);
    F2::sub(j, j, s);
    O::mul_by_fp(tx, theta, px);
    F2::neg(tx, tx);
    O::mul_by_fp(ly, lambda, py);
    if (T::kMType) {
      l.a = j;
      l.b = tx;
      l.c = ly;
    } else {
      l.a = ly;
      l.b = tx;
      l.c = j;
    }
  }
  // pi on the D-type twist: (conj(x) xi^((p-1)/3), conj(y) xi^((p-1)/2))
  static B200_HD void twist_frobenius(E2& rx, E2& ry, const E2& x, const E2& y) {
    const E2 gx = O::constant([](int l) { return T::twist_frob_x(l); });
    const E2 gy = O::constant([](int l) { return T::twist_frob_y(l); });
    O::conj(rx, x);
    F2::mul(rx, rx, gx);
    O::conj(ry, y);
    F2::mul(ry, ry, gy);
  }

  static B200_HD bool loop_bit(int i) {
    return i >= 64 ? ((T::kLoopHi >> (i - 64)) & 1u) : ((T::kLoopLo >> i) & 1u);
  }

  // The Miller function of `count` consecutive pairs into one accumulator; tp holds their points T
  static B200_HD void miller(E& f, const Pair* pairs, G2Proj* tp, u32 count) {
    f = F12::one();
    for (u32 k = 0; k < count; ++k) {
      tp[k].x = pairs[k].qx;
      tp[k].y = pairs[k].qy;
      tp[k].z = F2::one();
    }
    for (int bit = T::kLoopBits - 2; bit >= 0; --bit) {
      if (bit < T::kLoopBits - 2)
        F12::sqr(f, f);
      const bool add = loop_bit(bit);
      for (u32 k = 0; k < count; ++k) {
        const Pair& pr = pairs[k];
        if (pr.identity)
          continue;
        G2Proj t = tp[k];
        Line l;
        dbl_step(l, t, pr.px, pr.py);
        mul_by_line(f, l);
        if (add) {
          add_step(l, t, pr.qx, pr.qy, pr.px, pr.py);
          mul_by_line(f, l);
        }
        tp[k] = t;
      }
    }
    if (!T::kMType) {  // bn254: the lines through pi(Q) and -pi^2(Q)
      for (u32 k = 0; k < count; ++k) {
        const Pair& pr = pairs[k];
        if (pr.identity)
          continue;
        G2Proj t = tp[k];
        E2 x1, y1, x2, y2;
        twist_frobenius(x1, y1, pr.qx, pr.qy);
        twist_frobenius(x2, y2, x1, y1);
        F2::neg(y2, y2);
        Line l;
        add_step(l, t, x1, y1, pr.px, pr.py);
        mul_by_line(f, l);
        add_step(l, t, x2, y2, pr.px, pr.py);
        mul_by_line(f, l);
      }
    }
    if (T::kXNeg)
      F12::conj(f, f);
  }

  // a^e for e = hi 2^64 + lo, a in the cyclotomic subgroup
  static B200_NOINLINE void cyclotomic_pow(E& r, const E& a, u64 hi, u64 lo) {
    E acc = F12::one();
    bool started = false;
    for (int i = 127; i >= 0; --i) {
      const bool bit = i >= 64 ? ((hi >> (i - 64)) & 1u) : ((lo >> i) & 1u);
      if (started)
        F12::cyclotomic_sqr(acc, acc);
      if (bit) {
        if (started)
          F12::mul(acc, acc, a);
        else
          acc = a;
        started = true;
      }
    }
    r = acc;
  }
  // a^x for the family's parameter x (cyclotomic a: the inverse is the conjugate)
  static B200_HD void pow_x(E& r, const E& a) {
    cyclotomic_pow(r, a, 0, T::kXAbs);
    if (T::kXNeg)
      F12::conj(r, r);
  }

  // f^((p^12 - 1) / r): the easy part f^((p^6 - 1)(p^2 + 1)), then the hard part. The two parts and
  // the powers are called functions: composed inline in one frame, the bls12-381 exponentiation came
  // out wrong on sm_90a while every step of it was right on its own.
  static B200_NOINLINE void final_exp(E& r, const E& a) {
    E f;
    easy_part(f, a);
    hard_part(r, f);
  }
  static B200_NOINLINE void easy_part(E& r, const E& a) {
    E f, t;
    F12::conj(f, a);
    F12::invert(t, a);
    F12::mul(f, f, t);
    F12::template frobenius<2>(t, f);
    F12::mul(r, t, f);
  }
  // f^((p^4 - p^2 + 1) / r) for a cyclotomic f, (p^4 - p^2 + 1) / r = lambda_0 + lambda_1 p +
  // lambda_2 p^2 + lambda_3 p^3 (gen_constants.py)
  static B200_NOINLINE void hard_part(E& r, const E& f) {
    E t;
    E l0, l1, l2, l3;
    if (T::kXNeg) {  // bls12-381: lambda_3 = (x - 1)^2 / 3, then lambda_{i-1} from lambda_i by x
      cyclotomic_pow(l3, f, T::kLambda3Hi, T::kLambda3Lo);
      pow_x(l2, l3);
      pow_x(l1, l2);
      F12::conj(t, l3);
      F12::mul(l1, l1, t);  // lambda_1 = lambda_2 x - lambda_3
      pow_x(l0, l1);
      F12::mul(l0, l0, f);  // lambda_0 = lambda_1 x + 1
    } else {  // bn254: lambda_3 = 1, lambda_2 = 6x^2 + 1, lambda_1 = -36x^3 - 18x^2 - 12x + 1,
              //        lambda_0 = -36x^3 - 30x^2 - 18x - 2, from f^x, f^(x^2), f^(x^3)
      E fx, fx2, fx3, s;
      pow_x(fx, f);
      pow_x(fx2, fx);
      pow_x(fx3, fx2);
      l3 = f;
      cyclotomic_pow(l2, fx2, 0, 6);
      F12::mul(l2, l2, f);
      E t36;
      cyclotomic_pow(t36, fx3, 0, 36);
      cyclotomic_pow(s, fx2, 0, 18);
      F12::mul(l1, t36, s);
      cyclotomic_pow(s, fx, 0, 12);
      F12::mul(l1, l1, s);
      F12::conj(l1, l1);
      F12::mul(l1, l1, f);
      cyclotomic_pow(s, fx2, 0, 30);
      F12::mul(l0, t36, s);
      cyclotomic_pow(s, fx, 0, 18);
      F12::mul(l0, l0, s);
      F12::cyclotomic_sqr(s, f);
      F12::mul(l0, l0, s);
      F12::conj(l0, l0);
    }
    F12::template frobenius<1>(t, l1);
    F12::mul(l0, l0, t);
    F12::template frobenius<2>(t, l2);
    F12::mul(l0, l0, t);
    F12::template frobenius<3>(t, l3);
    F12::mul(r, l0, t);
  }
};

// ---- kernels ---------------------------------------------------------------------------------------
// projective ABI structs -> affine pairs (one thread per pair)
template <class T> struct PairingIngestBody {
  static constexpr int kBlock = 128;
  typedef Pairing<T> P;
  typedef typename T::B B;
  typedef typename T::F2 F2;
  const u32* g1;  // 3 B::N limbs per point (X, Y, Z)
  const u32* g2;  // 3 F2::N limbs per point
  typename P::Pair* pairs;

  B200_HD void operator()(u64 i) const {
    typename B::E x1, y1, z1;
    typename F2::E x2, y2, z2;
    const u32* a = g1 + i * 3 * B::N;
    const u32* b = g2 + i * 3 * F2::N;
    B::load(x1, a);
    B::load(y1, a + B::N);
    B::load(z1, a + 2 * B::N);
    F2::load(x2, b);
    F2::load(y2, b + F2::N);
    F2::load(z2, b + 2 * F2::N);
    typename P::Pair& pr = pairs[i];
    pr.identity = (B::is_zero(z1) || F2::is_zero(z2)) ? 1u : 0u;
    B::invert_eea(z1, z1);
    B::mul(pr.px, x1, z1);
    B::mul(pr.py, y1, z1);
    F2::invert_eea(z2, z2);
    F2::mul(pr.qx, x2, z2);
    F2::mul(pr.qy, y2, z2);
  }
};

// one Miller accumulator per thread over the pairs task[2t] .. task[2t] + task[2t + 1]
template <class T> struct PairingMillerBody {
  static constexpr int kBlock = 64;
  typedef Pairing<T> P;
  const u32* task;
  const typename P::Pair* pairs;
  typename P::G2Proj* tp;
  typename P::E* acc;

  B200_HD void operator()(u64 t) const {
    const u32 first = task[2 * t], count = task[2 * t + 1];
    typename P::E f;
    P::miller(f, pairs + first, tp + first, count);
    acc[t] = f;
  }
};

// one level of the segmented tree product: within each product's run of accumulators, local index
// j (a multiple of 2 stride) takes the product with j + stride
template <class T> struct PairingProductBody {
  static constexpr int kBlock = 128;
  typedef Pairing<T> P;
  typename P::E* acc;
  const u32* product_of;  // per accumulator
  const u32* begin;       // per product, and the end
  u32 stride;

  B200_HD void operator()(u64 i) const {
    const u32 k = product_of[i];
    const u32 j = (u32)i - begin[k], count = begin[k + 1] - begin[k];
    if (j % (2 * stride) == 0 && j + stride < count)
      Fp12<T>::mul(acc[i], acc[i], acc[i + stride]);
  }
};

// the final exponentiation of each product's accumulator, written in the GT ABI layout (one for an
// empty product)
template <class T> struct PairingFinalExpBody {
  static constexpr int kBlock = 32;
  typedef Pairing<T> P;
  const typename P::E* acc;
  const u32* begin;
  u32* out;

  B200_HD void operator()(u64 k) const {
    typename P::E f = Fp12<T>::one();
    if (begin[k + 1] > begin[k])
      P::final_exp(f, acc[begin[k]]);
    Fp12<T>::store(out + k * Fp12<T>::N, f);
  }
};

// Accumulators the Miller loop should spread a call over: 132 SMs x 256 threads resident at the Miller
// kernel's register count. Longer calls take several consecutive pairs of one product per thread.
constexpr u64 kMillerThreads = 132 * 256;

// out[k] = prod of e(g1[i], g2[i]) over product k's pairs (device pointers; lengths is a host array)
template <class T>
void multi_pairing(const EngineCtx& ctx, void* out, uint32_t num_products, const uint32_t* lengths,
                   const void* g1, const void* g2) {
  typedef Pairing<T> P;
  u64 total = 0;
  for (uint32_t k = 0; k < num_products; ++k)
    total += lengths[k];
  const u64 per_thread = std::max<u64>(1, (total + kMillerThreads - 1) / kMillerThreads);
  // accumulator t of product k covers pairs [first, first + count): product k's pairs split evenly
  std::vector<u32> task, product_of, begin(num_products + 1, 0);
  u64 first = 0;
  u32 longest = 0;
  for (uint32_t k = 0; k < num_products; ++k) {
    const u64 len = lengths[k], threads = (len + per_thread - 1) / per_thread;
    for (u64 j = 0; j < threads; ++j) {
      const u64 lo = len * j / threads, hi = len * (j + 1) / threads;
      task.push_back((u32)(first + lo));
      task.push_back((u32)(hi - lo));
      product_of.push_back(k);
    }
    first += len;
    begin[k + 1] = (u32)(begin[k] + threads);
    longest = std::max(longest, (u32)threads);
  }
  const u64 threads = product_of.size();
  stream_t s = ctx.s;
  u32* d_begin = (u32*)stage_to_device(s, begin.data(), begin.size() * sizeof(u32));
  DevBuf<typename P::E> acc(threads, s);
  if (threads) {
    u32* d_task = (u32*)stage_to_device(s, task.data(), task.size() * sizeof(u32));
    u32* d_product_of = (u32*)stage_to_device(s, product_of.data(), threads * sizeof(u32));
    DevBuf<typename P::Pair> pairs(total, s);
    DevBuf<typename P::G2Proj> tp(total, s);
    launch(PairingIngestBody<T>{(const u32*)g1, (const u32*)g2, pairs.p}, total, s);
    launch(PairingMillerBody<T>{d_task, pairs.p, tp.p, acc.p}, threads, s);
    for (u32 stride = 1; stride < longest; stride *= 2)
      launch(PairingProductBody<T>{acc.p, d_product_of, d_begin, stride}, threads, s);
    dev_free(d_task, s);
    dev_free(d_product_of, s);
  }
  launch(PairingFinalExpBody<T>{acc.p, d_begin, (u32*)out}, num_products, s);
  dev_free(d_begin, s);
}

// b200_field_op on Fp12 (fields 8 and 9): add, sub, neg, mul, sqr, invert, frobenius (a^p),
// cyclotomic_sqr and final_exp
template <class T> struct Fp12OpBody {
  static constexpr int kBlock = 32;
  typedef Fp12<T> F;
  u32 op;
  FieldOpShape w;
  const u32* a;
  const u32* b;
  u32* out;

  static B200_HD FieldOpShape shape(u32 op) {
    const u32 n = F::N;
    switch (op) {
    case kOpAdd: case kOpSub: case kOpMul: return FieldOpShape{n, n, n};
    case kOpNeg: case kOpSqr: case kOpInvert: case kOpFrobenius: case kOpCyclotomicSqr:
    case kOpFinalExp: return FieldOpShape{n, 0, n};
    default: return FieldOpShape{0, 0, 0};
    }
  }
  B200_HD void operator()(u64 i) const {
    typename F::E x, y, r;
    F::load(x, a + i * w.a);
    if (w.b)
      F::load(y, b + i * w.b);
    switch (op) {
    case kOpAdd: F::add(r, x, y); break;
    case kOpSub: F::sub(r, x, y); break;
    case kOpNeg: F::neg(r, x); break;
    case kOpMul: F::mul(r, x, y); break;
    case kOpSqr: F::sqr(r, x); break;
    case kOpInvert: F::invert(r, x); break;
    case kOpFrobenius: F::template frobenius<1>(r, x); break;
    case kOpCyclotomicSqr: F::cyclotomic_sqr(r, x); break;
    default: Pairing<T>::final_exp(r, x); break;  // kOpFinalExp
    }
    F::store(out + i * w.out, r);
  }
};

template <class T>
unsigned run_fp12_op(const EngineCtx& ctx, u32 op, u64 n, const u32* a, const u32* b, u32* out) {
  return run_elementwise(ctx, Fp12OpBody<T>{op, Fp12OpBody<T>::shape(op), a, b, out}, n, n, a, b, out);
}

}  // namespace b200
