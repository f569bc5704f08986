// Validation and decoding of points from outside the library (b200_check_points,
// b200_decode_points): one thread per point.
//
// A point is valid when, in this order,
//   1. every coordinate (each Fp component of an Fp2) is a Montgomery residue below p. This comes
//      before any arithmetic, because the Montgomery product needs a < p;
//   2. Z = 0: the identity, whatever X and Y are;
//   3. otherwise Y^2 Z = X^3 + b Z^3, checked as 3 (Y^2 Z - X^3) = 3b Z^3 with the curve's own 3b;
//   4. for the curves with a cofactor, the point lies in the order-r subgroup, by endomorphisms:
//        bls12-381 G1: phi(P) = (beta X : Y : Z) = [-x^2] P (Scott 2021);
//        bls12-381 G2: psi(Q) = (conj(X) cx : conj(Y) cy : conj(Z)) = [x] Q, the M-type twist's psi;
//        bn254 G2:     psi(Q) = [6 x^2] Q with the D-type pi of the Miller loop (pairing.cuh).
//      bn254 G1 and Grumpkin have prime order: the on-curve check suffices.
// The scalar multiples use the complete RCB16 add / dbl of curve.cuh. They are complete for these
// groups because every group order involved is odd (gen_constants.py asserts it).
//
// Decoding reads the commitment layouts the library writes: the zcash compressed encodings of
// bls12-381 G1 (48 bytes) and G2 (96 bytes), which need a square root in Fp or Fp2, and the affine
// {X, Y, u8 infinity, pad} structs of bn254 G1, Grumpkin and bn254 G2. A valid point is written as
// the projective struct {x R, y R, R}, the identity as identity() writes it, {0, R, 0}, and so is an
// invalid input, with valid = 0.
#pragma once
#include "pairing.cuh"

namespace b200 {

// the base field of F (F itself, or the field under an Fp2) and its number of components in F
template <class F> struct BaseField {
  typedef F B;
  static constexpr int kParts = 1;
};
template <class B_, class P> struct BaseField<Fp2<B_, P>> {
  typedef B_ B;
  static constexpr int kParts = 2;
};

// every Fp component of a is below p
template <class F> B200_HD bool reduced(const typename F::E& a) {
  typedef typename BaseField<F>::B B;
  const typename B::E p = B::modulus();
  bool ok = true;
#pragma unroll
  for (int k = 0; k < BaseField<F>::kParts; ++k) {
    u32 d[B::N];
    ok = ok && limbs_sub<B::N>(d, a.l + k * B::N, p.l) != 0;  // a borrow: the component is < p
  }
  return ok;
}

// ---- square roots in the bls12-381 Fp and Fp2 (both p = 3 mod 4) ---------------------------------
// Sqrt<F>::root(r, a) returns whether a is a square; r is then a root, else 0.
template <class F> struct Sqrt;
template <> struct Sqrt<FBls> {
  struct Exp {  // (p + 1) / 4
    B200_HD u32 operator()(int i) const { return BLS_SQRT_EXP(i); }
  };
  static B200_HD bool root(FBls::E& r, const FBls::E& a) {
    FBls::E c, s;
    FBls::pow(c, a, Exp{});
    FBls::sqr(s, c);
    const bool ok = FBls::equal(s, a);
    FBls::select(r, FBls::zero(), c, ok);
    return ok;
  }
};
// Adj and Rodriguez-Henriquez, Algorithm 9: a1 = a^((p-3)/4), alpha = a1^2 a, x0 = a1 a; the root is
// u x0 when alpha = -1, else (1 + alpha)^((p-1)/2) x0. The candidate is checked by squaring it.
template <> struct Sqrt<Fp2Bls> {
  typedef Fp2Bls F;
  struct Exp {  // (p - 3) / 4
    B200_HD u32 operator()(int i) const { return BLS2_SQRT_EXP(i); }
  };
  struct Half {  // (p - 1) / 2
    B200_HD u32 operator()(int i) const { return BLS_HALF(i); }
  };
  static B200_HD bool root(F::E& r, const F::E& a) {
    F::E a1, alpha, x0, c, s, minus_one;
    F::pow(a1, a, Exp{});
    F::sqr(alpha, a1);
    F::mul(alpha, alpha, a);
    F::mul(x0, a1, a);
    F::neg(minus_one, F::one());
    if (F::equal(alpha, minus_one)) {
      FBls::E n;  // u x0 = -x0.c1 + x0.c0 u
      FBls::neg(n, F::part(x0, 1));
      F::join(c, n, F::part(x0, 0));
    } else {
      F::E b;
      F::add(b, alpha, F::one());
      F::pow(b, b, Half{});
      F::mul(c, b, x0);
    }
    F::sqr(s, c);
    const bool ok = F::equal(s, a);
    F::select(r, F::zero(), c, ok);
    return ok;
  }
};

// ---- subgroup checks ---------------------------------------------------------------------------------
template <class C> struct PointOps {
  typedef typename C::F F;
  typedef typename C::fe fe;
  typedef typename C::Point Point;

  // [k] p, double-and-add from the top bit
  static B200_HD void mul_u64(Point& r, const Point& p, u64 k) {
    Point acc = C::identity();
#pragma unroll 1
    for (int i = 63; i >= 0; --i) {
      C::dbl(acc, acc);
      if ((k >> i) & 1u)
        C::add(acc, acc, p);
    }
    r = acc;
  }
  // [k]([k] p)
  static B200_HD void mul_u64_twice(Point& r, const Point& p, u64 k) {
    mul_u64(r, p, k);
    mul_u64(r, r, k);
  }
  // a and b are the same point (projective cross products; the identity only equals itself)
  static B200_HD bool same(const Point& a, const Point& b) {
    const bool ia = F::is_zero(a.Z), ib = F::is_zero(b.Z);
    if (ia || ib)
      return ia && ib;
    fe l, r;
    F::mul(l, a.X, b.Z);
    F::mul(r, b.X, a.Z);
    if (!F::equal(l, r))
      return false;
    F::mul(l, a.Y, b.Z);
    F::mul(r, b.Y, a.Z);
    return F::equal(l, r);
  }
  // Y^2 Z = X^3 + b Z^3, as 3 (Y^2 Z - X^3) = 3b Z^3
  static B200_HD bool on_curve(const Point& p) {
    fe y2z, x3, t, l, z3, r;
    F::sqr(y2z, p.Y);
    F::mul(y2z, y2z, p.Z);
    F::sqr(x3, p.X);
    F::mul(x3, x3, p.X);
    F::sub(t, y2z, x3);
    F::dbl(l, t);
    F::add(l, l, t);
    F::sqr(z3, p.Z);
    F::mul(z3, z3, p.Z);
    C::mul_by_3b(r, z3);
    return F::equal(l, r);
  }
};

// Subgroup<C>::contains(p) for an on-curve p other than the identity
template <class C> struct Subgroup {  // bn254 G1, Grumpkin: prime order
  static B200_HD bool contains(const typename C::Point&) { return true; }
};
template <> struct Subgroup<Bls12381G1> {
  typedef PointOps<Bls12381G1> O;
  // phi(P) = [-x^2] P = -[|x|]([|x|] P)
  static B200_HD bool contains(const Bls12381G1::Point& p) {
    Bls12381G1::Point q, phi = p;
    O::mul_u64_twice(q, p, BLS12_X_ABS);
    Bls12381G1::neg(q, q);
    FBls::mul(phi.X, p.X, FBls::constant([](int i) { return BLS_BETA(i); }));
    return O::same(phi, q);
  }
};
template <> struct Subgroup<Bls12381G2> {
  typedef PointOps<Bls12381G2> O;
  typedef Fp2Ops<BlsTower> T;
  // psi(Q) = [x] Q = -[|x|] Q
  static B200_HD bool contains(const Bls12381G2::Point& p) {
    Bls12381G2::Point q, psi;
    O::mul_u64(q, p, BLS12_X_ABS);
    Bls12381G2::neg(q, q);
    T::conj(psi.X, p.X);
    Fp2Bls::mul(psi.X, psi.X, T::constant([](int i) { return BLS2_PSI_X(i); }));
    T::conj(psi.Y, p.Y);
    Fp2Bls::mul(psi.Y, psi.Y, T::constant([](int i) { return BLS2_PSI_Y(i); }));
    T::conj(psi.Z, p.Z);
    return O::same(psi, q);
  }
};
template <> struct Subgroup<Bn254G2> {
  typedef PointOps<Bn254G2> O;
  // psi(Q) = [6 x^2] Q, psi = the twist Frobenius of the Miller loop on projective coordinates
  static B200_HD bool contains(const Bn254G2::Point& p) {
    Bn254G2::Point q, t, psi;
    O::mul_u64_twice(q, p, BN12_X_ABS);
    Bn254G2::dbl(t, q);
    Bn254G2::add(q, t, q);
    Bn254G2::dbl(q, q);
    Pairing<BnTower>::twist_frobenius(psi.X, psi.Y, p.X, p.Y);
    Fp2Ops<BnTower>::conj(psi.Z, p.Z);
    return O::same(psi, q);
  }
};

// ---- validation and decoding -------------------------------------------------------------------------
template <class C> struct PointCheck {
  typedef typename C::F F;
  typedef typename C::fe fe;
  typedef typename C::Point Point;
  typedef PointOps<C> O;
  static constexpr bool kCompressed = C::kCurveId == kBls12381 || C::kCurveId == kBls12381G2;

  // steps 1-4 of the header comment
  static B200_HD bool valid(const Point& p) {
    if (!reduced<F>(p.X) || !reduced<F>(p.Y) || !reduced<F>(p.Z))
      return false;
    if (F::is_zero(p.Z))
      return true;
    return O::on_curve(p) && Subgroup<C>::contains(p);
  }

  // the zcash compressed encoding (BlsCurveParams / Bls2CurveParams::store_commit): 4 N bytes, the
  // big-endian value x (G2: x.c1 then x.c0), flags in the top three bits
  static B200_HD bool decode_compressed(Point& p, const unsigned char* s) {
    constexpr int N = C::N;
    const u32 flags = s[0];
    fe x;
#pragma unroll
    for (int i = 0; i < N; ++i)
      x.l[N - 1 - i] = ((u32)s[4 * i] << 24) | ((u32)s[4 * i + 1] << 16) |
                       ((u32)s[4 * i + 2] << 8) | (u32)s[4 * i + 3];
    x.l[N - 1] &= 0x1fffffffu;
    if (!(flags & 0x80u))  // uncompressed forms are not accepted
      return false;
    if (flags & 0x40u) {  // the identity: no sign flag, every other bit zero
      p = C::identity();
      return !(flags & 0x20u) && F::is_zero(x);
    }
    if (!reduced<F>(x))
      return false;
    fe rhs, y, b;
#pragma unroll
    for (int i = 0; i < N; ++i)
      b.l[i] = C::kCurveId == kBls12381 ? BLS_B(i) : BLS2_B(i);
    F::to_mont(x, x);
    F::sqr(rhs, x);
    F::mul(rhs, rhs, x);
    F::add(rhs, rhs, b);
    if (!Sqrt<F>::root(y, rhs))
      return false;
    if (F::lexicographically_largest(y) != ((flags & 0x20u) != 0))
      F::neg(y, y);
    p.X = x;
    p.Y = y;
    p.Z = F::one();
    return Subgroup<C>::contains(p);
  }
  // the affine struct {X, Y, u8 infinity, pad} (store_affine_commit); the padding is not read
  static B200_HD bool decode_affine(Point& p, const unsigned char* s) {
    const unsigned char inf = s[8 * C::N];
    if (inf == 1) {
      p = C::identity();
      return true;
    }
    F::load(p.X, s);
    F::load(p.Y, s + 4 * C::N);
    p.Z = F::one();
    return inf == 0 && reduced<F>(p.X) && reduced<F>(p.Y) && O::on_curve(p) &&
           Subgroup<C>::contains(p);
  }
  static B200_HD bool decode(Point& p, const unsigned char* s) {
    bool ok;
    if constexpr (kCompressed)
      ok = decode_compressed(p, s);
    else
      ok = decode_affine(p, s);
    if (!ok)
      p = C::identity();
    return ok;
  }
};

template <class C> struct CheckPointsBody {
  static constexpr int kBlock = 64;
  const unsigned char* points;  // projective ABI structs
  unsigned char* valid;

  B200_HD void operator()(u64 i) const {
    typename C::Point p;
    const unsigned char* s = points + i * C::kAbiProjBytes;
    C::F::load(p.X, s);
    C::F::load(p.Y, s + 4 * C::N);
    C::F::load(p.Z, s + 8 * C::N);
    valid[i] = PointCheck<C>::valid(p) ? 1 : 0;
  }
};

template <class C> struct DecodePointsBody {
  static constexpr int kBlock = 64;
  const unsigned char* encoded;  // commitments, kAbiCommitBytes each
  unsigned char* out;            // projective ABI structs
  unsigned char* valid;

  B200_HD void operator()(u64 i) const {
    typename C::Point p;
    const bool ok = PointCheck<C>::decode(p, encoded + i * C::kAbiCommitBytes);
    C::store_proj_abi(out + i * C::kAbiProjBytes, p);
    valid[i] = ok ? 1 : 0;
  }
};

// b200_field_op op 27 (sqrt) on fields 1 and 6: the root, then the was-square flag
template <class F> struct SqrtOpBody {
  static constexpr int kBlock = 64;
  FieldOpShape w;
  const u32* a;
  const u32* b;
  u32* out;

  B200_HD void operator()(u64 i) const {
    typename F::E x, r;
    F::load(x, a + i * w.a);
    const bool ok = Sqrt<F>::root(r, x);
    F::store(out + i * w.out, r);
    out[i * w.out + F::N] = ok ? 1u : 0u;
  }
};
template <class F>
unsigned run_sqrt_op(const EngineCtx& ctx, uint64_t n, const uint32_t* a, uint32_t* out) {
  const FieldOpShape w{F::N, 0, F::N + 1};
  return run_elementwise(ctx, SqrtOpBody<F>{w, a, nullptr, out}, n, n, a, nullptr, out);
}

}  // namespace b200
