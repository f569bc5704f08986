// MEASURED AND REJECTED (round 1, DESIGN.md "What was measured and rejected"): kept out of the product,
// next to the micro-benchmark that produced the numbers (tests/micro/latency.cu).
//   * FP64-pipe field multiplication (F25519D) and the FP64 point accumulator built on it: exact, but
//     no faster per warp-multiplication and slower per point addition;
//   * one-level subtractive Karatsuba: slower per warp-multiplication.
// GF(2^255-19) multiplication on the FP64 pipe, for the bucket-accumulation kernel only.
//
// tests/micro/pipes.cu measures the issue rates of IMAD.WIDE.U32 and DFMA this trade rests on.
// A 52x52-bit product costs three FP64 instructions here (two DFMA.RZ + one DADD) against about
// six-and-a-half IMAD.WIDE for the same bits, so the field multiplication of the hot loop moves to
// double precision with EXACT integer semantics:
//
//   * a field element is five signed limbs, radix 2^51 ("balanced": |limb| <= 2^50 + 2^14), held as
//     int64; lazy add / sub are limb-wise on exact doubles (|operand limb| < 2^51.2);
//   * limb products p = a_i * b_j (|p| < 2^103) are split exactly with round-toward-zero FMAs:
//       h = fma_rz(a, b, 1.5*2^104)          = 1.5*2^104 + 2^52 * floor(p / 2^52)
//       l = fma_rz(a, b, (1.5*2^104 + 2^52) - h) = 2^52 + (p mod 2^52)
//     whose mantissas ARE the integers floor(p/2^52) and p mod 2^52, so the column sums are plain
//     int64 additions of the raw bit patterns (the exponent constants are subtracted once per column);
//   * columns 5..9 fold with 2^255 = 19, then one balanced carry chain renormalises.
//
// Host (emulation) builds evaluate fma_rz with exact 128-bit integer arithmetic, so the same
// schedule is verified bit-for-bit on a CPU (tests/emul: emul_check_fp64).
#pragma once
#include "../../blitzar_b200/csrc/curve.cuh"

namespace b200 {

typedef long long i64;

struct FeD {
  i64 l[5];  // value = sum l[i] * 2^(51 i), balanced limbs
};

B200_HD double fma_rz_exact(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rz(a, b, c);
#else
  // every use in this file has integer-valued operands below 2^106: evaluate exactly, then
  // truncate toward zero to 53 significant bits
  __int128 s = (__int128)(i64)a * (__int128)(i64)b;
  // c may exceed 2^63: decompose c = ch * 2^52 + cl with integer parts
  double ch = __builtin_floor(c / 4503599627370496.0);
  double cl = c - ch * 4503599627370496.0;
  s += ((__int128)(i64)ch << 52) + (__int128)(i64)cl;
  bool neg = s < 0;
  unsigned __int128 m = neg ? (unsigned __int128)(-s) : (unsigned __int128)s;
  int bits = 0;
  for (unsigned __int128 t = m; t; t >>= 1)
    ++bits;
  if (bits > 53)
    m = (m >> (bits - 53)) << (bits - 53);  // truncate toward zero
  double r = 0;
  for (int i = 0; i < 128; i += 32)
    r += __builtin_ldexp((double)(unsigned)(m >> i), i);
  return neg ? -r : r;
#endif
}
B200_HD i64 double_bits(double d) {
#ifdef __CUDA_ARCH__
  return __double_as_longlong(d);
#else
  i64 r;
  __builtin_memcpy(&r, &d, 8);
  return r;
#endif
}
B200_HD double bits_double(i64 v) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(v);
#else
  double r;
  __builtin_memcpy(&r, &v, 8);
  return r;
#endif
}

struct F25519D {
  static constexpr double kMagic = 6755399441055744.0;            // 1.5 * 2^52
  static constexpr i64 kMagicBits = 0x4338000000000000LL;
  static constexpr double kC1 = 30423614405477505635920876929024.0;  // 1.5 * 2^104
  static constexpr i64 kC1Bits = 0x4678000000000000LL;
  static constexpr double kC2 = 4503599627370496.0;               // 2^52
  static constexpr i64 kC2Bits = 0x4330000000000000LL;
  static constexpr double kC12 = 30423614405477510139520504299520.0;  // 1.5 * 2^104 + 2^52
  static constexpr i64 kMask51 = (1LL << 51) - 1;

  // exact int -> double for |x| < 2^51
  static B200_HD double to_double(i64 x) { return bits_double(x + kMagicBits) - kMagic; }

  // 8 x u32 canonical value (< 2^255) -> five unsigned 51-bit limbs
  static B200_HD void from_fe(FeD& r, const Fe<8>& a) {
    u64 w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      w[i] = (u64)a.l[2 * i] | ((u64)a.l[2 * i + 1] << 32);
    r.l[0] = (i64)(w[0] & (u64)kMask51);
    r.l[1] = (i64)(((w[0] >> 51) | (w[1] << 13)) & (u64)kMask51);
    r.l[2] = (i64)(((w[1] >> 38) | (w[2] << 26)) & (u64)kMask51);
    r.l[3] = (i64)(((w[2] >> 25) | (w[3] << 39)) & (u64)kMask51);
    r.l[4] = (i64)(w[3] >> 12);  // < 2^51 for canonical input (< 2^52 otherwise)
  }
  // balanced limbs -> loosely reduced 8 x u32 (adds 4p so every limb is non-negative)
  static B200_HD void to_fe(Fe<8>& r, const FeD& a) {
    u64 h[5];
    h[0] = (u64)(a.l[0] + 4 * ((1LL << 51) - 19));
#pragma unroll
    for (int i = 1; i < 5; ++i)
      h[i] = (u64)(a.l[i] + 4 * ((1LL << 51) - 1));
    F25519::from_radix51(r, h);
  }

  // r = a * b for exact-double operands with |limb| < 2^51.5; result balanced
  static B200_HD void mul(FeD& r, const double* a, const double* b) {
    u64 lo[9], hi[9];  // raw bit patterns, summed modulo 2^64
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      lo[k] = 0;
      hi[k] = 0;
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) {
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        double h = fma_rz_exact(a[i], b[j], kC1);
        double l = fma_rz_exact(a[i], b[j], kC12 - h);
        hi[i + j] += (u64)double_bits(h);
        lo[i + j] += (u64)double_bits(l);
      }
    }
    // strip the exponent constants: column k holds n_k products
    i64 R[10], L[9], H[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const u64 n = k < 5 ? k + 1 : 9 - k;
      L[k] = (i64)(lo[k] - n * (u64)kC2Bits);
      H[k] = (i64)(hi[k] - n * (u64)kC1Bits);
    }
    // 2^52 = 2 * 2^51: the high parts land one column up, doubled
    R[0] = L[0];
#pragma unroll
    for (int k = 1; k < 9; ++k)
      R[k] = L[k] + 2 * H[k - 1];
    R[9] = 2 * H[8];
    // fold columns 5..9 with 2^255 = 19
    i64 t[5];
#pragma unroll
    for (int k = 0; k < 5; ++k)
      t[k] = R[k] + 19 * R[k + 5];
    carry(r, t);
  }

  // balanced carry chain: limbs 1..4 end in [-2^50, 2^50), limb 0 within 2^50 + 2^14
  static B200_HD void carry(FeD& r, i64* t) {
    i64 c;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c = (t[k] + (1LL << 50)) >> 51;
      t[k] -= c << 51;
      t[k + 1] += c;
    }
    c = (t[4] + (1LL << 50)) >> 51;
    t[4] -= c << 51;
    t[0] += 19 * c;
#pragma unroll
    for (int k = 0; k < 5; ++k)
      r.l[k] = t[k];
  }
};


namespace rejected {
typedef F25519::E fe;
struct AccD {
    FeD X, Y, Z, T;
  };
static B200_HD void accd_to_doubles(double* d, const FeD& a) {
#pragma unroll
    for (int i = 0; i < 5; ++i)
      d[i] = F25519D::to_double(a.l[i]);
  }
static B200_HD void accd_from_gen(AccD& r, const Ed25519::Gen& g, bool negate) {
    FeD yp, ym, z2, t2d, invd;
    F25519D::from_fe(yp, g.YpX);
    F25519D::from_fe(ym, g.YmX);
    F25519D::from_fe(z2, g.Z2);
    F25519D::from_fe(t2d, g.T2d);
    F25519D::from_fe(invd, F25519::constant([](int i) { return F25_INVD(i); }));
    i64 x[5], y[5], z[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      x[i] = yp.l[i] - ym.l[i];
      y[i] = yp.l[i] + ym.l[i];
      z[i] = z2.l[i];
    }
    double dt[5], dk[5];
    accd_to_doubles(dt, t2d);
    accd_to_doubles(dk, invd);
    F25519D::mul(r.T, dt, dk);
    F25519D::carry(r.X, x);
    F25519D::carry(r.Y, y);
    F25519D::carry(r.Z, z);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      r.X.l[i] = negate ? -r.X.l[i] : r.X.l[i];
      r.T.l[i] = negate ? -r.T.l[i] : r.T.l[i];
    }
  }
  // a += (negate ? -g : g): the 8-multiplication cached-form addition with the products on the
  // FP64 pipe; lazy additions are exact double additions of converted limbs
static B200_HD void accd_add_gen(AccD& a, const Ed25519::Gen& g, bool negate) {
    FeD yp, ym, z2, t2d;
    F25519D::from_fe(yp, g.YpX);
    F25519D::from_fe(ym, g.YmX);
    F25519D::from_fe(z2, g.Z2);
    F25519D::from_fe(t2d, g.T2d);
    double qp[5], qm[5], qz[5], qt[5], x1[5], y1[5], z1[5], t1[5], t0[5], s1[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      qp[i] = F25519D::to_double(negate ? ym.l[i] : yp.l[i]);
      qm[i] = F25519D::to_double(negate ? yp.l[i] : ym.l[i]);
      qz[i] = F25519D::to_double(z2.l[i]);
      qt[i] = F25519D::to_double(negate ? -t2d.l[i] : t2d.l[i]);
    }
    accd_to_doubles(x1, a.X);
    accd_to_doubles(y1, a.Y);
    accd_to_doubles(z1, a.Z);
    accd_to_doubles(t1, a.T);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      t0[i] = y1[i] - x1[i];
      s1[i] = y1[i] + x1[i];
    }
    FeD A, B, C, D;
    F25519D::mul(A, t0, qm);
    F25519D::mul(B, s1, qp);
    F25519D::mul(C, t1, qt);
    F25519D::mul(D, z1, qz);
    double da[5], db[5], dc[5], dd[5], e[5], f[5], gg[5], h[5];
    accd_to_doubles(da, A);
    accd_to_doubles(db, B);
    accd_to_doubles(dc, C);
    accd_to_doubles(dd, D);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      e[i] = db[i] - da[i];
      f[i] = dd[i] - dc[i];
      gg[i] = dd[i] + dc[i];
      h[i] = db[i] + da[i];
    }
    F25519D::mul(a.X, e, f);
    F25519D::mul(a.Y, gg, h);
    F25519D::mul(a.T, e, h);
    F25519D::mul(a.Z, f, gg);
  }
static B200_HD void accd_to_point(Ed25519::Point& p, const AccD& a) {
    F25519D::to_fe(p.X, a.X);
    F25519D::to_fe(p.Y, a.Y);
    F25519D::to_fe(p.Z, a.Z);
    F25519D::to_fe(p.T, a.T);
  }

  // x = s ? -x : x over N limbs (two's complement); returns the carry out of the negation chain
  // (1 only for s = 1, x = 0)
template <int N> static B200_HD u32 cond_negate(u32* x, u32 s) {
    const u32 mask = 0u - s;
#pragma unroll
    for (int i = 0; i < N; ++i)
      x[i] ^= mask;
    x[0] = add_cc(x[0], s);
#pragma unroll
    for (int i = 1; i < N; ++i)
      x[i] = addc_cc(x[i], 0u);
    return addc(0u, 0u);
  }
  // E + (O << 32) of a 4x4-limb mul_wide_eo product -> 8 plain limbs
static B200_HD void merge_eo8(u32* z, const u32* Ev, const u32* Ov) {
    z[0] = Ev[0];
    z[1] = add_cc(Ev[1], Ov[0]);
#pragma unroll
    for (int k = 2; k < 7; ++k)
      z[k] = addc_cc(Ev[k], Ov[k - 1]);
    z[7] = addc(Ev[7], Ov[6]);
  }
  // One level of subtractive Karatsuba: 3 x 16 wide multiply-adds instead of 64, paid for with
  // ~90 additions / logic ops on the ALU pipe (the multiplier pipe is the kernel's bound).
  //   a*b = z0 + 2^128 (z0 + z2 + (a0-a1)(b1-b0)) + 2^256 z2
static B200_HD void mul_kara(F25519::E& r, const F25519::E& a, const F25519::E& b) {
    u32 Ev[8], Ov[8], z0[8], z2[8], m[8], da[4], db[4];
    mul_wide_eo<4>(Ev, Ov, a.l, b.l);
    merge_eo8(z0, Ev, Ov);
    mul_wide_eo<4>(Ev, Ov, a.l + 4, b.l + 4);
    merge_eo8(z2, Ev, Ov);
    const u32 sa = limbs_sub<4>(da, a.l, a.l + 4);  // a0 - a1
    const u32 sb = limbs_sub<4>(db, b.l + 4, b.l);  // b1 - b0
    cond_negate<4>(da, sa);
    cond_negate<4>(db, sb);
    mul_wide_eo<4>(Ev, Ov, da, db);
    merge_eo8(m, Ev, Ov);
    // t + top*2^256 = z0 + z2 +- m
    const u32 s = sa ^ sb;
    u32 t[8];
    const u32 c1 = limbs_add<8>(t, z0, z2);
    const u32 c3 = cond_negate<8>(m, s);
    const u32 c2 = limbs_add<8>(t, t, m);
    const u32 top = c1 + c2 + c3 - s;
    u32 R[16];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      R[k] = z0[k];
    R[4] = add_cc(z0[4], t[0]);
#pragma unroll
    for (int k = 1; k < 4; ++k)
      R[4 + k] = addc_cc(z0[4 + k], t[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      R[8 + k] = addc_cc(z2[k], t[4 + k]);
    R[12] = addc_cc(z2[4], top);
    R[13] = addc_cc(z2[5], 0u);
    R[14] = addc_cc(z2[6], 0u);
    R[15] = addc(z2[7], 0u);
    F25519::fold_cc(r, R);
  }

}  // namespace rejected
}  // namespace b200
