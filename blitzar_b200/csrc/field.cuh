// Prime-field arithmetic on 32-bit limbs for the four curves of the MSM hot path.
//
// Replaces (re-derived, not translated): sxt/field51/operation/{mul,sq,add,sub}.cc (radix-2^51
// curve25519 field), sxt/field12 (bls12-381), sxt/field25 (bn254), sxt/fieldgk (grumpkin) and
// sxt/base/field/arithmetic_utility.h:39-75 (mac/adc/sbb helpers).
//
// Representation on device:
//   * F25519: 8 x u32, plain residue, kept only loosely reduced (any value < 2^256 that is
//     congruent mod p = 2^255-19); products fold with 2^256 = 38 (mod p).
//   * Mont<P>: N x u32 Montgomery residues with R = 2^(32N). Because R equals the reference's
//     R (2^256 resp. 2^384, 64-bit limbs), the reference's in-memory Montgomery limbs are
//     bit-identical to ours: u64[N/2] little-endian == u32[N].
//
// All functions are __host__ __device__ so the same code is exercised by the CPU-side emulation
// tests (tests/emul); device builds replace the inner loops by carry-chain PTX.
#pragma once
#include "constants.cuh"

#define B200_HD __host__ __device__ __forceinline__

namespace b200 {

template <int N> struct alignas(16) Fe {
  u32 l[N];
};


// ------------------------------------------------------------------------------------------------
// carry-flag primitives. Device: single PTX instructions chained through CC.CF (ptxas fuses a
// mad.lo.cc / madc.hi.cc pair on one register pair into IMAD.WIDE.U32[.X]). Host (emulation and
// the never-executed host half of __host__ __device__ bodies): the same semantics on an explicit
// carry variable, so the identical limb schedules can be verified on a CPU.
// ------------------------------------------------------------------------------------------------
#ifdef __CUDA_ARCH__
#define B200_CF_DECL
B200_HD u32 add_cc(u32 a, u32 b) { u32 r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 addc_cc(u32 a, u32 b) { u32 r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 addc(u32 a, u32 b) { u32 r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 sub_cc(u32 a, u32 b) { u32 r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 subc_cc(u32 a, u32 b) { u32 r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 subc(u32 a, u32 b) { u32 r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B200_HD u32 mad_lo_cc(u32 a, u32 b, u32 c) { u32 r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B200_HD u32 madc_lo_cc(u32 a, u32 b, u32 c) { u32 r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B200_HD u32 mad_hi_cc(u32 a, u32 b, u32 c) { u32 r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B200_HD u32 madc_hi_cc(u32 a, u32 b, u32 c) { u32 r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B200_HD u32 madc_hi(u32 a, u32 b, u32 c) { u32 r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#else
struct CarryFlag {
  static u32& cf() {
    static thread_local u32 v = 0;
    return v;
  }
};
inline u32 add_cc(u32 a, u32 b) { u64 t = (u64)a + b; CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 addc_cc(u32 a, u32 b) { u64 t = (u64)a + b + CarryFlag::cf(); CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 addc(u32 a, u32 b) { return a + b + CarryFlag::cf(); }
inline u32 sub_cc(u32 a, u32 b) { u64 t = (u64)a - b; CarryFlag::cf() = (u32)(t >> 63); return (u32)t; }
inline u32 subc_cc(u32 a, u32 b) { u64 t = (u64)a - b - CarryFlag::cf(); CarryFlag::cf() = (u32)(t >> 63); return (u32)t; }
inline u32 subc(u32 a, u32 b) { return a - b - CarryFlag::cf(); }
inline u32 mad_lo_cc(u32 a, u32 b, u32 c) { u64 t = (u64)(u32)(a * b) + c; CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 madc_lo_cc(u32 a, u32 b, u32 c) { u64 t = (u64)(u32)(a * b) + c + CarryFlag::cf(); CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 mad_hi_cc(u32 a, u32 b, u32 c) { u64 t = (((u64)a * b) >> 32) + c; CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 madc_hi_cc(u32 a, u32 b, u32 c) { u64 t = (((u64)a * b) >> 32) + c + CarryFlag::cf(); CarryFlag::cf() = (u32)(t >> 32); return (u32)t; }
inline u32 madc_hi(u32 a, u32 b, u32 c) { return (u32)(((u64)a * b) >> 32) + c + CarryFlag::cf(); }
#endif

// acc[0..2*NP) += (x[0], x[2], x[4], ...)(NP limbs taken with stride 2) * y as NP non-overlapping
// 64-bit products on the register pairs (acc[0],acc[1]), (acc[2],acc[3]), ... — one carry chain.
// Leaves the carry-out in CC.CF. `first` = no incoming carry (starts the chain).
template <int NP, class XS> B200_HD void chain_mad_pairs(u32* acc, XS x, u32 y) {
  acc[0] = mad_lo_cc(x(0), y, acc[0]);
  acc[1] = madc_hi_cc(x(0), y, acc[1]);
#pragma unroll
  for (int k = 1; k < NP; ++k) {
    acc[2 * k] = madc_lo_cc(x(k), y, acc[2 * k]);
    acc[2 * k + 1] = madc_hi_cc(x(k), y, acc[2 * k + 1]);
  }
}
// same, but the chain starts by consuming the carry already in CC.CF
template <int NP, class XS> B200_HD void chain_madc_pairs(u32* acc, XS x, u32 y) {
#pragma unroll
  for (int k = 0; k < NP; ++k) {
    acc[2 * k] = madc_lo_cc(x(k), y, acc[2 * k]);
    acc[2 * k + 1] = madc_hi_cc(x(k), y, acc[2 * k + 1]);
  }
}

// 2N-limb product in even/odd form: E + (O << 32) = a * b, E[0..2N), O[0..2N-1) (O[k] sits at limb
// position k+1). Every mad pair lands on an even-aligned register pair of E or O.
template <int N> B200_HD void mul_wide_eo(u32* E, u32* O, const u32* a, const u32* b) {
#pragma unroll
  for (int i = 0; i < 2 * N; ++i) {
    E[i] = 0;
    O[i] = 0;
  }
#pragma unroll
  for (int i = 0; i < N; i += 2) {
    // row i (even): a_even*b[i] -> E[i..], a_odd*b[i] -> O[i..]
    chain_mad_pairs<N / 2>(E + i, [a](int k) { return a[2 * k]; }, b[i]);
    E[i + N] = addc(E[i + N], 0);
    chain_mad_pairs<N / 2>(O + i, [a](int k) { return a[2 * k + 1]; }, b[i]);
    O[i + N] = addc(O[i + N], 0);
    // row i+1 (odd): a_even*b[i+1] sits at odd positions -> O[i..], a_odd*b[i+1] -> E[i+2..]
    chain_mad_pairs<N / 2>(O + i, [a](int k) { return a[2 * k]; }, b[i + 1]);
    O[i + N] = addc(O[i + N], 0);
    chain_mad_pairs<N / 2>(E + i + 2, [a](int k) { return a[2 * k + 1]; }, b[i + 1]);
    if (i + 2 + N < 2 * N)
      E[i + 2 + N] = addc(E[i + 2 + N], 0);
  }
}

// ------------------------------------------------------------------------------------------------
// multi-limb add / sub
// ------------------------------------------------------------------------------------------------
template <int N> B200_HD u32 limbs_add(u32* r, const u32* a, const u32* b) {
#ifdef __CUDA_ARCH__
  asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int i = 1; i < N; ++i)
    asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r[i]) : "r"(a[i]), "r"(b[i]));
  u32 c;
  asm volatile("addc.u32 %0, 0, 0;" : "=r"(c));
  return c;
#else
  u64 c = 0;
  for (int i = 0; i < N; ++i) {
    c += (u64)a[i] + b[i];
    r[i] = (u32)c;
    c >>= 32;
  }
  return (u32)c;
#endif
}

// returns borrow (0 or 1)
template <int N> B200_HD u32 limbs_sub(u32* r, const u32* a, const u32* b) {
#ifdef __CUDA_ARCH__
  asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int i = 1; i < N; ++i)
    asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r[i]) : "r"(a[i]), "r"(b[i]));
  u32 bw;
  asm volatile("subc.u32 %0, 0, 0;" : "=r"(bw));
  return bw & 1u;
#else
  u64 bw = 0;
  for (int i = 0; i < N; ++i) {
    u64 t = (u64)a[i] - b[i] - bw;
    r[i] = (u32)t;
    bw = t >> 63;
  }
  return (u32)bw;
#endif
}

// r = a + k (small), returns carry: one add.cc chain on the device (the host runs the same schedule
// on the emulated carry)
template <int N> B200_HD u32 limbs_add_small(u32* r, const u32* a, u32 k) {
  r[0] = add_cc(a[0], k);
#pragma unroll
  for (int i = 1; i < N; ++i)
    r[i] = addc_cc(a[i], 0u);
  return addc(0u, 0u);
}

// r = a - k (small), returns borrow (0 or 1): one sub.cc chain
template <int N> B200_HD u32 limbs_sub_small(u32* r, const u32* a, u32 k) {
  r[0] = sub_cc(a[0], k);
#pragma unroll
  for (int i = 1; i < N; ++i)
    r[i] = subc_cc(a[i], 0u);
  return subc(0u, 0u) & 1u;
}

template <int N> B200_HD bool limbs_is_zero(const u32* a) {
  u32 x = 0;
#pragma unroll
  for (int i = 0; i < N; ++i)
    x |= a[i];
  return x == 0;
}

// schoolbook product t[2N] = a * b
template <int N> B200_HD void limbs_mul_wide(u32* t, const u32* a, const u32* b) {
#pragma unroll
  for (int i = 0; i < 2 * N; ++i)
    t[i] = 0;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    u64 c = 0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      c += (u64)a[j] * b[i] + t[i + j];
      t[i + j] = (u32)c;
      c >>= 32;
    }
    t[i + N] = (u32)c;
  }
}

// ------------------------------------------------------------------------------------------------
// F25519: GF(2^255-19), loosely reduced 8-limb residues
// ------------------------------------------------------------------------------------------------
struct F25519 {
  static constexpr int N = 8;
  typedef Fe<8> E;

  static B200_HD E zero() {
    E r;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r.l[i] = 0;
    return r;
  }
  static B200_HD E one() {
    E r = zero();
    r.l[0] = 1;
    return r;
  }
  template <class C> static B200_HD E constant(C c) {
    E r;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r.l[i] = c(i);
    return r;
  }

  static B200_HD void add(E& r, const E& a, const E& b) {
    u32 c = limbs_add<8>(r.l, a.l, b.l);
    c = limbs_add_small<8>(r.l, r.l, 38u * c);
    r.l[0] += 38u * c;  // after a second wrap the value is < 38, so this cannot carry
  }
  static B200_HD void sub(E& r, const E& a, const E& b) {
    u32 bw = limbs_sub<8>(r.l, a.l, b.l);
    bw = limbs_sub_small<8>(r.l, r.l, 38u * bw);
    r.l[0] -= 38u * bw;  // after a second wrap the value is >= 2^256-38, so this cannot borrow
  }
  static B200_HD void neg(E& r, const E& a) {
    E z = zero();
    sub(r, z, a);
  }
  static B200_HD void dbl(E& r, const E& a) { add(r, a, a); }

  // reference schedule (plain 64-bit C): r = a*b, 16-limb product folded twice with 2^256 = 38
  static B200_HD void mul_ref(E& r, const E& a, const E& b) {
    u32 t[16];
    limbs_mul_wide<8>(t, a.l, b.l);
    fold(r, t);
  }
  // production schedule: 64 wide multiply-adds on even/odd register pairs (mul_wide_eo), one
  // merge chain, then the 2^256 = 38 fold as 8 more wide multiply-adds and a merge (fold_cc).
  static B200_HD void mul(E& r, const E& a, const E& b) { mul_school(r, a, b); }
  static B200_HD void mul_school(E& r, const E& a, const E& b) {
    u32 Ev[16], Ov[16], R[16];
    mul_wide_eo<8>(Ev, Ov, a.l, b.l);
    R[0] = Ev[0];
    R[1] = add_cc(Ev[1], Ov[0]);
#pragma unroll
    for (int k = 2; k < 16; ++k)
      R[k] = addc_cc(Ev[k], Ov[k - 1]);
    fold_cc(r, R);
  }
  // 16-limb product -> loosely reduced residue, carry-chain form of fold() with the same result.
  // The eight products 38 h[k] of the high half h = R[8..16) are 64-bit multiply-adds on register
  // pairs: even k into (t[k], t[k+1]) on top of R_lo, odd k into a second set of pairs, which one
  // add chain then merges.
  static B200_HD void fold_cc(E& r, const u32* R) {
    const u32* h = R + 8;
    u32 t[8], u[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
      t[k] = R[k];
    chain_mad_pairs<4>(t, [h](int k) { return h[2 * k]; }, 38u);
    u32 top = addc(0u, 0u);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      u[k] = 0;
    chain_mad_pairs<4>(u, [h](int k) { return h[2 * k + 1]; }, 38u);  // u[k] sits at limb k+1
    t[1] = add_cc(t[1], u[0]);
#pragma unroll
    for (int k = 2; k < 8; ++k)
      t[k] = addc_cc(t[k], u[k - 1]);
    top = addc(top, u[7]);  // (R_lo + 38 h) >> 256 <= 38
    r.l[0] = mad_lo_cc(top, 38u, t[0]);
#pragma unroll
    for (int k = 1; k < 8; ++k)
      r.l[k] = addc_cc(t[k], 0u);
    u32 c2 = addc(0u, 0u);
    r.l[0] += 38u * c2;  // a wrap leaves a value < 2^11, so this cannot carry
  }

  static B200_HD void sqr(E& r, const E& a) { mul(r, a, a); }

  // latency-oriented schedule for the serial tail kernels (QuadExec): product scanning — the 15
  // column sums are independent 96-bit accumulations, so one warp can overlap them; more
  // instructions than mul() but a much shorter dependent chain.
  static B200_HD void mul_lat(E& r, const E& a, const E& b) {
    u64 lo[16];
    u32 hi[16];
#pragma unroll
    for (int k = 0; k < 15; ++k) {
      u64 acc = 0;
      u32 c = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int j = k - i;
        if (j >= 0 && j < 8) {
          u64 p = (u64)a.l[i] * b.l[j];
          acc += p;
          c += acc < p ? 1u : 0u;
        }
      }
      lo[k] = acc;
      hi[k] = c;
    }
    // column k contributes lo32 to limb k, hi32 to limb k+1 and its overflow count to limb k+2
    u32 t[16];
    u64 carry = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      u64 v = carry;
      if (k < 15)
        v += (u32)lo[k];
      if (k >= 1)
        v += (u32)(lo[k - 1] >> 32);
      if (k >= 2)
        v += hi[k - 2];
      t[k] = (u32)v;
      carry = v >> 32;
    }
    fold(r, t);
  }

  static B200_HD void fold(E& r, const u32* t) {
    u64 c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      c += (u64)t[i + 8] * 38u + t[i];
      r.l[i] = (u32)c;
      c >>= 32;
    }
    // c < 39; fold the ninth limb
    u32 c2 = limbs_add_small<8>(r.l, r.l, (u32)c * 38u);
    r.l[0] += 38u * c2;
  }

  // canonical representative in [0, p)
  static B200_HD void canonical(E& r, const E& a) {
    E v = a;
    u32 top = v.l[7] >> 31;
    v.l[7] &= 0x7fffffffu;
    limbs_add_small<8>(v.l, v.l, 19u * top);  // < 2^255 + 19
    E t;
    limbs_add_small<8>(t.l, v.l, 19u);  // v + 19 >= 2^255  <=>  v >= p
    u32 ge = t.l[7] >> 31;
    t.l[7] &= 0x7fffffffu;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r.l[i] = ge ? t.l[i] : v.l[i];
  }
  static B200_HD bool is_zero(const E& a) {
    E c;
    canonical(c, a);
    return limbs_is_zero<8>(c.l);
  }
  static B200_HD bool is_negative(const E& a) {  // f51p::is_negative: lsb of canonical form
    E c;
    canonical(c, a);
    return c.l[0] & 1u;
  }
  static B200_HD bool equal(const E& a, const E& b) {
    E d;
    sub(d, a, b);
    return is_zero(d);
  }
  static B200_HD void select(E& r, const E& a, const E& b, bool pick_b) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r.l[i] = pick_b ? b.l[i] : a.l[i];
  }
  static B200_HD void abs(E& r, const E& a) {
    E n;
    neg(n, a);
    select(r, a, n, is_negative(a));
  }

  // a^e for a public exponent given as 8 limbs
  template <class C> static B200_HD void pow(E& r, const E& a, C expo) {
    E acc = one();
    for (int i = 255; i >= 0; --i) {
      sqr(acc, acc);
      if ((expo(i >> 5) >> (i & 31)) & 1u)
        mul(acc, acc, a);
    }
    r = acc;
  }
  struct ExpPm2 {
    B200_HD u32 operator()(int i) const { return i == 0 ? 0xffffffebu : (i == 7 ? 0x7fffffffu : 0xffffffffu); }
  };
  struct ExpP58 {  // (p-5)/8 = 2^252 - 3
    B200_HD u32 operator()(int i) const { return i == 0 ? 0xfffffffdu : (i == 7 ? 0x0fffffffu : 0xffffffffu); }
  };
  static B200_HD void sqr_n(E& r, const E& a, int n) {
    r = a;
    for (int i = 0; i < n; ++i)
      sqr(r, r);
  }
  // a^(2^250 - 1), the shared prefix of the two fixed exponents (standard 2^k-1 ladder)
  static B200_HD void pow_2_250_m1(E& r, E& a11, const E& a) {
    E t0, t1, t2, t3;
    sqr(t0, a);             // 2
    sqr_n(t1, t0, 2);       // 8
    mul(t1, a, t1);         // 9
    mul(t0, t0, t1);        // 11
    a11 = t0;
    sqr(t2, t0);            // 22
    mul(t1, t1, t2);        // 31 = 2^5 - 1
    sqr_n(t2, t1, 5);
    mul(t1, t2, t1);        // 2^10 - 1
    sqr_n(t2, t1, 10);
    mul(t2, t2, t1);        // 2^20 - 1
    sqr_n(t3, t2, 20);
    mul(t2, t3, t2);        // 2^40 - 1
    sqr_n(t2, t2, 10);
    mul(t1, t2, t1);        // 2^50 - 1
    sqr_n(t2, t1, 50);
    mul(t2, t2, t1);        // 2^100 - 1
    sqr_n(t3, t2, 100);
    mul(t2, t3, t2);        // 2^200 - 1
    sqr_n(t2, t2, 50);
    mul(r, t2, t1);         // 2^250 - 1
  }
  // a^(p-2) = a^(2^255 - 21): (2^250-1) << 5 | 11
  static B200_HD void invert(E& r, const E& a) {
    E t, a11;
    pow_2_250_m1(t, a11, a);
    sqr_n(t, t, 5);
    mul(r, t, a11);
  }
  // the name the top of the batch-inversion tree calls (batch_affine.cuh); here the Fermat ladder
  static B200_HD void invert_eea(E& r, const E& a) { invert(r, a); }
  // a^((p-5)/8) = a^(2^252 - 3): (2^250-1) << 2 | 1
  static B200_HD void pow22523(E& r, const E& a) {
    E t, a11;
    pow_2_250_m1(t, a11, a);
    sqr_n(t, t, 2);
    mul(r, t, a);
  }

  // radix-2^51 limbs (sxt_ristretto255 / c21t::element_p3 field layout; limbs may be unreduced)
  static B200_HD void from_radix51(E& r, const u64* h) {
    u32 acc[10];
#pragma unroll
    for (int i = 0; i < 10; ++i)
      acc[i] = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int o = 51 * i, w = o >> 5, s = o & 31;
      u32 p0 = (u32)(h[i] << s);
      u32 p1 = (u32)((h[i] >> (32 - s)));
      u32 p2 = s ? (u32)(h[i] >> (64 - s)) : 0u;
      if (s == 0) {
        p0 = (u32)h[i];
        p1 = (u32)(h[i] >> 32);
      }
      u64 c = (u64)acc[w] + p0;
      acc[w] = (u32)c;
      c >>= 32;
      c += (u64)acc[w + 1] + p1;
      acc[w + 1] = (u32)c;
      c >>= 32;
      c += (u64)acc[w + 2] + p2;
      acc[w + 2] = (u32)c;
      c >>= 32;
#pragma unroll
      for (int k = w + 3; k < 10; ++k) {
        c += acc[k];
        acc[k] = (u32)c;
        c >>= 32;
      }
    }
    // value < 2^269: fold limbs 8,9 with 2^256 = 38
    u64 c = 0;
    u32 hi[8] = {acc[8], acc[9], 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      c += (u64)hi[i] * 38u + acc[i];
      r.l[i] = (u32)c;
      c >>= 32;
    }
    u32 c2 = limbs_add_small<8>(r.l, r.l, (u32)c * 38u);
    r.l[0] += 38u * c2;
  }
  static B200_HD void to_radix51(u64* h, const E& a) {
    E c;
    canonical(c, a);
    u64 w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      w[i] = (u64)c.l[2 * i] | ((u64)c.l[2 * i + 1] << 32);
    const u64 m = 0x7ffffffffffffULL;
    h[0] = w[0] & m;
    h[1] = ((w[0] >> 51) | (w[1] << 13)) & m;
    h[2] = ((w[1] >> 38) | (w[2] << 26)) & m;
    h[3] = ((w[2] >> 25) | (w[3] << 39)) & m;
    h[4] = (w[3] >> 12) & m;
  }
  // 32 little-endian bytes, top bit ignored (f51b::from_bytes semantics)
  static B200_HD void from_bytes(E& r, const unsigned char* s) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r.l[i] = (u32)s[4 * i] | ((u32)s[4 * i + 1] << 8) | ((u32)s[4 * i + 2] << 16) |
               ((u32)s[4 * i + 3] << 24);
    r.l[7] &= 0x7fffffffu;
  }
  static B200_HD void to_bytes(unsigned char* s, const E& a) {
    E c;
    canonical(c, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[4 * i] = (unsigned char)c.l[i];
      s[4 * i + 1] = (unsigned char)(c.l[i] >> 8);
      s[4 * i + 2] = (unsigned char)(c.l[i] >> 16);
      s[4 * i + 3] = (unsigned char)(c.l[i] >> 24);
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Mont<P>: Montgomery residues, fully reduced. P supplies N, p(i), one(i), r2(i), inv.
// ------------------------------------------------------------------------------------------------
template <class P> struct Mont {
  typedef P Params;
  static constexpr int N = P::N;
  typedef Fe<N> E;

  static B200_HD E zero() {
    E r;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = 0;
    return r;
  }
  static B200_HD E one() {
    E r;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = P::one(i);
    return r;
  }
  static B200_HD E modulus() {
    E r;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = P::p(i);
    return r;
  }
  template <class C> static B200_HD E constant(C c) {
    E r;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = c(i);
    return r;
  }

  // all moduli leave >= 2 spare bits in N limbs, so a+b never carries out
  static B200_HD void add(E& r, const E& a, const E& b) {
    E s, d, p = modulus();
    limbs_add<N>(s.l, a.l, b.l);
    u32 bw = limbs_sub<N>(d.l, s.l, p.l);
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = bw ? s.l[i] : d.l[i];
  }
  static B200_HD void sub(E& r, const E& a, const E& b) {
    E d, e, p = modulus();
    u32 bw = limbs_sub<N>(d.l, a.l, b.l);
    limbs_add<N>(e.l, d.l, p.l);
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = bw ? e.l[i] : d.l[i];
  }
  static B200_HD void neg(E& r, const E& a) {
    E z = zero();
    sub(r, z, a);
  }
  static B200_HD void dbl(E& r, const E& a) { add(r, a, a); }
  static B200_HD bool is_zero(const E& a) { return limbs_is_zero<N>(a.l); }
  static B200_HD bool equal(const E& a, const E& b) {
    u32 x = 0;
#pragma unroll
    for (int i = 0; i < N; ++i)
      x |= a.l[i] ^ b.l[i];
    return x == 0;
  }
  static B200_HD void select(E& r, const E& a, const E& b, bool pick_b) {
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = pick_b ? b.l[i] : a.l[i];
  }

  // production schedule: CIOS Montgomery product on even/odd accumulators. Two limbs of b are
  // consumed per frame (offsets 0 and 1) so that every multiply-add lands on an even-aligned
  // register pair of Ev (limb positions k) or Ov (limb positions k+1); the frame then moves down
  // by two limbs (register renaming). What the move cannot rename — Ov[1], which sits on the new
  // position 0, and the carry bit out of the two zeroed limbs — is added to the new Ev by one
  // N+1-instruction carry chain per frame.
  // Operands: a < p, b < R (b need not be reduced). The frame holds N + 2 limbs, enough for
  // t + a (b_i + 2^32 b_i+1) + p (m0 + 2^32 m1) with a < p; an a up to R would need one more, and
  // its carry out of the top limb would be lost.
  static B200_HD void mul(E& r, const E& a, const E& b) {
    u32 Ev[N + 2], Ov[N + 2];
#pragma unroll
    for (int k = 0; k < N + 2; ++k) {
      Ev[k] = 0;
      Ov[k] = 0;
    }
    const u32* al = a.l;
    auto a_even = [al](int k) { return al[2 * k]; };
    auto a_odd = [al](int k) { return al[2 * k + 1]; };
    auto p_even = [](int k) { return P::p(2 * k); };
    auto p_odd = [](int k) { return P::p(2 * k + 1); };
#pragma unroll
    for (int i = 0; i < N; i += 2) {
      // ---- round A: b[i] at frame offset 0
      chain_mad_pairs<N / 2>(Ev, a_even, b.l[i]);
      Ev[N] = addc_cc(Ev[N], 0u);
      Ev[N + 1] = addc(Ev[N + 1], 0u);
      chain_mad_pairs<N / 2>(Ov, a_odd, b.l[i]);
      Ov[N] = addc(Ov[N], 0u);
      u32 m0 = Ev[0] * P::inv;
      chain_mad_pairs<N / 2>(Ev, p_even, m0);
      Ev[N] = addc_cc(Ev[N], 0u);
      Ev[N + 1] = addc(Ev[N + 1], 0u);
      chain_mad_pairs<N / 2>(Ov, p_odd, m0);
      Ov[N] = addc(Ov[N], 0u);
      // ---- round B: b[i+1] at frame offset 1
      chain_mad_pairs<N / 2>(Ov, a_even, b.l[i + 1]);
      Ov[N] = addc(Ov[N], 0u);
      chain_mad_pairs<N / 2>(Ev + 2, a_odd, b.l[i + 1]);
      u32 m1 = (Ev[1] + Ov[0]) * P::inv;
      chain_mad_pairs<N / 2>(Ov, p_even, m1);
      Ov[N] = addc(Ov[N], 0u);
      chain_mad_pairs<N / 2>(Ev + 2, p_odd, m1);
      // ---- move the frame down two limbs: Ev'[k] = Ev[k+2] + (k == 0 ? Ov[1] + carry : 0)
      (void)add_cc(Ev[1], Ov[0]);  // the two dropped limbs sum to 0 mod 2^32; CF = their carry
      Ev[0] = addc_cc(Ev[2], Ov[1]);
#pragma unroll
      for (int k = 1; k < N; ++k)
        Ev[k] = addc_cc(Ev[k + 2], 0u);
      Ev[N] = 0;
      Ev[N + 1] = 0;
#pragma unroll
      for (int k = 0; k + 2 <= N; ++k)
        Ov[k] = Ov[k + 2];
      Ov[N - 1] = 0;
      Ov[N] = 0;
    }
    E s, d, p = modulus();
    s.l[0] = Ev[0];
    s.l[1] = add_cc(Ev[1], Ov[0]);
#pragma unroll
    for (int k = 2; k < N; ++k)
      s.l[k] = addc_cc(Ev[k], Ov[k - 1]);
    u32 bw = limbs_sub<N>(d.l, s.l, p.l);
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = bw ? s.l[i] : d.l[i];
  }
  static B200_HD void mul_lat(E& r, const E& a, const E& b) { mul(r, a, b); }
  // reference schedule (plain 64-bit C): CIOS Montgomery product r = a*b/R mod p
  static B200_HD void mul_ref(E& r, const E& a, const E& b) {
    u32 t[N + 2];
#pragma unroll
    for (int i = 0; i < N + 2; ++i)
      t[i] = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      u64 c = 0;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        c += (u64)a.l[j] * b.l[i] + t[j];
        t[j] = (u32)c;
        c >>= 32;
      }
      c += t[N];
      t[N] = (u32)c;
      t[N + 1] = (u32)(c >> 32);
      u32 m = t[0] * P::inv;
      c = ((u64)m * P::p(0) + t[0]) >> 32;
#pragma unroll
      for (int j = 1; j < N; ++j) {
        c += (u64)m * P::p(j) + t[j];
        t[j - 1] = (u32)c;
        c >>= 32;
      }
      c += t[N];
      t[N - 1] = (u32)c;
      t[N] = t[N + 1] + (u32)(c >> 32);
    }
    E s, d, p = modulus();
#pragma unroll
    for (int i = 0; i < N; ++i)
      s.l[i] = t[i];
    u32 bw = limbs_sub<N>(d.l, s.l, p.l);
    bool keep = bw && (t[N] == 0);
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = keep ? s.l[i] : d.l[i];
  }
  static B200_HD void sqr(E& r, const E& a) { mul(r, a, a); }

  template <class C> static B200_HD void pow(E& r, const E& a, C expo) {
    E acc = one();
    for (int i = 32 * N - 1; i >= 0; --i) {
      sqr(acc, acc);
      if ((expo(i >> 5) >> (i & 31)) & 1u)
        mul(acc, acc, a);
    }
    r = acc;
  }
  struct ExpPm2 {
    B200_HD u32 operator()(int i) const { return P::pm2(i); }
  };
  // r = 1/a (0 -> 0), Montgomery domain preserved
  static B200_HD void invert(E& r, const E& a) { pow(r, a, ExpPm2{}); }

  // r = 1/a (0 -> 0), Montgomery domain preserved, by the binary extended Euclidean algorithm: about
  // 2 * bits halving / subtraction steps of N-limb shifts and additions instead of the ~1.5 * bits field
  // multiplications of the Fermat power — an order of magnitude less latency for ONE dependent
  // inversion (the affine conversion of an output point, the top of a batch-inversion tree). Control
  // flow depends on the data, so the throughput kernels (one inversion per thread of a full grid) keep
  // invert().
  static B200_HD void invert_eea(E& r, const E& a) {
    if (is_zero(a)) {
      r = zero();
      return;
    }
    const E p = modulus();
    E u = a, v = p, b = zero(), c = zero();
    b.l[0] = 1u;
    // invariants: b * a == u, c * a == v (mod p); u, v odd after the halving loops
    for (;;) {
      while (!(u.l[0] & 1u)) {
        shr1(u, 0u);
        halve_mod(b, p);
      }
      if (is_plain_one(u))
        break;
      while (!(v.l[0] & 1u)) {
        shr1(v, 0u);
        halve_mod(c, p);
      }
      if (is_plain_one(v))
        break;
      E d;
      if (limbs_sub<N>(d.l, u.l, v.l) == 0) {  // u >= v
        u = d;
        sub(b, b, c);
      } else {
        limbs_sub<N>(v.l, v.l, u.l);
        sub(c, c, b);
      }
    }
    E y = is_plain_one(u) ? b : c;
    // y = (a R)^-1 = a^-1 R^-1 as a plain residue; two Montgomery products by R^2 give a^-1 R
    E r2;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r2.l[i] = P::r2(i);
    mul(y, y, r2);
    mul(r, y, r2);
  }
  static B200_HD bool is_plain_one(const E& x) {
    u32 t = x.l[0] ^ 1u;
#pragma unroll
    for (int i = 1; i < N; ++i)
      t |= x.l[i];
    return t == 0;
  }
  static B200_HD void shr1(E& x, u32 top_bit) {
#pragma unroll
    for (int i = 0; i < N - 1; ++i)
      x.l[i] = (x.l[i] >> 1) | (x.l[i + 1] << 31);
    x.l[N - 1] = (x.l[N - 1] >> 1) | (top_bit << 31);
  }
  // x / 2 mod p for x < p
  static B200_HD void halve_mod(E& x, const E& p) {
    if (x.l[0] & 1u) {
      E t;
      const u32 cy = limbs_add<N>(t.l, x.l, p.l);
      x = t;
      shr1(x, cy);
    } else {
      shr1(x, 0u);
    }
  }
  static B200_HD void from_mont(E& r, const E& a) {
    E o = zero();
    o.l[0] = 1;
    mul(r, a, o);
  }
  // any a < R (reduces a raw N-limb value): a R mod p
  static B200_HD void to_mont(E& r, const E& a) {
    E r2;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r2.l[i] = P::r2(i);
    mul(r, r2, a);
  }
  // f12p::lexicographically_largest: plain value > (p-1)/2
  static B200_HD bool lexicographically_largest(const E& a) {
    E v, h, d;
    from_mont(v, a);
#pragma unroll
    for (int i = 0; i < N; ++i)
      h.l[i] = P::half(i);
    u32 bw = limbs_sub<N>(d.l, h.l, v.l);  // borrow <=> v > half
    return bw != 0;
  }
  // reference memory layout: u64 limbs little-endian == u32 limbs
  static B200_HD void load(E& r, const void* src) {
    const u32* s = (const u32*)src;
#pragma unroll
    for (int i = 0; i < N; ++i)
      r.l[i] = s[i];
  }
  static B200_HD void store(void* dst, const E& a) {
    u32* d = (u32*)dst;
#pragma unroll
    for (int i = 0; i < N; ++i)
      d[i] = a.l[i];
  }
};

struct BnParams {
  static constexpr int N = 8;
  static constexpr u32 inv = BN_INV;
  static B200_HD u32 p(int i) { return BN_P(i); }
  static B200_HD u32 one(int i) { return BN_ONE(i); }
  static B200_HD u32 r2(int i) { return BN_R2(i); }
  static B200_HD u32 pm2(int i) { return BN_PM2(i); }
  static B200_HD u32 half(int i) { return BN_HALF(i); }
  static B200_HD u32 gx(int i) { return BN_GX(i); }
  static B200_HD u32 gy(int i) { return BN_GY(i); }
};
struct GkParams {
  static constexpr int N = 8;
  static constexpr u32 inv = GK_INV;
  static B200_HD u32 p(int i) { return GK_P(i); }
  static B200_HD u32 one(int i) { return GK_ONE(i); }
  static B200_HD u32 r2(int i) { return GK_R2(i); }
  static B200_HD u32 pm2(int i) { return GK_PM2(i); }
  static B200_HD u32 half(int i) { return GK_HALF(i); }
  static B200_HD u32 gx(int i) { return GK_GX(i); }
  static B200_HD u32 gy(int i) { return GK_GY(i); }
};
struct BlsParams {
  static constexpr int N = 12;
  static constexpr u32 inv = BLS_INV;
  static B200_HD u32 p(int i) { return BLS_P(i); }
  static B200_HD u32 one(int i) { return BLS_ONE(i); }
  static B200_HD u32 r2(int i) { return BLS_R2(i); }
  static B200_HD u32 pm2(int i) { return BLS_PM2(i); }
  static B200_HD u32 half(int i) { return BLS_HALF(i); }
  static B200_HD u32 gx(int i) { return BLS_GX(i); }
  static B200_HD u32 gy(int i) { return BLS_GY(i); }
};
// scalars modulo the ristretto255 group order l (inner-product argument; replaces the device half of
// sxt/scalar25/operation/{mul,muladd,add}.cc)
struct Sc25Params {
  static constexpr int N = 8;
  static constexpr u32 inv = SC25_INV;
  static B200_HD u32 p(int i) { return SC25_P(i); }
  static B200_HD u32 one(int i) { return SC25_ONE(i); }
  static B200_HD u32 r2(int i) { return SC25_R2(i); }
  static B200_HD u32 pm2(int i) { return SC25_PM2(i); }
  static B200_HD u32 half(int i) { return SC25_HALF(i); }
};
typedef Mont<Sc25Params> FSc25;
typedef Mont<BnParams> FBn;
typedef Mont<GkParams> FGk;
typedef Mont<BlsParams> FBls;

}  // namespace b200
