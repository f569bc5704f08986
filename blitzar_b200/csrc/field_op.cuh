// Element-wise field arithmetic for the tests (b200_field_op; the CPU emulation's emul_field_op runs
// the same bodies with emulated carries): one operation of field.cuh / lanefield.cuh per element,
// operands and results as little-endian u32 limbs. Each curve unit instantiates its own base field;
// curve_ed25519.cu also the scalars mod l and the lane-sliced field.
#pragma once
#include <type_traits>

#include "curve.cuh"
#include "engine_api.cuh"
#include "lanefield.cuh"

namespace b200 {

// operation codes of b200_field_op (include/blitzar_b200.h lists which field offers which)
enum : u32 {
  kOpAdd, kOpSub, kOpNeg, kOpDbl, kOpMul, kOpMulRef, kOpSqr,         // every field (lane: add, mul)
  kOpMulLat, kOpCanonical, kOpIsNegative, kOpInvert, kOpPow22523,    // F25519 (invert: Mont too,
  kOpFromRadix51, kOpToRadix51, kOpSqrtRatioM1,                      // pow22523: lane too)
  kOpInvertEea, kOpFromMont, kOpToMont, kOpLexLargest,               // Montgomery fields
  kOpCarry1, kOpSub2p, kOpSub4p, kOpSlice, kOpGather,                // lane-sliced F25519
  kOpFrobenius, kOpCyclotomicSqr, kOpFinalExp,                       // Fp12 (pairing.cuh)
  kOpSqrt,                                                           // bls12-381 Fp, Fp2 (points.cuh)
};

// u32 limbs per element of operand a, operand b (0 = unary) and the result; out = 0: not offered
struct FieldOpShape {
  u32 a, b, out;
};

template <class F> B200_HD FieldOpShape field_op_shape(u32 op) {
  constexpr u32 N = F::N;
  const FieldOpShape unary{N, 0, N}, binary{N, N, N}, none{0, 0, 0};
  switch (op) {
  case kOpAdd: case kOpSub: case kOpMul: case kOpMulRef: return binary;
  case kOpNeg: case kOpDbl: case kOpSqr: case kOpInvert: return unary;
  default: break;
  }
  if (std::is_same<F, F25519>::value) {
    switch (op) {
    case kOpMulLat: return binary;
    case kOpCanonical: case kOpPow22523: return unary;
    case kOpIsNegative: return FieldOpShape{N, 0, 1};
    case kOpFromRadix51: return FieldOpShape{10, 0, N};  // 5 x u64
    case kOpToRadix51: return FieldOpShape{N, 0, 10};
    case kOpSqrtRatioM1: return FieldOpShape{N, N, N + 1};  // x, then the was-square flag
    default: return none;
    }
  }
  switch (op) {
  case kOpInvertEea: case kOpFromMont: case kOpToMont: return unary;
  case kOpLexLargest: return FieldOpShape{N, 0, 1};
  default: return none;
  }
}

template <class F> struct FieldOpBody {
  static constexpr int kBlock = 128;
  typedef typename F::E E;
  u32 op;
  FieldOpShape w;
  const u32* a;
  const u32* b;
  u32* out;

  // the operations only F25519 has
  static B200_HD void plain_op(u32 op, u32* o, const E& x, const E& y, const u32* pa) {
    if constexpr (std::is_same<F, F25519>::value) {
      E r;
      switch (op) {
      case kOpMulLat: F::mul_lat(r, x, y); break;
      case kOpCanonical: F::canonical(r, x); break;
      case kOpPow22523: F::pow22523(r, x); break;
      case kOpIsNegative: o[0] = F::is_negative(x) ? 1u : 0u; return;
      case kOpFromRadix51: {
        u64 h[5];
        for (int i = 0; i < 5; ++i)
          h[i] = (u64)pa[2 * i] | ((u64)pa[2 * i + 1] << 32);
        F::from_radix51(r, h);
        break;
      }
      case kOpToRadix51: {
        u64 h[5];
        F::to_radix51(h, x);
        for (int i = 0; i < 5; ++i) {
          o[2 * i] = (u32)h[i];
          o[2 * i + 1] = (u32)(h[i] >> 32);
        }
        return;
      }
      default:  // kOpSqrtRatioM1
        o[F::N] = (u32)Ed25519::sqrt_ratio_m1(r, x, y);
        break;
      }
      for (int i = 0; i < F::N; ++i)
        o[i] = r.l[i];
    }
  }
  // the operations only the Montgomery fields have
  static B200_HD void mont_op(u32 op, u32* o, const E& x) {
    if constexpr (!std::is_same<F, F25519>::value) {
      E r;
      switch (op) {
      case kOpInvertEea: F::invert_eea(r, x); break;
      case kOpFromMont: F::from_mont(r, x); break;
      case kOpToMont: F::to_mont(r, x); break;
      default: o[0] = F::lexicographically_largest(x) ? 1u : 0u; return;  // kOpLexLargest
      }
      for (int i = 0; i < F::N; ++i)
        o[i] = r.l[i];
    }
  }

  B200_HD void operator()(u64 i) const {
    const u32* pa = a + i * w.a;
    const u32* pb = b + i * w.b;
    u32* o = out + i * w.out;
    E x, y, r;
    for (int k = 0; k < F::N; ++k) {
      x.l[k] = pa[k];
      y.l[k] = w.b ? pb[k] : 0u;
    }
    switch (op) {
    case kOpAdd: F::add(r, x, y); break;
    case kOpSub: F::sub(r, x, y); break;
    case kOpNeg: F::neg(r, x); break;
    case kOpDbl: F::dbl(r, x); break;
    case kOpMul: F::mul(r, x, y); break;
    case kOpMulRef: F::mul_ref(r, x, y); break;
    case kOpSqr: F::sqr(r, x); break;
    case kOpInvert: F::invert(r, x); break;
    default:
      if (std::is_same<F, F25519>::value)
        plain_op(op, o, x, y, pa);
      else
        mont_op(op, o, x);
      return;
    }
    for (int k = 0; k < F::N; ++k)
      o[k] = r.l[k];
  }
};

// copies the operands to the device, runs `threads` threads of body (which reads operands and writes
// results at body.a, body.b, body.out) and copies n results back; synchronises
template <class Body>
unsigned run_elementwise(const EngineCtx& ctx, Body body, u64 n, u64 threads, const u32* a,
                         const u32* b, u32* out) {
  if (!body.w.out)
    return ~0u;
  const FieldOpShape w = body.w;
  DevBuf<u32> da(n * w.a, ctx.s), db(n * w.b, ctx.s), dout(n * w.out, ctx.s);
  copy_h2d(da.p, a, n * w.a * sizeof(u32), ctx.s);
  if (w.b)
    copy_h2d(db.p, b, n * w.b * sizeof(u32), ctx.s);
  body.a = da.p;
  body.b = db.p;
  body.out = dout.p;
  launch(body, threads, ctx.s);
  copy_d2h(out, dout.p, n * w.out * sizeof(u32), ctx.s);
  stream_sync(ctx.s);
  return 0;
}

template <class F>
unsigned run_field_op(const EngineCtx& ctx, u32 op, u64 n, const u32* a, const u32* b, u32* out) {
  return run_elementwise(ctx, FieldOpBody<F>{op, field_op_shape<F>(op), a, b, out}, n, n, a, b,
                         out);
}

#ifdef B200_LANE_TAIL
// lane-sliced F25519: one element per group of 10 lanes (three per warp), limb m in lane 10 g + m.
// Operands and results are the 10 radix-2^25.5 limbs, except slice's operand and gather's result (8
// x 32-bit limbs). Every lane reaches every shuffle: lanes without an element compute on zeros.
struct LaneFieldOpBody {
  static constexpr int kBlock = 32;
  u32 op;
  FieldOpShape w;
  u64 n;
  const u32* a;
  const u32* b;
  u32* out;

  static B200_HD FieldOpShape shape(u32 op) {
    switch (op) {
    case kOpAdd: case kOpMul: case kOpSub2p: case kOpSub4p: return FieldOpShape{10, 10, 10};
    case kOpCarry1: case kOpPow22523: return FieldOpShape{10, 0, 10};
    case kOpSlice: return FieldOpShape{8, 0, 10};
    case kOpGather: return FieldOpShape{10, 0, 8};
    default: return FieldOpShape{0, 0, 0};
    }
  }
  __device__ void operator()(u64 tid) const {
    using namespace lane10;
    const Lane L = lane_info();
    const u32 g = L.base / 10u, gg = g < 3 ? g : 0u;
    const u64 e = (tid >> 5) * 3 + g;
    const bool live = g < 3 && e < n;
    const u32 va = live && L.m < w.a ? a[e * w.a + L.m] : 0u;
    const u32 vb = live && w.b ? b[e * w.b + L.m] : 0u;
    u32 v = 0;
    switch (op) {
    case kOpAdd: v = add(va, vb); break;
    case kOpMul: v = mul(L, va, vb); break;
    case kOpSub2p: v = sub2p(L, va, vb); break;
    case kOpSub4p: v = sub4p(L, va, vb); break;
    case kOpCarry1: v = carry1(L, va); break;
    case kOpPow22523: v = pow22523(L, va); break;
    case kOpSlice: {
      F25519::E x;
      for (int k = 0; k < 8; ++k)
        x.l[k] = live ? a[e * 8 + k] : 0u;
      v = slice(L, x);
      break;
    }
    default: {  // kOpGather
      F25519::E x;
      gather(x, va, gg);
      if (live && L.m == 0)
        for (int k = 0; k < 8; ++k)
          out[e * 8 + k] = x.l[k];
      return;
    }
    }
    if (live)
      out[e * 10 + L.m] = v;
  }
};
#endif

}  // namespace b200
