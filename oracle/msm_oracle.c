/* TEST INFRASTRUCTURE — CPU restatement ("port") of the reference's MSM / Pedersen-commitment path.
 *
 * Plain C (gcc, unsigned __int128). Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this; the product never does.
 *
 * Parity is PINNED: this file is checked (tests/test_oracle.py) against
 *   - the reference's own golden commitments (rust/tests/src/main.rs:30-49), and
 *   - the reference's own CPU implementation compiled from a reference checkout (oracle/_ref), on
 *     random inputs for all four curves, both APIs, and committed fixtures (tests/golden/).
 *
 * What is restated (reference file:line):
 *   field25519      radix-2^51 limbs, sxt/field51/operation/mul.cc:36-95, add.h:40-52, sub.cc:24-56,
 *                   base/reduce.cc:24-97, base/byte_conversion.cc:24-66
 *   Montgomery      u64 limbs, R = 2^(64 N): sxt/field12|field25|fieldgk/operation/mul.cc,
 *                   base/reduce.h:44-112, base/subtract_p.h, operation/add.h, sub.h, neg.h, invert.cc
 *   ed25519 group   extended coordinates: sxt/curve21/operation/add.cc:41-55 (+ add.h:39-80),
 *                   type/double_impl.cc:43-55, operation/neg.h
 *   Weierstrass     complete projective formulas, a = 0: sxt/curve_g1/operation/add.h:46-84,
 *                   double.cc:43-71 (curve_bng1 / curve_gk: same lines), mul_by_3b.h
 *   ristretto       encode: sxt/ristretto/base/byte_conversion.cc:74-129; sqrt_ratio_m1.cc:33-67;
 *                   elligator.cc:47-93; generator g(i): sxt/seqcommit/generator/base_element.cc:30-35,
 *                   sxt/base/num/fast_random_number_generator.h:27-50
 *   output forms    sxt/curve_g1/operation/compression.cc:34-62; curve_bng1/type/conversion_utility.h:38-60
 *   MSM             res[j] = sum_i int(s_ji) * G_i with the scalar semantics of
 *                   sxt/multiexp/base/exponent_sequence.h:25-42 (1..32-byte little-endian unsigned, or
 *                   two's-complement signed) — computed with the reference's bucket method shape
 *                   (c = 8 windows, 255 buckets per window, running-sum reduction, Horner over
 *                   windows: sxt/multiexp/bucket_method/accumulation_kernel.h:38-75,
 *                   combination_kernel.h:81-106, combination.h:28-62), serial on one core.
 *   fixed-base      row-major scalar table, packed and variable-length variants:
 *                   cbindings/blitzar_api.h:663-744, sxt/multiexp/pippenger2/reduce.h:37-47.
 *   inner product   prover / verifier, Merlin transcript and scalars mod l: see the banner above
 *                   oracle_prove_inner_product (bottom of this file).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef unsigned __int128 u128;

/* ================================================================================================
 * GF(2^255-19), five 51-bit limbs
 * ==============================================================================================*/
typedef struct { u64 v[5]; } fe;
#define MASK51 0x7ffffffffffffULL

static void fe_carry(fe* r, u128 t[5]) {
  u64 c;
  u64 r0, r1, r2, r3, r4;
  r0 = (u64)t[0] & MASK51; c = (u64)(t[0] >> 51);
  t[1] += c; r1 = (u64)t[1] & MASK51; c = (u64)(t[1] >> 51);
  t[2] += c; r2 = (u64)t[2] & MASK51; c = (u64)(t[2] >> 51);
  t[3] += c; r3 = (u64)t[3] & MASK51; c = (u64)(t[3] >> 51);
  t[4] += c; r4 = (u64)t[4] & MASK51; c = (u64)(t[4] >> 51);
  r0 += 19 * c; c = r0 >> 51; r0 &= MASK51;
  r1 += c; c = r1 >> 51; r1 &= MASK51;
  r2 += c;
  r->v[0] = r0; r->v[1] = r1; r->v[2] = r2; r->v[3] = r3; r->v[4] = r4;
}
/* inputs may be unreduced user limbs (up to 64 bits): normalise to < 2^52 first */
static void fe_weak(fe* r, const fe* a) {
  u128 t[5];
  for (int i = 0; i < 5; ++i) t[i] = a->v[i];
  fe_carry(r, t);
}
static void fe_mul(fe* r, const fe* a, const fe* b) {
  fe x, y;
  fe_weak(&x, a); fe_weak(&y, b);
  u128 t[5];
  const u64 *f = x.v, *g = y.v;
  u64 g1 = 19 * g[1], g2 = 19 * g[2], g3 = 19 * g[3], g4 = 19 * g[4];
  t[0] = (u128)f[0] * g[0] + (u128)f[1] * g4 + (u128)f[2] * g3 + (u128)f[3] * g2 + (u128)f[4] * g1;
  t[1] = (u128)f[0] * g[1] + (u128)f[1] * g[0] + (u128)f[2] * g4 + (u128)f[3] * g3 + (u128)f[4] * g2;
  t[2] = (u128)f[0] * g[2] + (u128)f[1] * g[1] + (u128)f[2] * g[0] + (u128)f[3] * g4 + (u128)f[4] * g3;
  t[3] = (u128)f[0] * g[3] + (u128)f[1] * g[2] + (u128)f[2] * g[1] + (u128)f[3] * g[0] + (u128)f[4] * g4;
  t[4] = (u128)f[0] * g[4] + (u128)f[1] * g[3] + (u128)f[2] * g[2] + (u128)f[3] * g[1] + (u128)f[4] * g[0];
  fe_carry(r, t);
}
static void fe_sq(fe* r, const fe* a) { fe_mul(r, a, a); }
static void fe_add(fe* r, const fe* a, const fe* b) {
  fe x, y;
  fe_weak(&x, a); fe_weak(&y, b);
  for (int i = 0; i < 5; ++i) r->v[i] = x.v[i] + y.v[i];
}
static void fe_sub(fe* r, const fe* a, const fe* b) {
  /* a + 4p - b keeps every limb non-negative for operands < 2^53 */
  fe x, y;
  fe_weak(&x, a); fe_weak(&y, b);
  r->v[0] = x.v[0] + 0x1fffffffffffb4ULL - y.v[0];
  for (int i = 1; i < 5; ++i) r->v[i] = x.v[i] + 0x1ffffffffffffcULL - y.v[i];
}
static void fe_neg(fe* r, const fe* a) { fe z = {{0, 0, 0, 0, 0}}; fe_sub(r, &z, a); }
static void fe_reduce(fe* r, const fe* a) { /* canonical representative */
  fe t; fe_weak(&t, a); fe_weak(&t, &t);
  /* t < 2^255 + small: subtract p if t >= p */
  u64 c = (t.v[0] + 19) >> 51;
  c = (t.v[1] + c) >> 51; c = (t.v[2] + c) >> 51; c = (t.v[3] + c) >> 51; c = (t.v[4] + c) >> 51;
  t.v[0] += 19 * c;
  c = t.v[0] >> 51; t.v[0] &= MASK51;
  t.v[1] += c; c = t.v[1] >> 51; t.v[1] &= MASK51;
  t.v[2] += c; c = t.v[2] >> 51; t.v[2] &= MASK51;
  t.v[3] += c; c = t.v[3] >> 51; t.v[3] &= MASK51;
  t.v[4] += c; t.v[4] &= MASK51;
  *r = t;
}
static void fe_tobytes(uint8_t s[32], const fe* a) {
  fe t; fe_reduce(&t, a);
  u64 w[4];
  w[0] = t.v[0] | (t.v[1] << 51);
  w[1] = (t.v[1] >> 13) | (t.v[2] << 38);
  w[2] = (t.v[2] >> 26) | (t.v[3] << 25);
  w[3] = (t.v[3] >> 39) | (t.v[4] << 12);
  memcpy(s, w, 32);
}
static u64 load64(const uint8_t* s) { u64 w; memcpy(&w, s, 8); return w; }
static void fe_frombytes(fe* r, const uint8_t s[32]) {
  r->v[0] = load64(s) & MASK51;
  r->v[1] = (load64(s + 6) >> 3) & MASK51;
  r->v[2] = (load64(s + 12) >> 6) & MASK51;
  r->v[3] = (load64(s + 19) >> 1) & MASK51;
  r->v[4] = (load64(s + 24) >> 12) & MASK51;
}
static int fe_iszero(const fe* a) { uint8_t s[32]; fe_tobytes(s, a); int z = 0; for (int i = 0; i < 32; ++i) z |= s[i]; return z == 0; }
static int fe_isneg(const fe* a) { uint8_t s[32]; fe_tobytes(s, a); return s[0] & 1; }
static void fe_cmov(fe* r, const fe* a, int pick) { if (pick) *r = *a; }
static void fe_abs(fe* r, const fe* a) { fe n; fe_neg(&n, a); *r = *a; fe_cmov(r, &n, fe_isneg(a)); }
static void fe_pow(fe* r, const fe* a, const uint8_t e[32]) { /* little-endian exponent */
  fe acc = {{1, 0, 0, 0, 0}};
  for (int i = 255; i >= 0; --i) {
    fe_sq(&acc, &acc);
    if ((e[i >> 3] >> (i & 7)) & 1) fe_mul(&acc, &acc, a);
  }
  *r = acc;
}
static void fe_pow22523(fe* r, const fe* a) { /* (p-5)/8 = 2^252 - 3 */
  uint8_t e[32]; memset(e, 0xff, 32); e[0] = 0xfd; e[31] = 0x0f;
  fe_pow(r, a, e);
}
static const fe FE_ONE = {{1, 0, 0, 0, 0}};
/* curve constants as little-endian byte strings of their canonical values (mathematical constants
 * of ed25519 / ristretto255, RFC 9496 §4.1) */
static fe FE_D, FE_D2, FE_SQRTM1, FE_ONEMSQD, FE_SQDMONE, FE_SQRTADM1, FE_INVSQRTAMD;
static void fe_from_u64x4(fe* r, u64 w0, u64 w1, u64 w2, u64 w3) {
  u64 w[4] = {w0, w1, w2, w3}; uint8_t s[32]; memcpy(s, w, 32); fe_frombytes(r, s);
}
static void fe_invert(fe* r, const fe* a) {
  uint8_t e[32]; memset(e, 0xff, 32); e[0] = 0xeb; e[31] = 0x7f; fe_pow(r, a, e);
}
static void fe_init(void) {
  /* d = -121665/121666 */
  fe a = {{121665, 0, 0, 0, 0}}, b = {{121666, 0, 0, 0, 0}}, bi;
  fe_invert(&bi, &b); fe_mul(&FE_D, &a, &bi); fe_neg(&FE_D, &FE_D); fe_reduce(&FE_D, &FE_D);
  fe_add(&FE_D2, &FE_D, &FE_D);
  /* sqrt(-1) = 2^((p-1)/4) */
  uint8_t e[32]; memset(e, 0xff, 32); e[0] = 0xfb; e[31] = 0x1f; /* (p-1)/4 = 2^253 - 5 */
  fe two = {{2, 0, 0, 0, 0}}; fe_pow(&FE_SQRTM1, &two, e);
  fe dd, t; fe_sq(&dd, &FE_D); fe_sub(&FE_ONEMSQD, &FE_ONE, &dd);
  fe_sub(&t, &FE_D, &FE_ONE); fe_sq(&FE_SQDMONE, &t);
  /* sqrt(a*d - 1), a = -1: the odd root; 1/sqrt(a - d): the even root (RFC 9496 constants) */
  fe x, u, c;
  fe_neg(&u, &FE_D); fe_sub(&u, &u, &FE_ONE);            /* -d - 1 */
  uint8_t e38[32]; memset(e38, 0xff, 32); e38[0] = 0xfe; e38[31] = 0x0f; /* (p+3)/8 = 2^252 - 2 */
  fe_pow(&x, &u, e38); fe_sq(&c, &x); fe_sub(&c, &c, &u);
  if (!fe_iszero(&c)) fe_mul(&x, &x, &FE_SQRTM1);
  if (!fe_isneg(&x)) fe_neg(&x, &x);
  FE_SQRTADM1 = x;
  fe_neg(&u, &FE_ONE); fe_sub(&u, &u, &FE_D);            /* a - d */
  fe_pow(&x, &u, e38); fe_sq(&c, &x); fe_sub(&c, &c, &u);
  if (!fe_iszero(&c)) fe_mul(&x, &x, &FE_SQRTM1);
  fe_invert(&x, &x);
  if (fe_isneg(&x)) fe_neg(&x, &x);
  FE_INVSQRTAMD = x;
}

/* ---- ed25519 extended points ---- */
typedef struct { fe X, Y, Z, T; } ge;
static void ge_identity(ge* r) { memset(r, 0, sizeof(*r)); r->Y.v[0] = 1; r->Z.v[0] = 1; }
static void ge_add(ge* r, const ge* p, const ge* q) {
  fe a, b, c, d, e, f, g, h, t0, t1;
  fe_sub(&t0, &p->Y, &p->X); fe_sub(&t1, &q->Y, &q->X); fe_mul(&a, &t0, &t1);
  fe_add(&t0, &p->Y, &p->X); fe_add(&t1, &q->Y, &q->X); fe_mul(&b, &t0, &t1);
  fe_mul(&c, &p->T, &q->T); fe_mul(&c, &c, &FE_D2);
  fe_mul(&d, &p->Z, &q->Z); fe_add(&d, &d, &d);
  fe_sub(&e, &b, &a); fe_sub(&f, &d, &c); fe_add(&g, &d, &c); fe_add(&h, &b, &a);
  fe_mul(&r->X, &e, &f); fe_mul(&r->Y, &g, &h); fe_mul(&r->T, &e, &h); fe_mul(&r->Z, &f, &g);
}
static void ge_dbl(ge* r, const ge* p) {
  fe a, b, c, e, f, g, h, t0;
  fe_sq(&a, &p->X); fe_sq(&b, &p->Y); fe_sq(&c, &p->Z); fe_add(&c, &c, &c);
  fe_add(&h, &a, &b); fe_add(&t0, &p->X, &p->Y); fe_sq(&t0, &t0); fe_sub(&e, &h, &t0);
  fe_sub(&g, &a, &b); fe_add(&f, &c, &g);
  fe_mul(&r->X, &e, &f); fe_mul(&r->Y, &g, &h); fe_mul(&r->T, &e, &h); fe_mul(&r->Z, &f, &g);
}
static void ge_neg(ge* r, const ge* p) { fe_neg(&r->X, &p->X); r->Y = p->Y; r->Z = p->Z; fe_neg(&r->T, &p->T); }

static int sqrt_ratio_m1(fe* x, const fe* u, const fe* v) {
  fe v3, vxx, t, chk, xs;
  fe_sq(&v3, v); fe_mul(&v3, &v3, v);
  fe_sq(x, &v3); fe_mul(x, x, u); fe_mul(x, x, v);
  fe_pow22523(x, x); fe_mul(x, x, &v3); fe_mul(x, x, u);
  fe_sq(&vxx, x); fe_mul(&vxx, &vxx, v);
  fe_sub(&chk, &vxx, u); int m_root = fe_iszero(&chk);
  fe_add(&chk, &vxx, u); int p_root = fe_iszero(&chk);
  fe_mul(&t, u, &FE_SQRTM1); fe_add(&chk, &vxx, &t); int f_root = fe_iszero(&chk);
  fe_mul(&xs, x, &FE_SQRTM1);
  fe_cmov(x, &xs, p_root | f_root);
  fe_abs(x, x);
  return m_root | p_root;
}
static void ristretto_encode(uint8_t s[32], const ge* p) {
  fe u1, u2, zmy, u1u2u2, inv_sqrt, den1, den2, z_inv, ix, iy, eden, tz, x_, y_, den_inv, xz, s_, ny;
  fe_add(&u1, &p->Z, &p->Y); fe_sub(&zmy, &p->Z, &p->Y); fe_mul(&u1, &u1, &zmy);
  fe_mul(&u2, &p->X, &p->Y);
  fe_sq(&u1u2u2, &u2); fe_mul(&u1u2u2, &u1, &u1u2u2);
  (void)sqrt_ratio_m1(&inv_sqrt, &FE_ONE, &u1u2u2);
  fe_mul(&den1, &inv_sqrt, &u1); fe_mul(&den2, &inv_sqrt, &u2);
  fe_mul(&z_inv, &den1, &den2); fe_mul(&z_inv, &z_inv, &p->T);
  fe_mul(&ix, &p->X, &FE_SQRTM1); fe_mul(&iy, &p->Y, &FE_SQRTM1);
  fe_mul(&eden, &den1, &FE_INVSQRTAMD);
  fe_mul(&tz, &p->T, &z_inv);
  int rotate = fe_isneg(&tz);
  x_ = p->X; y_ = p->Y; den_inv = den2;
  fe_cmov(&x_, &iy, rotate); fe_cmov(&y_, &ix, rotate); fe_cmov(&den_inv, &eden, rotate);
  fe_mul(&xz, &x_, &z_inv);
  fe_neg(&ny, &y_); fe_cmov(&y_, &ny, fe_isneg(&xz));
  fe_sub(&s_, &p->Z, &y_); fe_mul(&s_, &den_inv, &s_); fe_abs(&s_, &s_);
  fe_tobytes(s, &s_);
}
static void elligator(ge* p, const fe* t) {
  fe r, u, c, rpd, v, s, s_prime, n, w0, w1, w2, w3, ss;
  fe_sq(&r, t); fe_mul(&r, &FE_SQRTM1, &r);
  fe_add(&u, &r, &FE_ONE); fe_mul(&u, &u, &FE_ONEMSQD);
  fe_neg(&c, &FE_ONE);
  fe_add(&rpd, &r, &FE_D);
  fe_mul(&v, &r, &FE_D); fe_sub(&v, &c, &v); fe_mul(&v, &v, &rpd);
  int wasnt_square = 1 - sqrt_ratio_m1(&s, &u, &v);
  fe_mul(&s_prime, &s, t); fe_abs(&s_prime, &s_prime); fe_neg(&s_prime, &s_prime);
  fe_cmov(&s, &s_prime, wasnt_square); fe_cmov(&c, &r, wasnt_square);
  fe_sub(&n, &r, &FE_ONE); fe_mul(&n, &n, &c); fe_mul(&n, &n, &FE_SQDMONE); fe_sub(&n, &n, &v);
  fe_add(&w0, &s, &s); fe_mul(&w0, &w0, &v);
  fe_mul(&w1, &n, &FE_SQRTADM1);
  fe_sq(&ss, &s); fe_sub(&w2, &FE_ONE, &ss); fe_add(&w3, &FE_ONE, &ss);
  fe_mul(&p->X, &w0, &w3); fe_mul(&p->Y, &w2, &w1); fe_mul(&p->Z, &w1, &w3); fe_mul(&p->T, &w0, &w2);
}
static void builtin_generator(ge* g, u64 index) {
  u64 sa = index + 1, sb = index + 2;
  fe r[2];
  for (int k = 0; k < 2; ++k) {
    u64 w[4];
    for (int j = 0; j < 4; ++j) {
      u64 t = sa, s = sb;
      sa = s; t ^= t << 23; t ^= t >> 17; t ^= s ^ (s >> 26); sb = t;
      w[j] = t + s;
    }
    uint8_t bytes[32]; memcpy(bytes, w, 32); fe_frombytes(&r[k], bytes);
  }
  ge p0, p1; elligator(&p0, &r[0]); elligator(&p1, &r[1]); ge_add(g, &p1, &p0);
}

/* ================================================================================================
 * Montgomery fields, u64 limbs (N = 4 or 6), R = 2^(64 N)
 * ==============================================================================================*/
#define MAXN 6
typedef struct { u64 v[MAXN]; } mf;
typedef struct {
  int n;
  u64 p[MAXN], one[MAXN], r2[MAXN], inv, pm2[MAXN], half[MAXN];
  mf b3; /* 3b, Montgomery form */
  int b; /* curve constant */
} mfield;
static int mf_geq(const u64* a, const u64* b, int n) {
  for (int i = n - 1; i >= 0; --i) { if (a[i] > b[i]) return 1; if (a[i] < b[i]) return 0; }
  return 1;
}
static u64 mf_addn(u64* r, const u64* a, const u64* b, int n) {
  u128 c = 0; for (int i = 0; i < n; ++i) { c += (u128)a[i] + b[i]; r[i] = (u64)c; c >>= 64; } return (u64)c;
}
static u64 mf_subn(u64* r, const u64* a, const u64* b, int n) {
  u64 bw = 0; for (int i = 0; i < n; ++i) { u128 t = (u128)a[i] - b[i] - bw; r[i] = (u64)t; bw = (u64)(t >> 127); } return bw;
}
static void mf_add(const mfield* F, mf* r, const mf* a, const mf* b) {
  u64 s[MAXN]; u64 c = mf_addn(s, a->v, b->v, F->n);
  if (c || mf_geq(s, F->p, F->n)) mf_subn(s, s, F->p, F->n);
  memset(r->v, 0, sizeof(r->v)); memcpy(r->v, s, 8 * F->n);
}
static void mf_sub(const mfield* F, mf* r, const mf* a, const mf* b) {
  u64 s[MAXN]; if (mf_subn(s, a->v, b->v, F->n)) mf_addn(s, s, F->p, F->n);
  memset(r->v, 0, sizeof(r->v)); memcpy(r->v, s, 8 * F->n);
}
static void mf_neg(const mfield* F, mf* r, const mf* a) { mf z; memset(&z, 0, sizeof(z)); mf_sub(F, r, &z, a); }
static void mf_mul(const mfield* F, mf* r, const mf* a, const mf* b) {
  int n = F->n; u64 t[MAXN + 2]; memset(t, 0, sizeof(t));
  for (int i = 0; i < n; ++i) {
    u128 c = 0;
    for (int j = 0; j < n; ++j) { c += (u128)a->v[j] * b->v[i] + t[j]; t[j] = (u64)c; c >>= 64; }
    c += t[n]; t[n] = (u64)c; t[n + 1] = (u64)(c >> 64);
    u64 m = t[0] * F->inv;
    c = ((u128)m * F->p[0] + t[0]) >> 64;
    for (int j = 1; j < n; ++j) { c += (u128)m * F->p[j] + t[j]; t[j - 1] = (u64)c; c >>= 64; }
    c += t[n]; t[n - 1] = (u64)c; t[n] = t[n + 1] + (u64)(c >> 64);
  }
  if (t[n] || mf_geq(t, F->p, n)) mf_subn(t, t, F->p, n);
  memset(r->v, 0, sizeof(r->v)); memcpy(r->v, t, 8 * n);
}
static int mf_iszero(const mfield* F, const mf* a) { u64 x = 0; for (int i = 0; i < F->n; ++i) x |= a->v[i]; return x == 0; }
static void mf_one(const mfield* F, mf* r) { memset(r, 0, sizeof(*r)); memcpy(r->v, F->one, 8 * F->n); }
static void mf_pow(const mfield* F, mf* r, const mf* a, const u64* e) {
  mf acc; mf_one(F, &acc);
  for (int i = 64 * F->n - 1; i >= 0; --i) {
    mf_mul(F, &acc, &acc, &acc);
    if ((e[i >> 6] >> (i & 63)) & 1) mf_mul(F, &acc, &acc, a);
  }
  *r = acc;
}
static void mf_inv(const mfield* F, mf* r, const mf* a) { mf_pow(F, r, a, F->pm2); }
static void mf_from_mont(const mfield* F, mf* r, const mf* a) { mf o; memset(&o, 0, sizeof(o)); o.v[0] = 1; mf_mul(F, r, a, &o); }
static void mf_to_mont(const mfield* F, mf* r, const mf* a) { mf r2; memset(&r2, 0, sizeof(r2)); memcpy(r2.v, F->r2, 8 * F->n); mf_mul(F, r, a, &r2); }
static void mf_small(const mfield* F, mf* r, int k) { /* Montgomery form of a small signed integer */
  mf x; memset(&x, 0, sizeof(x)); x.v[0] = (u64)(k < 0 ? -k : k); mf_to_mont(F, r, &x); if (k < 0) mf_neg(F, r, r);
}
static void mfield_init(mfield* F, int n, const u64* p, int b) {
  memset(F, 0, sizeof(*F)); F->n = n; F->b = b; memcpy(F->p, p, 8 * n);
  u64 inv = 1; for (int i = 0; i < 6; ++i) inv *= 2 - p[0] * inv; F->inv = (u64)0 - inv;
  /* R mod p and R^2 mod p by repeated doubling of 1 */
  u64 x[MAXN]; memset(x, 0, sizeof(x)); x[0] = 1;
  for (int i = 0; i < 128 * n; ++i) {
    u64 c = mf_addn(x, x, x, n);
    if (c || mf_geq(x, p, n)) mf_subn(x, x, p, n);
    if (i == 64 * n - 1) memcpy(F->one, x, 8 * n);
  }
  memcpy(F->r2, x, 8 * n);
  u64 two[MAXN] = {2}, onev[MAXN] = {1};
  mf_subn(F->pm2, p, two, n);
  mf_subn(F->half, p, onev, n);
  for (int i = 0; i < n; ++i) F->half[i] = (F->half[i] >> 1) | (i + 1 < n ? F->half[i + 1] << 63 : 0);
  mf_small(F, &F->b3, 3 * b);
}

/* ---- homogeneous projective points, y^2 = x^3 + b ---- */
typedef struct { mf X, Y, Z; } wp;
static void wp_identity(const mfield* F, wp* r) { memset(r, 0, sizeof(*r)); mf_one(F, &r->Y); }
static void wp_add(const mfield* F, wp* r, const wp* p, const wp* q) { /* RCB16 Alg. 7 */
  mf t0, t1, t2, t3, t4, x3, y3, z3;
  mf_mul(F, &t0, &p->X, &q->X); mf_mul(F, &t1, &p->Y, &q->Y); mf_mul(F, &t2, &p->Z, &q->Z);
  mf_add(F, &t3, &p->X, &p->Y); mf_add(F, &t4, &q->X, &q->Y); mf_mul(F, &t3, &t3, &t4);
  mf_add(F, &t4, &t0, &t1); mf_sub(F, &t3, &t3, &t4);
  mf_add(F, &t4, &p->Y, &p->Z); mf_add(F, &x3, &q->Y, &q->Z); mf_mul(F, &t4, &t4, &x3);
  mf_add(F, &x3, &t1, &t2); mf_sub(F, &t4, &t4, &x3);
  mf_add(F, &x3, &p->X, &p->Z); mf_add(F, &y3, &q->X, &q->Z); mf_mul(F, &x3, &x3, &y3);
  mf_add(F, &y3, &t0, &t2); mf_sub(F, &y3, &x3, &y3);
  mf_add(F, &x3, &t0, &t0); mf_add(F, &t0, &x3, &t0);
  mf_mul(F, &t2, &F->b3, &t2);
  mf_add(F, &z3, &t1, &t2); mf_sub(F, &t1, &t1, &t2);
  mf_mul(F, &y3, &F->b3, &y3);
  mf_mul(F, &x3, &t4, &y3); mf_mul(F, &t2, &t3, &t1); mf_sub(F, &x3, &t2, &x3);
  mf_mul(F, &y3, &y3, &t0); mf_mul(F, &t1, &t1, &z3); mf_add(F, &y3, &t1, &y3);
  mf_mul(F, &t0, &t0, &t3); mf_mul(F, &z3, &z3, &t4); mf_add(F, &z3, &z3, &t0);
  r->X = x3; r->Y = y3; r->Z = z3;
}
static void wp_dbl(const mfield* F, wp* r, const wp* p) { /* RCB16 Alg. 9 */
  mf t0, t1, t2, x3, y3, z3;
  mf_mul(F, &t0, &p->Y, &p->Y);
  mf_add(F, &z3, &t0, &t0); mf_add(F, &z3, &z3, &z3); mf_add(F, &z3, &z3, &z3);
  mf_mul(F, &t1, &p->Y, &p->Z); mf_mul(F, &t2, &p->Z, &p->Z); mf_mul(F, &t2, &F->b3, &t2);
  mf_mul(F, &x3, &t2, &z3); mf_add(F, &y3, &t0, &t2); mf_mul(F, &z3, &t1, &z3);
  mf_add(F, &t1, &t2, &t2); mf_add(F, &t2, &t1, &t2); mf_sub(F, &t0, &t0, &t2);
  mf_mul(F, &y3, &t0, &y3); mf_add(F, &y3, &x3, &y3);
  mf_mul(F, &t1, &p->X, &p->Y); mf_mul(F, &x3, &t0, &t1); mf_add(F, &x3, &x3, &x3);
  r->X = x3; r->Y = y3; r->Z = z3;
}
static void wp_neg(const mfield* F, wp* r, const wp* p) { r->X = p->X; mf_neg(F, &r->Y, &p->Y); r->Z = p->Z; }
/* returns infinity flag; identity -> {0, R, 1} */
static int wp_to_affine(const mfield* F, mf* x, mf* y, const wp* p) {
  if (mf_iszero(F, &p->Z)) { memset(x, 0, sizeof(*x)); mf_one(F, y); return 1; }
  mf zi; mf_inv(F, &zi, &p->Z); mf_mul(F, x, &p->X, &zi); mf_mul(F, y, &p->Y, &zi); return 0;
}

/* ================================================================================================
 * generic group interface used by the MSM restatement
 * ==============================================================================================*/
enum { C_RISTRETTO = 0, C_BLS = 1, C_BN = 2, C_GK = 3 };
typedef union { ge e; wp w; } pt;
static mfield FBLS, FBN, FGK;
static int g_init = 0;
static const mfield* fld(int c) { return c == C_BLS ? &FBLS : (c == C_BN ? &FBN : &FGK); }
static void oracle_init(void) {
  if (g_init) return;
  fe_init();
  static const u64 pbls[6] = {0xb9feffffffffaaabULL, 0x1eabfffeb153ffffULL, 0x6730d2a0f6b0f624ULL,
                              0x64774b84f38512bfULL, 0x4b1ba7b6434bacd7ULL, 0x1a0111ea397fe69aULL};
  static const u64 pbn[4] = {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
  static const u64 pgk[4] = {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
  mfield_init(&FBLS, 6, pbls, 4);
  mfield_init(&FBN, 4, pbn, 3);
  mfield_init(&FGK, 4, pgk, -17);
  g_init = 1;
}
static void pt_identity(int c, pt* r) { if (c == C_RISTRETTO) ge_identity(&r->e); else wp_identity(fld(c), &r->w); }
static void pt_add(int c, pt* r, const pt* a, const pt* b) { if (c == C_RISTRETTO) ge_add(&r->e, &a->e, &b->e); else wp_add(fld(c), &r->w, &a->w, &b->w); }
static void pt_dbl(int c, pt* r, const pt* a) { if (c == C_RISTRETTO) ge_dbl(&r->e, &a->e); else wp_dbl(fld(c), &r->w, &a->w); }
static void pt_neg(int c, pt* r, const pt* a) { if (c == C_RISTRETTO) ge_neg(&r->e, &a->e); else wp_neg(fld(c), &r->w, &a->w); }

static int proj_bytes(int c) { return c == C_RISTRETTO ? 160 : (c == C_BLS ? 144 : 96); }
static int affine_stride(int c) { return c == C_RISTRETTO ? 160 : (c == C_BLS ? 104 : 72); }
static int commit_bytes(int c) { return c == C_RISTRETTO ? 32 : (c == C_BLS ? 48 : 72); }

/* ABI loads / stores */
static void load_proj(int c, pt* r, const uint8_t* s) {
  if (c == C_RISTRETTO) { memcpy(&r->e, s, 160); return; }
  int nb = 8 * fld(c)->n; memset(&r->w, 0, sizeof(r->w));
  memcpy(r->w.X.v, s, nb); memcpy(r->w.Y.v, s + nb, nb); memcpy(r->w.Z.v, s + 2 * nb, nb);
}
static void store_proj(int c, uint8_t* d, const pt* p) {
  if (c == C_RISTRETTO) {
    ge t; fe_reduce(&t.X, &p->e.X); fe_reduce(&t.Y, &p->e.Y); fe_reduce(&t.Z, &p->e.Z); fe_reduce(&t.T, &p->e.T);
    memcpy(d, &t, 160); return;
  }
  int nb = 8 * fld(c)->n;
  memcpy(d, p->w.X.v, nb); memcpy(d + nb, p->w.Y.v, nb); memcpy(d + 2 * nb, p->w.Z.v, nb);
}
/* commitment-API generator: ristretto = element_p3; Weierstrass = affine {X, Y, infinity} */
static void load_commit_gen(int c, pt* r, const uint8_t* s) {
  if (c == C_RISTRETTO) { memcpy(&r->e, s, 160); return; }
  const mfield* F = fld(c); int nb = 8 * F->n;
  if (s[2 * nb]) { wp_identity(F, &r->w); return; }
  memset(&r->w, 0, sizeof(r->w));
  memcpy(r->w.X.v, s, nb); memcpy(r->w.Y.v, s + nb, nb); mf_one(F, &r->w.Z);
}
static void store_commit(int c, uint8_t* d, const pt* p) {
  if (c == C_RISTRETTO) { ristretto_encode(d, &p->e); return; }
  const mfield* F = fld(c); int nb = 8 * F->n;
  mf x, y; int inf = wp_to_affine(F, &x, &y, &p->w);
  if (c == C_BLS) {
    mf xp; if (inf) memset(&x, 0, sizeof(x));
    mf_from_mont(F, &xp, &x);
    for (int i = 0; i < 6; ++i) for (int k = 0; k < 8; ++k) d[8 * i + k] = (uint8_t)(xp.v[5 - i] >> (56 - 8 * k));
    d[0] |= 0x80;
    if (inf) d[0] |= 0x40;
    else {
      mf yp; mf_from_mont(F, &yp, &y);
      u64 t[MAXN]; if (mf_subn(t, F->half, yp.v, F->n)) d[0] |= 0x20; /* y > (p-1)/2 */
    }
    return;
  }
  memset(d, 0, 72); memcpy(d, x.v, nb); memcpy(d + nb, y.v, nb); d[2 * nb] = (uint8_t)inf;
}

/* ================================================================================================
 * scalar access (exponent_sequence semantics + bit-packed rows) and the bucket-method MSM
 * ==============================================================================================*/
typedef struct { const uint8_t* base; u64 row_stride; unsigned bit_offset, bit_width; u64 n; int is_signed; } column;

/* magnitude bytes (32, little-endian) and sign of term i */
static int load_scalar(uint8_t mag[32], const column* col, u64 i) {
  memset(mag, 0, 32);
  const uint8_t* row = col->base + i * col->row_stride;
  for (unsigned b = 0; b < col->bit_width; ++b) {
    unsigned pos = col->bit_offset + b;
    if ((row[pos >> 3] >> (pos & 7)) & 1) mag[b >> 3] |= (uint8_t)(1u << (b & 7));
  }
  if (!col->is_signed) return 0;
  unsigned top = col->bit_width - 1;
  if (!((mag[top >> 3] >> (top & 7)) & 1)) return 0;
  /* two's complement negate within bit_width */
  unsigned carry = 1;
  for (unsigned k = 0; k < (col->bit_width + 7) / 8; ++k) {
    unsigned m = 0xff; if (8 * k + 8 > col->bit_width) m = (1u << (col->bit_width - 8 * k)) - 1;
    unsigned v = ((~mag[k]) & m) + carry; mag[k] = (uint8_t)(v & m); carry = (m == 0xff) ? (v >> 8) : 0;
  }
  return 1;
}

static void msm_column(int c, pt* out, const pt* gens, const column* col) {
  /* 32 byte-windows x 255 buckets */
  pt* buckets = (pt*)malloc(sizeof(pt) * 32 * 255);
  for (int k = 0; k < 32 * 255; ++k) pt_identity(c, &buckets[k]);
  int max_window = 0;
  for (u64 i = 0; i < col->n; ++i) {
    uint8_t mag[32]; int neg = load_scalar(mag, col, i);
    pt g = gens[i]; if (neg) pt_neg(c, &g, &g);
    for (int w = 0; w < 32; ++w) {
      if (!mag[w]) continue;
      pt* b = &buckets[w * 255 + mag[w] - 1];
      pt_add(c, b, b, &g);
      if (w > max_window) max_window = w;
    }
  }
  pt acc; pt_identity(c, &acc);
  for (int w = max_window; w >= 0; --w) {
    for (int k = 0; k < 8; ++k) pt_dbl(c, &acc, &acc);
    pt run, sum; pt_identity(c, &run); pt_identity(c, &sum);
    for (int d = 254; d >= 0; --d) { pt_add(c, &run, &run, &buckets[w * 255 + d]); pt_add(c, &sum, &sum, &run); }
    pt_add(c, &acc, &acc, &sum);
  }
  *out = acc;
  free(buckets);
}

/* ================================================================================================
 * exported API
 * ==============================================================================================*/
typedef struct { uint8_t element_nbytes; u64 n; const uint8_t* data; int is_signed; } oracle_sequence_descriptor;

void oracle_ristretto255_get_generators(uint8_t* out160, u64 num, u64 offset) {
  oracle_init();
  for (u64 i = 0; i < num; ++i) {
    pt g; builtin_generator(&g.e, offset + i);
    store_proj(C_RISTRETTO, out160 + 160 * i, &g);
  }
}

/* same contract as the five sxt_*_compute_pedersen_commitments* calls (generators == NULL: built-in
 * ristretto generators at offset_generators) */
void oracle_commit(unsigned curve, uint8_t* commitments, uint32_t num_sequences,
                   const oracle_sequence_descriptor* d, const uint8_t* generators, u64 offset_generators) {
  oracle_init();
  if (num_sequences == 0) return;
  u64 n = 0;
  for (uint32_t j = 0; j < num_sequences; ++j) if (d[j].n > n) n = d[j].n;
  pt* gens = (pt*)malloc(sizeof(pt) * (n ? n : 1));
  for (u64 i = 0; i < n; ++i) {
    if (generators) load_commit_gen((int)curve, &gens[i], generators + (u64)affine_stride((int)curve) * i);
    else builtin_generator(&gens[i].e, offset_generators + i);
  }
  for (uint32_t j = 0; j < num_sequences; ++j) {
    column col = {d[j].data, d[j].element_nbytes, 0, 8u * d[j].element_nbytes, d[j].n, d[j].is_signed};
    pt r; msm_column((int)curve, &r, gens, &col);
    store_commit((int)curve, commitments + (u64)commit_bytes((int)curve) * j, &r);
  }
  free(gens);
}

/* fixed-base MSM over projective ABI generators. mode 0: fixed width; 1: packed; 2: variable length.
 * res: projective ABI structs. */
void oracle_fixed_msm(unsigned curve, uint8_t* res, const uint8_t* generators_proj, unsigned num_generators,
                      int mode, unsigned element_num_bytes, const unsigned* output_bit_table,
                      const unsigned* output_lengths, unsigned num_outputs, unsigned n, const uint8_t* scalars) {
  oracle_init();
  int c = (int)curve;
  pt* gens = (pt*)malloc(sizeof(pt) * (num_generators ? num_generators : 1));
  for (unsigned i = 0; i < num_generators; ++i) load_proj(c, &gens[i], generators_proj + (u64)proj_bytes(c) * i);
  u64 row_bits = 0;
  for (unsigned j = 0; j < num_outputs; ++j) row_bits += mode == 0 ? 8u * element_num_bytes : output_bit_table[j];
  u64 stride = (row_bits + 7) / 8, off = 0;
  for (unsigned j = 0; j < num_outputs; ++j) {
    unsigned width = mode == 0 ? 8u * element_num_bytes : output_bit_table[j];
    column col = {scalars, stride, (unsigned)off, width, mode == 2 ? output_lengths[j] : n, 0};
    pt r; msm_column(c, &r, gens, &col);
    store_proj(c, res + (u64)proj_bytes(c) * j, &r);
    off += width;
  }
  free(gens);
}

/* projective ABI structs -> canonical comparison form (ristretto 32 B, bls 48 B, bn254/grumpkin 72 B) */
void oracle_normalize(unsigned curve, uint8_t* out, const uint8_t* in_projective, u64 n) {
  oracle_init();
  for (u64 i = 0; i < n; ++i) {
    pt p; load_proj((int)curve, &p, in_projective + (u64)proj_bytes((int)curve) * i);
    store_commit((int)curve, out + (u64)commit_bytes((int)curve) * i, &p);
  }
}

/* Deterministic test points: P_i = k_i * G for pseudo-random 64-bit k_i (xorshift of seed + i) and the
 * curve's standard generator. Writes the commitment-API layout (affine, curve stride) and/or the
 * projective ABI layout. Not for ristretto (use oracle_ristretto255_get_generators). */
void oracle_test_points(unsigned curve, uint8_t* out_affine, uint8_t* out_proj, u64 n, u64 seed) {
  oracle_init();
  int c = (int)curve; const mfield* F = fld(c); int nb = 8 * F->n;
  wp G; memset(&G, 0, sizeof(G)); mf_one(F, &G.Z);
  if (c == C_BLS) {
    static const u64 gx[6] = {0xfb3af00adb22c6bbULL, 0x6c55e83ff97a1aefULL, 0xa14e3a3f171bac58ULL,
                              0xc3688c4f9774b905ULL, 0x2695638c4fa9ac0fULL, 0x17f1d3a73197d794ULL};
    static const u64 gy[6] = {0x0caa232946c5e7e1ULL, 0xd03cc744a2888ae4ULL, 0x00db18cb2c04b3edULL,
                              0xfcf5e095d5d00af6ULL, 0xa09e30ed741d8ae4ULL, 0x08b3f481e3aaa0f1ULL};
    mf x, y; memset(&x, 0, sizeof(x)); memset(&y, 0, sizeof(y)); memcpy(x.v, gx, 48); memcpy(y.v, gy, 48);
    mf_to_mont(F, &G.X, &x); mf_to_mont(F, &G.Y, &y);
  } else if (c == C_BN) {
    mf_small(F, &G.X, 1); mf_small(F, &G.Y, 2);
  } else {
    static const u64 gy[4] = {0x833fc48d823f272cULL, 0x2d270d45f1181294ULL, 0xcf135e7506a45d63ULL, 0x2ULL};
    mf y; memset(&y, 0, sizeof(y)); memcpy(y.v, gy, 32);
    mf_small(F, &G.X, 1); mf_to_mont(F, &G.Y, &y);
  }
  for (u64 i = 0; i < n; ++i) {
    u64 k = (seed + i + 1) * 0x9E3779B97F4A7C15ULL; k ^= k >> 29; k *= 0xBF58476D1CE4E5B9ULL; k ^= k >> 32; k |= 1;
    wp acc; wp_identity(F, &acc);
    for (int b = 63; b >= 0; --b) { wp_dbl(F, &acc, &acc); if ((k >> b) & 1) wp_add(F, &acc, &acc, &G); }
    if (out_proj) { pt p; p.w = acc; store_proj(c, out_proj + (u64)proj_bytes(c) * i, &p); }
    if (out_affine) {
      mf x, y; int inf = wp_to_affine(F, &x, &y, &acc);
      uint8_t* d = out_affine + (u64)affine_stride(c) * i; memset(d, 0, affine_stride(c));
      memcpy(d, x.v, nb); memcpy(d + nb, y.v, nb); d[2 * nb] = (uint8_t)inf;
    }
  }
}

/* ================================================================================================
 * Inner-product argument (restated from cbindings/inner_product_proof.cc:101-167,
 * sxt/proof/inner_product/proof_computation.cc:61-155, cpu_driver.cc:47-257, fold.cc:28-49,
 * verification_computation.cc:31-127) with its Merlin transcript (sxt/proof/transcript/
 * strobe128.cc:47-160, transcript.cc:41-88, transcript_utility.cc:27-31, keccakf.cc) and the scalar
 * field mod l (sxt/scalar25/operation/{mul,muladd,inv,reduce}.cc).
 * ==============================================================================================*/
typedef struct { u64 v[4]; } sc;
static const u64 SC_L[4] = {0x5812631a5cf5d3edULL, 0x14def9dea2f79cd6ULL, 0ULL, 0x1000000000000000ULL};
static u64 SC_INV, SC_R2[4];
static int sc_ready = 0;
static void sc_init(void) {
  if (sc_ready) return;
  u64 x = 1; for (int i = 0; i < 6; ++i) x *= 2 - SC_L[0] * x; SC_INV = (u64)0 - x;
  u64 t[MAXN]; memset(t, 0, sizeof(t)); t[0] = 1;
  for (int i = 0; i < 512; ++i) { u64 c = mf_addn(t, t, t, 4); if (c || mf_geq(t, SC_L, 4)) mf_subn(t, t, SC_L, 4); }
  memcpy(SC_R2, t, 32); sc_ready = 1;
}
static void sc_mont(sc* r, const sc* a, const u64* b) {
  u64 t[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; ++i) {
    u128 c = 0;
    for (int j = 0; j < 4; ++j) { c += (u128)a->v[j] * b[i] + t[j]; t[j] = (u64)c; c >>= 64; }
    c += t[4]; t[4] = (u64)c; t[5] = (u64)(c >> 64);
    u64 m = t[0] * SC_INV;
    c = ((u128)m * SC_L[0] + t[0]) >> 64;
    for (int j = 1; j < 4; ++j) { c += (u128)m * SC_L[j] + t[j]; t[j - 1] = (u64)c; c >>= 64; }
    c += t[4]; t[3] = (u64)c; t[4] = t[5] + (u64)(c >> 64);
  }
  if (t[4] || mf_geq(t, SC_L, 4)) mf_subn(t, t, SC_L, 4);
  memcpy(r->v, t, 32);
}
static sc sc_mul(sc a, sc b) { sc t, r; sc_mont(&t, &a, b.v); sc_mont(&r, &t, SC_R2); return r; }
static sc sc_reduce32(sc a) { sc t, r; u64 one[4] = {1, 0, 0, 0}; sc_mont(&t, &a, SC_R2); sc_mont(&r, &t, one); return r; }
static sc sc_add(sc a, sc b) { sc r; u64 c = mf_addn(r.v, a.v, b.v, 4); if (c || mf_geq(r.v, SC_L, 4)) mf_subn(r.v, r.v, SC_L, 4); return r; }
static sc sc_sub(sc a, sc b) { sc r; if (mf_subn(r.v, a.v, b.v, 4)) mf_addn(r.v, r.v, SC_L, 4); return r; }
static sc sc_neg(sc a) { sc z = {{0, 0, 0, 0}}; return sc_sub(z, a); }
static sc sc_inv(sc a) {
  u64 e[4], two[4] = {2, 0, 0, 0}; mf_subn(e, SC_L, two, 4);
  sc acc = {{1, 0, 0, 0}};
  for (int i = 255; i >= 0; --i) { acc = sc_mul(acc, acc); if ((e[i >> 6] >> (i & 63)) & 1) acc = sc_mul(acc, a); }
  return acc;
}
static sc sc_load(const uint8_t* b) { sc r; memcpy(r.v, b, 32); return r; }
static sc sc_inner(const uint8_t* a, const uint8_t* b, u64 n) {
  sc acc = {{0, 0, 0, 0}};
  for (u64 i = 0; i < n; ++i) acc = sc_add(acc, sc_mul(sc_load(a + 32 * i), sc_load(b + 32 * i)));
  return acc;
}

/* Keccak-f[1600] (FIPS 202) */
static u64 rotl64(u64 x, int s) { return (x << s) | (x >> (64 - s)); }
static void keccakf(uint8_t* st) {
  static const u64 RC[24] = {
      0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
      0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
      0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
      0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
      0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
      0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
  u64 a[25]; memcpy(a, st, 200);
  for (int round = 0; round < 24; ++round) {
    u64 c[5], b[25];
    for (int x = 0; x < 5; ++x) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    for (int x = 0; x < 5; ++x) { u64 d = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1); for (int y = 0; y < 25; y += 5) a[y + x] ^= d; }
    /* rho + pi from the definition: B[y][2x+3y] = rot(A[x][y], r[x][y]) */
    static const int R[5][5] = {{0, 36, 3, 41, 18}, {1, 44, 10, 45, 2}, {62, 6, 43, 15, 61}, {28, 55, 25, 21, 56}, {27, 20, 39, 8, 14}};
    for (int x = 0; x < 5; ++x) for (int y = 0; y < 5; ++y) {
      int nx = y, ny = (2 * x + 3 * y) % 5;
      u64 v = a[5 * y + x];
      b[5 * ny + nx] = R[x][y] ? rotl64(v, R[x][y]) : v;
    }
    for (int y = 0; y < 5; ++y) for (int x = 0; x < 5; ++x) a[5 * y + x] = b[5 * y + x] ^ (~b[5 * y + (x + 1) % 5] & b[5 * y + (x + 2) % 5]);
    a[0] ^= RC[round];
  }
  memcpy(st, a, 200);
}
/* STROBE-128 subset used by Merlin, on the 203-byte transcript {state[200], pos, pos_begin, cur_flags} */
#define ST_R 166
static void st_run_f(uint8_t* s) { s[s[200]] ^= s[201]; s[s[200] + 1] ^= 0x04; s[ST_R + 1] ^= 0x80; keccakf(s); s[200] = 0; s[201] = 0; }
static void st_absorb(uint8_t* s, const uint8_t* d, size_t n) { for (size_t i = 0; i < n; ++i) { s[s[200]] ^= d[i]; s[200] += 1; if (s[200] == ST_R) st_run_f(s); } }
static void st_squeeze(uint8_t* s, uint8_t* d, size_t n) { for (size_t i = 0; i < n; ++i) { d[i] = s[s[200]]; s[s[200]] = 0; s[200] += 1; if (s[200] == ST_R) st_run_f(s); } }
static void st_begin(uint8_t* s, uint8_t flags, int more) {
  if (more) return;
  uint8_t old = s[201]; s[201] = (uint8_t)(s[200] + 1); s[202] = flags;
  uint8_t d[2] = {old, flags}; st_absorb(s, d, 2);
  if ((flags & (4 | 32)) && s[200] != 0) st_run_f(s);
}
static void st_meta_ad(uint8_t* s, const uint8_t* d, size_t n, int more) { st_begin(s, 16 | 2, more); st_absorb(s, d, n); }
static void tr_append(uint8_t* s, const char* label, const uint8_t* msg, size_t n) {
  uint32_t len = (uint32_t)n;
  st_meta_ad(s, (const uint8_t*)label, strlen(label), 0); st_meta_ad(s, (const uint8_t*)&len, 4, 1);
  st_begin(s, 2, 0); st_absorb(s, msg, n);
}
static void tr_challenge(uint8_t* s, uint8_t* out, size_t n, const char* label) {
  uint32_t len = (uint32_t)n;
  st_meta_ad(s, (const uint8_t*)label, strlen(label), 0); st_meta_ad(s, (const uint8_t*)&len, 4, 1);
  st_begin(s, 1 | 2 | 4, 0); st_squeeze(s, out, n);
}
void oracle_transcript_new(uint8_t* t203, const char* label) {
  static const uint8_t init[19] = {1, 168, 1, 0, 1, 96, 83, 84, 82, 79, 66, 69, 118, 49, 46, 48, 46, 50, 0};
  memset(t203, 0, 203); memcpy(t203, init, 19);
  keccakf(t203);
  st_meta_ad(t203, (const uint8_t*)"Merlin v1.0", 11, 0);
  tr_append(t203, "dom-sep", (const uint8_t*)label, strlen(label));
}
static sc ipa_challenge(uint8_t* t, const uint8_t* l32, const uint8_t* r32) {
  tr_append(t, "L", l32, 32); tr_append(t, "R", r32, 32);
  uint8_t buf[32]; tr_challenge(t, buf, 32, "x");
  return sc_reduce32(sc_load(buf));
}
static void ipa_init(uint8_t* t, u64 n) {
  const char* dom = "inner product proof v1";
  tr_append(t, "domain-sep", (const uint8_t*)dom, strlen(dom)); tr_append(t, "n", (const uint8_t*)&n, 8);
}
static void ge_scalarmult(ge* r, const ge* p, const sc* k) {
  ge acc; ge_identity(&acc);
  for (int i = 255; i >= 0; --i) { ge_dbl(&acc, &acc); if ((k->v[i >> 6] >> (i & 63)) & 1) ge_add(&acc, &acc, p); }
  *r = acc;
}
/* sum_i s_i * g_i with 32-byte scalars (naive double-and-add: the oracle favours obviousness) */
static void ge_msm(ge* r, const ge* g, const uint8_t* scalars, u64 n) {
  ge acc; ge_identity(&acc);
  for (u64 i = 0; i < n; ++i) { sc k = sc_load(scalars + 32 * i); ge t; ge_scalarmult(&t, &g[i], &k); ge_add(&acc, &acc, &t); }
  *r = acc;
}
static unsigned ipa_log2(u64 n) { unsigned k = 0; while ((1ull << k) < n) ++k; return k; }

/* Test-only encodings of a 32-byte little-endian s < p: the bytes a prover could emit for the same
 * decoded point, or for none. ENC_NEGATED writes p - s (odd, |p - s| = s), ENC_PLUS_P the 256-bit
 * integer s + p, ENC_TOP_BIT s + 2^255 (s to a decoder that drops bit 255), ENC_REPLACE the
 * caller's 32 bytes. */
enum { ENC_CANONICAL = 0, ENC_NEGATED = 1, ENC_PLUS_P = 2, ENC_TOP_BIT = 3, ENC_REPLACE = 4 };
static const uint8_t P25519_BYTES[32] = {0xed, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                         0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                         0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x7f};
static void ipa_reencode(uint8_t* s, uint8_t mode, const uint8_t* replacement) {
  u64 v[4], pw[4];
  memcpy(v, s, 32); memcpy(pw, P25519_BYTES, 32);
  if (mode == ENC_NEGATED) mf_subn(v, pw, v, 4);
  else if (mode == ENC_PLUS_P) mf_addn(v, v, pw, 4);
  else if (mode == ENC_TOP_BIT) v[3] |= 1ull << 63;
  else if (mode == ENC_REPLACE) memcpy(v, replacement, 32);
  memcpy(s, v, 32);
}

/* modes: NULL, or 2k bytes [L_0 .. L_(k-1) | R_0 .. R_(k-1)]; replacements: 2k * 32 bytes in the same
 * order, read for ENC_REPLACE; challenges: NULL, or k * 32 bytes for the round challenges x_j. Every
 * challenge is taken over the bytes emitted. */
static void prove_inner_product(uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value, uint8_t* t203,
                                u64 n, u64 generators_offset, const uint8_t* a_vector, const uint8_t* b_vector,
                                const uint8_t* modes, const uint8_t* replacements, uint8_t* challenges) {
  oracle_init(); sc_init();
  unsigned k = ipa_log2(n); u64 np = 1ull << k;
  ipa_init(t203, n);
  if (n == 1) { memcpy(ap_value, a_vector, 32); return; }
  ge* G = (ge*)malloc(sizeof(ge) * (np + 1));
  for (u64 i = 0; i <= np; ++i) builtin_generator(&G[i], generators_offset + i);
  ge Q = G[np];
  uint8_t* a = (uint8_t*)malloc(32 * np); uint8_t* b = (uint8_t*)malloc(32 * np);
  memcpy(a, a_vector, 32 * n); memcpy(b, b_vector, 32 * n);
  u64 na = n, nb = n, len = np;
  for (unsigned round = 0; round < k; ++round) {
    u64 mid = len / 2, a_hi = na - mid, b_hi = nb - mid;
    sc c_l = sc_inner(a, b + 32 * mid, mid < b_hi ? mid : b_hi);
    sc c_r = sc_inner(a + 32 * mid, b, a_hi < mid ? a_hi : mid);
    ge L, R, t;
    ge_msm(&L, G + mid, a, mid); ge_scalarmult(&t, &Q, &c_l); ge_add(&L, &L, &t);
    ge_msm(&R, G, a + 32 * mid, a_hi); ge_scalarmult(&t, &Q, &c_r); ge_add(&R, &R, &t);
    ristretto_encode(l_vector + 32 * round, &L); ristretto_encode(r_vector + 32 * round, &R);
    if (modes) {
      ipa_reencode(l_vector + 32 * round, modes[round], replacements + 32 * round);
      ipa_reencode(r_vector + 32 * round, modes[k + round], replacements + 32 * (k + round));
    }
    sc x = ipa_challenge(t203, l_vector + 32 * round, r_vector + 32 * round), xi = sc_inv(x);
    if (challenges) memcpy(challenges + 32 * round, x.v, 32);
    for (u64 i = 0; i < mid; ++i) { /* a' = x a_lo + x^-1 a_hi (zero padded) */
      sc v = sc_mul(x, sc_load(a + 32 * i));
      if (i < a_hi) v = sc_add(v, sc_mul(xi, sc_load(a + 32 * (mid + i))));
      memcpy(a + 32 * i, v.v, 32);
    }
    na = mid;
    if (mid == 1) break;
    for (u64 i = 0; i < mid; ++i) { /* b' = x^-1 b_lo + x b_hi */
      sc v = sc_mul(xi, sc_load(b + 32 * i));
      if (i < b_hi) v = sc_add(v, sc_mul(x, sc_load(b + 32 * (mid + i))));
      memcpy(b + 32 * i, v.v, 32);
    }
    nb = mid;
    for (u64 i = 0; i < mid; ++i) { /* G' = x^-1 G_lo + x G_hi */
      ge lo, hi; ge_scalarmult(&lo, &G[i], &xi); ge_scalarmult(&hi, &G[mid + i], &x); ge_add(&G[i], &lo, &hi);
    }
    len = mid;
  }
  memcpy(ap_value, a, 32);
  free(G); free(a); free(b);
}
void oracle_prove_inner_product(uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value, uint8_t* t203,
                                u64 n, u64 generators_offset, const uint8_t* a_vector, const uint8_t* b_vector) {
  prove_inner_product(l_vector, r_vector, ap_value, t203, n, generators_offset, a_vector, b_vector, NULL,
                      NULL, NULL);
}
void oracle_prove_inner_product_encoded(uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
                                        uint8_t* t203, u64 n, u64 generators_offset, const uint8_t* a_vector,
                                        const uint8_t* b_vector, const uint8_t* modes,
                                        const uint8_t* replacements, uint8_t* challenges) {
  prove_inner_product(l_vector, r_vector, ap_value, t203, n, generators_offset, a_vector, b_vector, modes,
                      replacements, challenges);
}

/* ristretto255 decoding (RFC 9496 4.3.1; sxt/ristretto/base/byte_conversion.cc:135-). Test-only lax
 * decoders skip the checks named in the LAX_* bits of `lax`; LAX_MOD_P reads s as the 256-bit integer
 * mod p instead of from its low 255 bits. */
enum { LAX_NONE = 0, LAX_CANONICAL = 1, LAX_SIGN = 2, LAX_MOD_P = 4, LAX_T = 8, LAX_Y = 16 };
static int ristretto_decode_lax(ge* p, const uint8_t* bytes, int lax) {
  fe s, ss, u1, u2, u2sq, v, t, inv_sqrt, den_x, den_y;
  uint8_t back[32];
  fe_frombytes(&s, bytes); fe_tobytes(back, &s);
  if ((lax & LAX_MOD_P) && (bytes[31] & 0x80)) { /* 2^255 = 19 */
    fe nineteen = {{19, 0, 0, 0, 0}};
    fe_add(&s, &s, &nineteen);
  }
  if (!(lax & LAX_CANONICAL) && memcmp(back, bytes, 32) != 0) return 0;
  if (!(lax & LAX_SIGN) && (bytes[0] & 1)) return 0;
  fe_sq(&ss, &s); fe_sub(&u1, &FE_ONE, &ss); fe_add(&u2, &FE_ONE, &ss); fe_sq(&u2sq, &u2);
  fe_sq(&t, &u1); fe_mul(&t, &t, &FE_D); fe_neg(&v, &t); fe_sub(&v, &v, &u2sq);
  fe_mul(&t, &v, &u2sq);
  int was_square = sqrt_ratio_m1(&inv_sqrt, &FE_ONE, &t);
  fe_mul(&den_x, &inv_sqrt, &u2); fe_mul(&den_y, &inv_sqrt, &den_x); fe_mul(&den_y, &den_y, &v);
  fe_mul(&p->X, &s, &den_x); fe_add(&p->X, &p->X, &p->X); fe_abs(&p->X, &p->X);
  fe_mul(&p->Y, &u1, &den_y); p->Z = FE_ONE; fe_mul(&p->T, &p->X, &p->Y);
  return was_square && ((lax & LAX_T) || !fe_isneg(&p->T)) && ((lax & LAX_Y) || !fe_iszero(&p->Y));
}
static int ristretto_decode(ge* p, const uint8_t* bytes) { return ristretto_decode_lax(p, bytes, LAX_NONE); }

int oracle_verify_inner_product_lax(uint8_t* t203, u64 n, u64 generators_offset, const uint8_t* b_vector,
                                    const uint8_t* product, const uint8_t* a_commit160,
                                    const uint8_t* l_vector, const uint8_t* r_vector, const uint8_t* ap_value,
                                    int lax) {
  oracle_init(); sc_init();
  unsigned k = ipa_log2(n); u64 np = 1ull << k;
  ipa_init(t203, n);
  sc* x = (sc*)malloc(sizeof(sc) * (k ? k : 1));
  for (unsigned j = 0; j < k; ++j) x[j] = ipa_challenge(t203, l_vector + 32 * j, r_vector + 32 * j);
  ge* G = (ge*)malloc(sizeof(ge) * (np + 1));
  for (u64 i = 0; i <= np; ++i) builtin_generator(&G[i], generators_offset + i);
  /* s_i = ap * prod_j x_j^(+-1), bit t of i <-> x_{k-1-t} */
  sc ap = sc_load(ap_value), allinv = {{1, 0, 0, 0}};
  for (unsigned j = 0; j < k; ++j) allinv = sc_mul(allinv, sc_inv(x[j]));
  sc* g = (sc*)malloc(sizeof(sc) * np);
  g[0] = sc_mul(allinv, ap);
  u64 filled = 1;
  for (unsigned t = 0; t < k; ++t) { sc m = sc_mul(x[k - 1 - t], x[k - 1 - t]); for (u64 i = 0; i < filled; ++i) g[filled + i] = sc_mul(m, g[i]); filled *= 2; }
  sc prod = {{0, 0, 0, 0}};
  for (u64 i = 0; i < n; ++i) prod = sc_add(prod, sc_mul(g[i], sc_load(b_vector + 32 * i)));
  ge expected, t; ge_scalarmult(&expected, &G[np], &prod);
  for (u64 i = 0; i < np; ++i) { ge_scalarmult(&t, &G[i], &g[i]); ge_add(&expected, &expected, &t); }
  int ok = 1;
  for (unsigned j = 0; j < k; ++j) {
    ge Lp, Rp; sc xi = sc_inv(x[j]);
    sc el = sc_neg(sc_mul(x[j], x[j])), er = sc_neg(sc_mul(xi, xi));
    ok &= ristretto_decode_lax(&Lp, l_vector + 32 * j, lax);
    ok &= ristretto_decode_lax(&Rp, r_vector + 32 * j, lax);
    if (!ok) break;
    ge_scalarmult(&t, &Lp, &el); ge_add(&expected, &expected, &t);
    ge_scalarmult(&t, &Rp, &er); ge_add(&expected, &expected, &t);
  }
  ge commit, A; sc pr = sc_load(product);
  memcpy(&A, a_commit160, 160);
  ge_scalarmult(&commit, &G[np], &pr); ge_add(&commit, &commit, &A);
  uint8_t e1[32], e2[32]; ristretto_encode(e1, &expected); ristretto_encode(e2, &commit);
  free(x); free(G); free(g);
  return ok && memcmp(e1, e2, 32) == 0;
}
int oracle_verify_inner_product(uint8_t* t203, u64 n, u64 generators_offset, const uint8_t* b_vector,
                                const uint8_t* product, const uint8_t* a_commit160, const uint8_t* l_vector,
                                const uint8_t* r_vector, const uint8_t* ap_value) {
  return oracle_verify_inner_product_lax(t203, n, generators_offset, b_vector, product, a_commit160,
                                         l_vector, r_vector, ap_value, LAX_NONE);
}
