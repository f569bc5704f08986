// Inner-product argument (Bulletproofs-style) over ristretto255 on top of the MSM engine:
// sxt_curve25519_prove_inner_product / sxt_curve25519_verify_inner_product (SURVEY §8f N1).
//
// Replaces sxt/proof/inner_product/{proof_computation,gpu_driver,fold,generator_fold,
// verification_computation}.cc (+ generator_fold_kernel / scalar_fold_kernel). Protocol restated
// from cbindings/blitzar_api.h:479-611 and proof_computation.cc:61-155:
//   round j: L = <a_lo, G_hi> + <a_lo, b_hi> Q,  R = <a_hi, G_lo> + <a_hi, b_lo> Q
//            x  = transcript("L", L; "R", R; challenge "x")
//            a' = x a_lo + x^-1 a_hi,  b' = x^-1 b_lo + x b_hi,  G' = x^-1 G_lo + x G_hi
// Generators stay resident in HBM across rounds (folded in place by one kernel); the two MSMs of a
// round run through the Pippenger engine; scalar folds and the transcript are host work.
#pragma once
#include <vector>

#include "engine.cuh"
#include "transcript.h"

namespace b200 {

// G'[i] = m_lo * G[i] + m_hi * G[mid + i] by a shared-doubling (Shamir) ladder; the two scalars are
// the same for every thread, so the table index is warp-uniform.
struct FoldGeneratorsBody {
  static constexpr int kBlock = 64;
  const Ed25519::Gen* g;
  u32 mid;
  u32 m_lo[8], m_hi[8];
  Ed25519::Gen* out;
  B200_HD void operator()(u64 i) const {
    typedef Ed25519 C;
    C::Gen table[3];
    table[0] = g[i];
    table[1] = g[(u64)mid + i];
    C::Point p0, p1, p2;
    C::gen_to_point(p0, table[0], false);
    C::gen_to_point(p1, table[1], false);
    C::add(p2, p0, p1);
    C::point_to_gen(table[2], p2);
    C::Point acc = C::identity();
    for (int bit = 252; bit >= 0; --bit) {
      C::dbl(acc, acc);
      u32 sel = ((m_lo[bit >> 5] >> (bit & 31)) & 1u) | (((m_hi[bit >> 5] >> (bit & 31)) & 1u) << 1);
      if (sel)
        C::add_gen(acc, acc, table[sel - 1], false);
    }
    C::Gen r;
    C::point_to_gen(r, acc);
    out[i] = r;
  }
};
// compressed ristretto points -> device generator layout (invalid encodings become the identity
// and raise *bad)
struct DecodeToGenBody {
  static constexpr int kBlock = 32;
  const unsigned char* bytes;
  Ed25519::Gen* out;
  u32* bad;
  B200_HD void operator()(u64 i) const {
    Ed25519::Point p;
    if (!Ed25519::decode(p, bytes + 32 * i)) {
      p = Ed25519::identity();
      B200_ATOMIC_ADD(bad, 1u);
    }
    Ed25519::point_to_gen(out[i], p);
  }
};

// ---- scalar work of the prover on the device (FSc25: Montgomery arithmetic mod l on 8 x u32 limbs;
// a 32-byte little-endian scalar IS an FSc25 element in plain form). Replaces the reference's
// scalar_fold_kernel / inner-product kernels (sxt/proof/inner_product/gpu_driver.cc:104-221,
// sxt/scalar25/operation/inner_product.cc). mul(x R, y) = x y keeps vectors in plain form.
typedef FSc25 FS;
typedef FS::E ScE;
B200_HD ScE sc_r2() {
  ScE r;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    r.l[i] = Sc25Params::r2(i);
  return r;
}
// any 256-bit value -> canonical residue (s25o::reduce32)
struct IpaReduceBody {
  static constexpr int kBlock = 128;
  ScE* v;
  B200_HD void operator()(u64 i) const {
    ScE t;
    FS::mul(t, v[i], sc_r2());
    FS::from_mont(v[i], t);
  }
};
// per-thread partial sums of <a_lo, b_hi> and <a_hi, b_lo> (each product carries a factor R^-1)
struct IpaDotBody {
  static constexpr int kBlock = 64;
  const ScE* a;
  const ScE* b;
  u64 mid, nl, nr;  // products in the left / right sum
  u32 K;
  ScE* partial;  // 2 per thread
  B200_HD void operator()(u64 t) const {
    ScE cl = FS::zero(), cr = FS::zero(), p;
    const u64 b0 = t * K, e0 = b0 + K;
    for (u64 i = b0; i < e0; ++i) {
      if (i < nl) {
        FS::mul(p, a[i], b[mid + i]);
        FS::add(cl, cl, p);
      }
      if (i < nr) {
        FS::mul(p, a[mid + i], b[i]);
        FS::add(cr, cr, p);
      }
    }
    partial[2 * t] = cl;
    partial[2 * t + 1] = cr;
  }
};
// sums the partials (thread 0: left, thread 1: right), removes the R^-1 and writes the scalar of Q
struct IpaDotFinalBody {
  static constexpr int kBlock = 32;
  const ScE* partial;
  u64 T;
  ScE* out_l;
  ScE* out_r;
  B200_HD void operator()(u64 side) const {
    ScE acc = FS::zero();
    for (u64 t = 0; t < T; ++t)
      FS::add(acc, acc, partial[2 * t + side]);
    FS::mul(acc, acc, sc_r2());
    *(side ? out_r : out_l) = acc;
  }
};
// out[i] = m_lo * v[i] + m_hi * v[mid + i] (v zero-padded to 2 mid; prfip::fold_scalars); the
// multipliers are in Montgomery form
struct IpaFoldScalarsBody {
  static constexpr int kBlock = 128;
  const ScE* v;
  u64 mid, hi;  // hi = number of elements in the upper half
  ScE m_lo, m_hi;
  ScE* out;
  B200_HD void operator()(u64 i) const {
    ScE t, u;
    FS::mul(t, m_lo, v[i]);
    if (i < hi) {
      FS::mul(u, m_hi, v[mid + i]);
      FS::add(t, t, u);
    }
    out[i] = t;
  }
};

// The two MSMs of a round as TWO COLUMNS of one engine call over the generator array
// [G_lo | G_hi | Q] (len + 1 entries): column L = [0 .. 0 | a_lo | c_L], column R = [a_hi, 0 .. | 0 .. 0
// | c_R]. Zero scalars produce no bucket entries, and the latency-bound tail of a small MSM (bucket
// reduction, 240 Horner doublings, ristretto encoding) is paid once per round instead of twice.
struct IpaRoundColumnsBody {
  static constexpr int kBlock = 128;
  const ScE* a;
  const ScE* cq;  // c_L, c_R
  u64 mid, a_hi;
  ScE* col_l;  // 2 mid + 1 entries each
  ScE* col_r;
  B200_HD void operator()(u64 i) const {
    const ScE zero = FS::zero();
    if (i < mid) {
      col_l[i] = zero;
      col_l[mid + i] = a[i];
      col_r[i] = i < a_hi ? a[mid + i] : zero;
      col_r[mid + i] = zero;
    } else {
      col_l[2 * mid] = cq[0];
      col_r[2 * mid] = cq[1];
    }
  }
};

// verifier exponents g_i = ap * prod_j x_j^(+-1) (prfip::compute_verification_exponents,
// sxt/proof/inner_product/verification_computation.cc:86-127): g_0 = ap * prod_j x_j^-1 and every set
// bit t of i multiplies by x_(k-1-t)^2. One thread per i, at most k products; the multipliers are in
// Montgomery form, so the values stay in plain form.
struct IpaVerifyExponentsBody {
  static constexpr int kBlock = 128;
  ScE g0;            // plain form
  const ScE* xsq_m;  // k squares of the challenges, Montgomery form
  u32 k;
  ScE* out;          // np entries
  B200_HD void operator()(u64 i) const {
    ScE g = g0;
    for (u32 t = 0; t < k; ++t)
      if ((i >> t) & 1u)
        FS::mul(g, xsq_m[k - 1 - t], g);
    out[i] = g;
  }
};
// per-thread partial sums of <g, b> (each product carries a factor R^-1; slot 2t + 1 stays zero so
// that IpaDotFinalBody can finish the sum)
struct IpaDot1Body {
  static constexpr int kBlock = 64;
  const ScE* a;
  const ScE* b;
  u64 n;
  u32 K;
  ScE* partial;
  B200_HD void operator()(u64 t) const {
    ScE acc = FS::zero(), p;
    const u64 b0 = t * K, e0 = b0 + K < n ? b0 + K : n;
    for (u64 i = b0; i < e0; ++i) {
      FS::mul(p, a[i], b[i]);
      FS::add(acc, acc, p);
    }
    partial[2 * t] = acc;
    partial[2 * t + 1] = FS::zero();
  }
};

struct Ipa {
  typedef Ed25519 C;
  typedef CurveOps<C> Ops;

  static unsigned ceil_log2(uint64_t n) {
    unsigned k = 0;
    while ((1ull << k) < n)
      ++k;
    return k;
  }
  static void scalar_words(u32 w[8], const Sc& s) {
    for (int i = 0; i < 4; ++i) {
      w[2 * i] = (u32)s.v[i];
      w[2 * i + 1] = (u32)(s.v[i] >> 32);
    }
  }
  // device generators g(offset .. offset+count): the precomputed table when it covers the range
  static const C::Gen* generators(const EngineCtx& ctx, DevBuf<C::Gen>& storage, uint64_t offset,
                                  uint64_t count) {
    if (offset + count <= ctx.num_builtin)
      return (const C::Gen*)ctx.builtin + offset;
    launch(BuiltinGeneratorBody{storage.p, offset}, count, ctx.s);
    return storage.p;
  }
  // both points of a round: out64_dev = [L | R] encodings; gens = [G (len) | Q]
  static void round_msms_device(const EngineCtx& ctx, unsigned char* out64_dev, const C::Gen* gens_q,
                                uint64_t len, const ScE* col_l, const ScE* col_r) {
    stream_t s = ctx.s;
    std::vector<ColumnDesc> cols(2);
    for (int j = 0; j < 2; ++j) {
      cols[j].base = (const unsigned char*)(j ? col_r : col_l);
      cols[j].row_stride = 32;
      cols[j].bit_offset = 0;
      cols[j].bit_width = 256;
      cols[j].n = (u32)(len + 1);
      cols[j].is_signed = 0;
      cols[j].first_window = cols[j].num_windows = 0;
    }
    DevBuf<C::Point> pt(2, s);
    Ops::run_columns(ctx, gens_q, cols, pt.p);
    launch_store_commit<C>(s, pt.p, out64_dev, 2, ctx.opt.lane_tail != 0);
  }
  static ScE to_device_mont(const Sc& x) {  // x R mod l as device limbs
    const Sc m = sc_to_mont(x);
    ScE r;
    for (int i = 0; i < 4; ++i) {
      r.l[2 * i] = (u32)m.v[i];
      r.l[2 * i + 1] = (u32)(m.v[i] >> 32);
    }
    return r;
  }
  static void init_transcript(Transcript& t, uint64_t n) {
    const char* domain = "inner product proof v1";
    t.append_message("domain-sep", (const uint8_t*)domain, std::strlen(domain));
    t.append_message("n", (const uint8_t*)&n, 8);
  }
  static Sc round_challenge(Transcript& t, const uint8_t* l32, const uint8_t* r32) {
    t.append_message("L", l32, 32);
    t.append_message("R", r32, 32);
    return t.challenge_scalar("x");
  }

  static void prove(const EngineCtx& ctx, uint8_t* l_vector, uint8_t* r_vector, uint8_t* ap_value,
                    uint8_t* transcript203, uint64_t n, uint64_t generators_offset,
                    const uint8_t* a_vector, const uint8_t* b_vector) {
    stream_t s = ctx.s;
    const unsigned k = ceil_log2(n);
    const uint64_t np = 1ull << k;
    Transcript tr(transcript203);
    init_transcript(tr, n);
    if (n == 1) {
      std::memcpy(ap_value, a_vector, 32);
      return;
    }
    DevBuf<C::Gen> gstore(np + 1, s);
    const C::Gen* G0 = generators(ctx, gstore, generators_offset, np + 1);
    const C::Gen* Q = G0 + np;
    // folded generators: every buffer keeps Q in the slot after its last generator
    DevBuf<C::Gen> gwork(np / 2 + 1, s), gwork2(np / 4 + 2, s);
    const C::Gen* G = G0;  // G0[np] is Q already
    // a, b live in HBM for the whole proof (ping-pong halves); the host sees only L, R (64 bytes) and
    // the challenge of every round — one stream synchronisation per round, for the transcript
    DevBuf<ScE> abuf(np + np / 2 + 2, s), bbuf(np + np / 2 + 2, s);
    ScE* a = abuf.p;
    ScE* b = bbuf.p;
    ScE* a_next = abuf.p + np;
    ScE* b_next = bbuf.p + np;
    copy_h2d(a, a_vector, 32 * n, s);
    copy_h2d(b, b_vector, 32 * n, s);
    launch(IpaReduceBody{a}, n, s);
    launch(IpaReduceBody{b}, n, s);
    const u32 K = 64;
    DevBuf<ScE> partial(2 * ((np / 2 + K - 1) / K) + 2, s), cq(2, s), col_l(np + 1, s),
        col_r(np + 1, s);
    DevBuf<unsigned char> lr(64, s);
    uint64_t len = np, na = n, nb = n;
    for (unsigned round = 0; round < k; ++round) {
      const uint64_t mid = len / 2;
      const uint64_t a_hi = na - mid, b_hi = nb - mid;
      const uint64_t nl = std::min<uint64_t>(mid, b_hi), nr = std::min<uint64_t>(a_hi, mid);
      const uint64_t T = (mid + K - 1) / K;
      launch(IpaDotBody{a, b, mid, nl, nr, K, partial.p}, T, s);
      launch(IpaDotFinalBody{partial.p, T, cq.p, cq.p + 1}, 2, s);
      uint8_t* l_out = l_vector + 32 * round;
      uint8_t* r_out = r_vector + 32 * round;
      launch(IpaRoundColumnsBody{a, cq.p, mid, a_hi, col_l.p, col_r.p}, mid + 1, s);
      round_msms_device(ctx, lr.p, G, len, col_l.p, col_r.p);
      uint8_t lr_host[64];
      copy_d2h(lr_host, lr.p, 64, s);
      stream_sync(s);
      std::memcpy(l_out, lr_host, 32);
      std::memcpy(r_out, lr_host + 32, 32);
      Sc x = round_challenge(tr, l_out, r_out);
      Sc x_inv = sc_inv(x);
      const ScE xm = to_device_mont(x), xim = to_device_mont(x_inv);
      launch(IpaFoldScalarsBody{a, mid, a_hi, xm, xim, a_next}, mid, s);
      std::swap(a, a_next);
      na = mid;
      if (mid == 1)
        break;
      launch(IpaFoldScalarsBody{b, mid, b_hi, xim, xm, b_next}, mid, s);
      std::swap(b, b_next);
      nb = mid;
      FoldGeneratorsBody body;
      body.g = G;
      body.mid = (u32)mid;
      scalar_words(body.m_lo, x_inv);
      scalar_words(body.m_hi, x);
      C::Gen* gout = (G == gwork.p) ? gwork2.p : gwork.p;
      body.out = gout;
      launch(body, mid, s);
      copy_d2d(gout + mid, Q, sizeof(C::Gen), s);
      G = gout;
      len = mid;
    }
    copy_d2h(ap_value, a, 32, s);
    stream_sync(s);
  }
};

// ---- many independent proofs per call (IpaBatch) ----------------------------------------------------
// Round r of every proof with r < k_p runs in the same launches. Each segmented body below finds its
// proof by binary search (column_of) over a prefix of per-proof thread counts, reads the proof's row of
// a small per-round table and runs the single-proof body's element code on the proof's segment.
// Element segments are padded to whole kIpaPad threads, so that a warp never spans two proofs and the
// ladder index of FoldGeneratorsBody stays warp-uniform.
constexpr u64 kIpaPad = 64;
struct IpaRoundRow {  // one proof in one round of the batched prover
  u64 a_off;          // its scalars in the a / b arenas (np_p entries)
  u64 col_off;        // its two engine columns, 2 (len + 1) scalars
  u64 gin, gout;      // its generators [G (len) | Q] read and [G' (mid) | Q] written this round
  u64 mid, a_hi, b_hi, nl, nr;
  u64 proof;          // index in the batch (ap output slot)
};
struct IpaChallengeRow {  // x and x^-1 of the round: plain (ladder words) and Montgomery form
  ScE x, xi, xm, xim;
};
struct IpaSegments {  // thread t belongs to proof column_of(start, count, t)
  const u64* start;   // [count + 1]
  u32 count;
  B200_HD u32 of(u64 t) const { return column_of(start, count, t); }
};

// concatenated caller scalars (proof p from start[p]) -> the proofs' arena segments, reduced
struct IpaLoadBody {
  static constexpr int kBlock = 128;
  IpaSegments seg;
  const u64* dst_off;
  const ScE* src;
  ScE* dst;
  B200_HD void operator()(u64 i) const {
    const u32 p = seg.of(i);
    ScE t;
    FS::mul(t, src[i], sc_r2());
    FS::from_mont(dst[dst_off[p] + (i - seg.start[p])], t);
  }
};
// IpaDotBody per proof (ceil(mid / K) threads each); partials in the proof's thread range
struct IpaDotSegBody {
  static constexpr int kBlock = 64;
  IpaSegments seg;
  const IpaRoundRow* rows;
  const ScE* a;
  const ScE* b;
  u32 K;
  ScE* partial;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaRoundRow& r = rows[p];
    IpaDotBody{a + r.a_off, b + r.a_off, r.mid, r.nl, r.nr, K, partial + 2 * seg.start[p]}(
        t - seg.start[p]);
  }
};
// thread pair (2p, 2p + 1) finishes proof p's left and right sums into cq[2p], cq[2p + 1]
struct IpaDotFinalSegBody {
  static constexpr int kBlock = 32;
  IpaSegments seg;  // the dot threads' segments
  const ScE* partial;
  ScE* cq;
  B200_HD void operator()(u64 t) const {
    const u64 p = t >> 1;
    IpaDotFinalBody{partial + 2 * seg.start[p], seg.start[p + 1] - seg.start[p], cq + 2 * p,
                    cq + 2 * p + 1}(t & 1);
  }
};
// IpaRoundColumnsBody per proof (mid + 1 threads of the padded segment)
struct IpaRoundColumnsSegBody {
  static constexpr int kBlock = 128;
  IpaSegments seg;
  const IpaRoundRow* rows;
  const ScE* a;
  const ScE* cq;
  ScE* cols;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaRoundRow& r = rows[p];
    const u64 i = t - seg.start[p];
    if (i > r.mid)
      return;
    ScE* col_l = cols + r.col_off;
    IpaRoundColumnsBody{a + r.a_off, cq + 2 * p, r.mid, r.a_hi, col_l, col_l + 2 * r.mid + 1}(i);
  }
};
// IpaFoldScalarsBody per proof: a (b_side 0: x a_lo + x^-1 a_hi; in its last round, mid == 1, the
// folded value is also proof p's ap) or b (b_side 1: x^-1 b_lo + x b_hi; not in the last round)
struct IpaFoldScalarsSegBody {
  static constexpr int kBlock = 128;
  IpaSegments seg;
  const IpaRoundRow* rows;
  const IpaChallengeRow* ch;
  const ScE* v;
  ScE* out;
  u32 b_side;
  ScE* ap;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaRoundRow& r = rows[p];
    const u64 i = t - seg.start[p];
    if (i >= r.mid || (b_side && r.mid == 1))
      return;
    const IpaChallengeRow& c = ch[p];
    IpaFoldScalarsBody{v + r.a_off, r.mid, b_side ? r.b_hi : r.a_hi, b_side ? c.xim : c.xm,
                       b_side ? c.xm : c.xim, out + r.a_off}(i);
    if (!b_side && r.mid == 1)
      ap[r.proof] = out[r.a_off];
  }
};
// FoldGeneratorsBody per proof (G' = x^-1 G_lo + x G_hi); thread mid carries Q over. Not in the last
// round.
struct FoldGeneratorsSegBody {
  static constexpr int kBlock = FoldGeneratorsBody::kBlock;
  IpaSegments seg;
  const IpaRoundRow* rows;
  const IpaChallengeRow* ch;
  const Ed25519::Gen* gin;
  Ed25519::Gen* gout;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaRoundRow& r = rows[p];
    const u64 i = t - seg.start[p];
    if (i > r.mid || r.mid == 1)
      return;
    if (i == r.mid) {
      gout[r.gout + r.mid] = gin[r.gin + 2 * r.mid];
      return;
    }
    FoldGeneratorsBody body;
    body.g = gin + r.gin;
    body.mid = (u32)r.mid;
    const IpaChallengeRow& c = ch[p];
    for (int w = 0; w < 8; ++w) {
      body.m_lo[w] = c.xi.l[w];
      body.m_hi[w] = c.x.l[w];
    }
    body.out = gout + r.gout;
    body(i);
  }
};

struct IpaVerifyRow {  // one proof of the batched verifier
  u64 e_off;           // its exponents [product', g (np), -x_j^2 (k), -x_j^-2 (k)]
  u64 g_off;           // its generators [Q, G (np), L_j (k), R_j (k)]
  u64 b_off;           // its b in the concatenated (reduced) b vectors
  u64 ch_off;          // its k challenges in xsq_m, and 2k tail values / L,R encodings from 2 ch_off
  u64 n, np, offset;
  u32 k, builtin;      // builtin: g(offset .. offset + np] lies in the precomputed table
  ScE g0;              // g_0 (plain form)
  ScE product1;        // n == 1: product' as the single call computes it on the host
};
// g(offset + i) for i <= np: G_i to slot 1 + i, Q to slot 0 and to the proof's [Q, A] pair
struct IpaVerifyGensBody {
  static constexpr int kBlock = 64;
  IpaSegments seg;  // np + 1 threads per proof
  const IpaVerifyRow* rows;
  const Ed25519::Gen* builtin;
  Ed25519::Gen* gens;
  Ed25519::Gen* pairs;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaVerifyRow& r = rows[p];
    const u64 i = t - seg.start[p];
    Ed25519::Gen g;
    if (r.builtin) {
      g = builtin[r.offset + i];
    } else {
      Ed25519::Point pt;
      Ed25519::builtin_generator(pt, r.offset + i);
      Ed25519::point_to_gen(g, pt);
    }
    if (i < r.np) {
      gens[r.g_off + 1 + i] = g;
    } else {
      gens[r.g_off] = g;
      pairs[2 * p] = g;
    }
  }
};
// L_j, R_j of proof p (packed [L (k) | R (k)] from 64 ch_off) -> generators, bad encodings to bad[p]
struct IpaVerifyDecodeBody {
  static constexpr int kBlock = 32;
  IpaSegments seg;  // 2k threads per proof
  const IpaVerifyRow* rows;
  const unsigned char* lr;
  Ed25519::Gen* gens;
  u32* bad;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaVerifyRow& r = rows[p];
    DecodeToGenBody{lr + 64 * r.ch_off, gens + r.g_off + 1 + r.np, bad + p}(t - seg.start[p]);
  }
};
struct IpaVerifyCommitsBody {  // a_commit p (ABI struct) -> the second generator of pair p
  static constexpr int kBlock = 32;
  const unsigned char* raw;
  Ed25519::Gen* pairs;
  B200_HD void operator()(u64 p) const {
    IngestBody<Ed25519, false>{raw + p * Ed25519::kAbiGenBytes, pairs + 2 * p + 1}(0);
  }
};
// IpaVerifyExponentsBody per proof (np threads) followed by the 2k tail values
struct IpaVerifyExponentsSegBody {
  static constexpr int kBlock = 128;
  IpaSegments seg;  // np + 2k threads per proof
  const IpaVerifyRow* rows;
  const ScE* xsq_m;
  const ScE* tail;
  ScE* e;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaVerifyRow& r = rows[p];
    const u64 i = t - seg.start[p];
    if (i < r.np)
      IpaVerifyExponentsBody{r.g0, xsq_m + r.ch_off, r.k, e + r.e_off + 1}(i);
    else
      e[r.e_off + 1 + i] = tail[2 * r.ch_off + (i - r.np)];
  }
};
// IpaDot1Body per proof (ceil(n / K) threads): <g, b>
struct IpaDot1SegBody {
  static constexpr int kBlock = 64;
  IpaSegments seg;
  const IpaVerifyRow* rows;
  const ScE* e;
  const ScE* b;
  u32 K;
  ScE* partial;
  B200_HD void operator()(u64 t) const {
    const u32 p = seg.of(t);
    const IpaVerifyRow& r = rows[p];
    IpaDot1Body{e + r.e_off + 1, b + r.b_off, r.n, K, partial + 2 * seg.start[p]}(t - seg.start[p]);
  }
};
// thread p writes proof p's product' (the host's value when n == 1)
struct IpaDot1FinalSegBody {
  static constexpr int kBlock = 32;
  IpaSegments seg;  // the dot threads' segments
  const IpaVerifyRow* rows;
  const ScE* partial;
  ScE* e;
  B200_HD void operator()(u64 p) const {
    const IpaVerifyRow& r = rows[p];
    if (r.n == 1) {
      e[r.e_off] = r.product1;
      return;
    }
    IpaDotFinalBody{partial + 2 * seg.start[p], seg.start[p + 1] - seg.start[p], e + r.e_off,
                    nullptr}(0);
  }
};

struct IpaBatch {
  typedef Ed25519 C;
  typedef CurveOps<C> Ops;
  static constexpr u32 K = 64;  // products per dot-product thread

  static ScE plain(const Sc& s) {
    ScE r;
    Ipa::scalar_words(r.l, s);
    return r;
  }
  static u64 pad(u64 v) { return (v + kIpaPad - 1) / kIpaPad * kIpaPad; }
  // Montgomery's trick: v[i] <- v[i]^-1 (0 stays 0, as sc_inv leaves it)
  static void batch_invert(std::vector<Sc>& v) {
    std::vector<Sc> pre(v.size());
    Sc acc = sc_one();
    for (size_t i = 0; i < v.size(); ++i) {
      pre[i] = acc;
      if (!sc_is_zero(v[i]))
        acc = sc_mul(acc, v[i]);
    }
    Sc inv = sc_inv(acc);
    for (size_t i = v.size(); i-- > 0;) {
      if (sc_is_zero(v[i]))
        continue;
      const Sc vi = v[i];
      v[i] = sc_mul(inv, pre[i]);
      inv = sc_mul(inv, vi);
    }
  }
  static bool sc_is_zero(const Sc& s) { return (s.v[0] | s.v[1] | s.v[2] | s.v[3]) == 0; }
  static ColumnDesc column(const void* base, u64 n, u64 gen_base) {
    ColumnDesc c = ColumnDesc();
    c.base = (const unsigned char*)base;
    c.row_stride = 32;
    c.bit_width = 256;
    c.n = (u32)n;
    c.gen_base = (u32)gen_base;
    return c;
  }
  // staged copy of a host table; freed (stream-ordered) by the caller
  template <class T> static const T* stage(stream_t s, const std::vector<T>& v) {
    return (const T*)stage_to_device(s, v.data(), v.size() * sizeof(T));
  }

  // Proof p as Ipa::prove alone; a, b, l, r concatenated in proof order (prefix sums of n_p, k_p).
  static void prove(const EngineCtx& ctx, uint32_t P, uint8_t* l_vectors, uint8_t* r_vectors,
                    uint8_t* ap_values, uint8_t* transcripts, const uint64_t* n,
                    const uint64_t* offsets, const uint8_t* a_vectors, const uint8_t* b_vectors) {
    stream_t s = ctx.s;
    std::vector<unsigned> k(P);
    std::vector<u64> np(P), kstart(P + 1, 0), nstart(P + 1, 0), a_off(P + 1, 0), gout(P + 1, 0);
    unsigned kmax = 0;
    bool direct = true;  // round 0 reads the precomputed generators in place
    for (uint32_t p = 0; p < P; ++p) {
      k[p] = Ipa::ceil_log2(n[p]);
      np[p] = 1ull << k[p];
      kstart[p + 1] = kstart[p] + k[p];
      nstart[p + 1] = nstart[p] + n[p];
      a_off[p + 1] = a_off[p] + np[p];
      gout[p + 1] = gout[p] + (k[p] ? np[p] / 2 + 1 : 0);
      kmax = std::max(kmax, k[p]);
      Transcript tr(transcripts + 203 * (size_t)p);
      Ipa::init_transcript(tr, n[p]);
      if (n[p] == 1)
        std::memcpy(ap_values + 32 * (size_t)p, a_vectors + 32 * nstart[p], 32);
      else if (offsets[p] + np[p] + 1 > ctx.num_builtin)
        direct = false;
    }
    if (kmax == 0)
      return;
    // scalars: one upload each, then reduced into per-proof segments of np_p (ping-pong arenas)
    const u64 total_n = nstart[P], total_np = a_off[P];
    DevBuf<ScE> raw(total_n, s), abuf(2 * total_np, s), bbuf(2 * total_np, s), ap_dev(P, s);
    ScE *a = abuf.p, *a_next = abuf.p + total_np, *b = bbuf.p, *b_next = bbuf.p + total_np;
    {
      std::vector<u64> block(nstart);  // [nstart (P + 1) | a_off (P)]
      block.insert(block.end(), a_off.begin(), a_off.end() - 1);
      const u64* d_block = stage(s, block);
      const IpaSegments seg{d_block, P};
      copy_h2d(raw.p, a_vectors, 32 * total_n, s);
      launch(IpaLoadBody{seg, d_block + P + 1, raw.p, a}, total_n, s);
      copy_h2d(raw.p, b_vectors, 32 * total_n, s);
      launch(IpaLoadBody{seg, d_block + P + 1, raw.p, b}, total_n, s);
      dev_free((void*)d_block, s);
    }
    // generators: round 0 reads [G_p (np_p) | Q_p] from the precomputed table at offset_p, or from
    // an arena generated in one launch; round r >= 1 from the folded arena of round r - 1
    std::vector<u64> gin(P, 0);
    DevBuf<C::Gen> g0(direct ? 1 : a_off[P] + P, s), ga(gout[P] + 1, s), gb(gout[P] + 1, s);
    const C::Gen* G = direct ? (const C::Gen*)ctx.builtin : g0.p;
    if (!direct) {
      std::vector<u64> pieces;  // [start (P + 1) | from (P) | to (P)], one piece per proof
      for (uint32_t p = 0; p <= P; ++p)
        pieces.push_back(a_off[p] + p);
      for (uint32_t p = 0; p < P; ++p)
        pieces.push_back(offsets[p]);
      for (uint32_t p = 0; p < P; ++p)
        pieces.push_back(a_off[p] + p);
      const u64* d_pieces = stage(s, pieces);
      launch(BuiltinPiecesBody{g0.p, GenPieces{d_pieces, d_pieces + P + 1, d_pieces + 2 * P + 1, P}},
             a_off[P] + P, s);
      dev_free((void*)d_pieces, s);
    }
    for (uint32_t p = 0; p < P; ++p)
      gin[p] = direct ? offsets[p] : a_off[p] + p;
    C::Gen* Gout = ga.p;
    DevBuf<ScE> cols(2 * (total_np + P), s), cq(2 * P, s);
    DevBuf<ScE> partial(2 * (total_np / (2 * K) + P) + 2, s);
    DevBuf<C::Point> pts(2 * P, s);
    DevBuf<unsigned char> enc(64 * P, s);
    std::vector<uint8_t> lr_host(64 * P);
    std::vector<u64> na(n, n + P), nb(n, n + P);
    std::vector<uint32_t> act;
    std::vector<IpaRoundRow> rows;
    std::vector<u64> starts;  // [element segments (A + 1) | dot segments (A + 1)]
    std::vector<Sc> x, xi;
    std::vector<IpaChallengeRow> chrows;
    std::vector<ColumnDesc> colv;
    for (unsigned round = 0; round < kmax; ++round) {
      act.clear();
      rows.clear();
      for (uint32_t p = 0; p < P; ++p)
        if (k[p] > round)
          act.push_back(p);
      const uint32_t A = (uint32_t)act.size();
      starts.assign(2 * (A + 1), 0);
      colv.clear();
      u64 col_off = 0;
      for (uint32_t q = 0; q < A; ++q) {
        const uint32_t p = act[q];
        const u64 len = np[p] >> round, mid = len / 2;
        IpaRoundRow r;
        r.a_off = a_off[p];
        r.col_off = col_off;
        r.gin = gin[p];
        r.gout = gout[p];
        r.mid = mid;
        r.a_hi = na[p] - mid;
        r.b_hi = nb[p] - mid;
        r.nl = std::min<u64>(mid, r.b_hi);
        r.nr = std::min<u64>(r.a_hi, mid);
        r.proof = p;
        rows.push_back(r);
        starts[q + 1] = starts[q] + pad(mid + 1);
        starts[A + 1 + q + 1] = starts[A + 1 + q] + (mid + K - 1) / K;
        colv.push_back(column(cols.p + col_off, len + 1, gin[p]));
        colv.push_back(column(cols.p + col_off + len + 1, len + 1, gin[p]));
        col_off += 2 * (len + 1);
      }
      const IpaRoundRow* d_rows = stage(s, rows);
      const u64* d_starts = stage(s, starts);
      const IpaSegments eseg{d_starts, A}, dseg{d_starts + A + 1, A};
      const u64 ethreads = starts[A], dthreads = starts[2 * A + 1];
      launch(IpaDotSegBody{dseg, d_rows, a, b, K, partial.p}, dthreads, s);
      launch(IpaDotFinalSegBody{dseg, partial.p, cq.p}, 2 * (u64)A, s);
      launch(IpaRoundColumnsSegBody{eseg, d_rows, a, cq.p, cols.p}, ethreads, s);
      // both MSMs of every active proof: one engine pass, one encoding launch, one copy back
      Ops::run_columns(ctx, G, colv, pts.p);
      launch_store_commit<C>(s, pts.p, enc.p, 2 * (u64)A, ctx.opt.lane_tail != 0);
      copy_d2h(lr_host.data(), enc.p, 64 * (size_t)A, s);
      stream_sync(s);
      x.resize(A);
      for (uint32_t q = 0; q < A; ++q) {
        const uint32_t p = act[q];
        uint8_t* l_out = l_vectors + 32 * (kstart[p] + round);
        uint8_t* r_out = r_vectors + 32 * (kstart[p] + round);
        std::memcpy(l_out, &lr_host[64 * q], 32);
        std::memcpy(r_out, &lr_host[64 * q + 32], 32);
        Transcript tr(transcripts + 203 * (size_t)p);
        x[q] = Ipa::round_challenge(tr, l_out, r_out);
      }
      xi = x;
      batch_invert(xi);
      chrows.resize(A);
      for (uint32_t q = 0; q < A; ++q)
        chrows[q] = IpaChallengeRow{plain(x[q]), plain(xi[q]), Ipa::to_device_mont(x[q]),
                                    Ipa::to_device_mont(xi[q])};
      const IpaChallengeRow* d_ch = stage(s, chrows);
      launch(IpaFoldScalarsSegBody{eseg, d_rows, d_ch, a, a_next, 0, ap_dev.p}, ethreads, s);
      launch(IpaFoldScalarsSegBody{eseg, d_rows, d_ch, b, b_next, 1, nullptr}, ethreads, s);
      launch(FoldGeneratorsSegBody{eseg, d_rows, d_ch, G, Gout}, ethreads, s);
      std::swap(a, a_next);
      std::swap(b, b_next);
      G = Gout;
      Gout = Gout == ga.p ? gb.p : ga.p;
      for (uint32_t q = 0; q < A; ++q) {
        const uint32_t p = act[q];
        na[p] = nb[p] = rows[q].mid;
        gin[p] = gout[p];
      }
      dev_free((void*)d_rows, s);
      dev_free((void*)d_starts, s);
      dev_free((void*)d_ch, s);
    }
    std::vector<uint8_t> ap_host(32 * (size_t)P);
    copy_d2h(ap_host.data(), ap_dev.p, 32 * (size_t)P, s);
    stream_sync(s);
    for (uint32_t p = 0; p < P; ++p)
      if (k[p])
        std::memcpy(ap_values + 32 * (size_t)p, &ap_host[32 * (size_t)p], 32);
  }

  // results[p] = 1 when proof p verifies, 0 otherwise (sxt_curve25519_verify_inner_product is a
  // batch of one); returns the number of accepted proofs
  static uint32_t verify(const EngineCtx& ctx, uint32_t P, int* results, uint8_t* transcripts,
                         const uint64_t* n, const uint64_t* offsets, const uint8_t* b_vectors,
                         const uint8_t* products, const uint8_t* a_commits, const uint8_t* l_vectors,
                         const uint8_t* r_vectors, const uint8_t* ap_values) {
    stream_t s = ctx.s;
    if (P == 0)
      return 0;
    std::vector<IpaVerifyRow> rows(P);
    std::vector<u64> starts(4 * (P + 1), 0);  // [gens (np + 1) | decode (2k) | exps (np + 2k) | dot]
    u64 sum_k = 0, e_total = 0, nsum = 0;
    std::vector<Sc> x;
    for (uint32_t p = 0; p < P; ++p) {
      IpaVerifyRow& r = rows[p];
      r.k = Ipa::ceil_log2(n[p]);
      r.n = n[p];
      r.np = 1ull << r.k;
      r.offset = offsets[p];
      r.builtin = offsets[p] + r.np + 1 <= ctx.num_builtin ? 1u : 0u;
      r.ch_off = sum_k;
      r.e_off = e_total;
      r.g_off = e_total;
      r.b_off = nsum;
      const u64 num = 1 + r.np + 2 * r.k;  // [Q, G, L, R] / [product', g, -x^2, -x^-2]
      Transcript tr(transcripts + 203 * (size_t)p);
      Ipa::init_transcript(tr, n[p]);
      for (unsigned j = 0; j < r.k; ++j)
        x.push_back(Ipa::round_challenge(tr, l_vectors + 32 * (sum_k + j),
                                         r_vectors + 32 * (sum_k + j)));
      starts[p + 1] = starts[p] + r.np + 1;
      starts[P + 1 + p + 1] = starts[P + 1 + p] + 2 * r.k;
      starts[2 * (P + 1) + p + 1] = starts[2 * (P + 1) + p] + r.np + 2 * r.k;
      starts[3 * (P + 1) + p + 1] = starts[3 * (P + 1) + p] + (r.n + K - 1) / K;
      sum_k += r.k;
      e_total += num;
      nsum += n[p];
    }
    // host work that depends on the challenges alone: 2k + 1 values per proof, one batch inversion
    std::vector<Sc> xinv(x);
    batch_invert(xinv);
    std::vector<ScE> xsq_m(sum_k + 1), tail(2 * sum_k + 1);
    std::vector<uint8_t> lr(64 * sum_k + 64), sc2(64 * (size_t)P);
    for (uint32_t p = 0; p < P; ++p) {
      IpaVerifyRow& r = rows[p];
      const Sc ap = sc_load(ap_values + 32 * (size_t)p);
      Sc allinv = sc_one();
      for (unsigned j = 0; j < r.k; ++j) {
        const u64 c = r.ch_off + j;
        allinv = sc_mul(allinv, xinv[c]);
        const Sc xs = sc_mul(x[c], x[c]);
        tail[2 * r.ch_off + j] = plain(sc_neg(xs));
        tail[2 * r.ch_off + r.k + j] = plain(sc_neg(sc_mul(xinv[c], xinv[c])));
        xsq_m[c] = plain(sc_to_mont(xs));
      }
      if (r.k) {
        std::memcpy(&lr[64 * r.ch_off], l_vectors + 32 * r.ch_off, 32 * r.k);
        std::memcpy(&lr[64 * r.ch_off + 32 * r.k], r_vectors + 32 * r.ch_off, 32 * r.k);
      }
      if (r.n == 1) {
        r.g0 = plain(ap);
        r.product1 = plain(sc_mul(sc_load(b_vectors + 32 * r.b_off), ap));
      } else {
        r.g0 = plain(sc_mul(allinv, ap));
        r.product1 = FS::zero();
      }
      std::memcpy(&sc2[64 * (size_t)p], products + 32 * (size_t)p, 32);
      sc_store(&sc2[64 * (size_t)p + 32], sc_one());
    }
    const IpaVerifyRow* d_rows = stage(s, rows);
    const u64* d_starts = stage(s, starts);
    const IpaSegments gseg{d_starts, P}, lseg{d_starts + (P + 1), P},
        xseg{d_starts + 2 * (P + 1), P}, dseg{d_starts + 3 * (P + 1), P};
    // exponents of every proof in one arena
    DevBuf<ScE> e(e_total, s), bred(nsum, s), d_xsq(sum_k + 1, s), d_tail(2 * sum_k + 1, s);
    DevBuf<ScE> partial(2 * starts[4 * (P + 1) - 1] + 2, s);
    copy_h2d(bred.p, b_vectors, 32 * nsum, s);
    copy_h2d(d_xsq.p, xsq_m.data(), 32 * sum_k, s);
    copy_h2d(d_tail.p, tail.data(), 64 * sum_k, s);
    launch(IpaReduceBody{bred.p}, nsum, s);
    launch(IpaVerifyExponentsSegBody{xseg, d_rows, d_xsq.p, d_tail.p, e.p}, starts[3 * (P + 1) - 1],
           s);
    launch(IpaDot1SegBody{dseg, d_rows, e.p, bred.p, K, partial.p}, starts[4 * (P + 1) - 1], s);
    launch(IpaDot1FinalSegBody{dseg, d_rows, partial.p, e.p}, P, s);
    // generators of every proof in one arena, then the [Q_p, A_p] pairs of the commit check
    DevBuf<C::Gen> gens(e_total + 2 * (u64)P, s);
    C::Gen* pairs = gens.p + e_total;
    DevBuf<unsigned char> d_lr(64 * sum_k + 64, s), araw((size_t)P * C::kAbiGenBytes, s),
        d_sc2(64 * (size_t)P, s);
    DevBuf<u32> bad(P, s);
    dev_zero(bad.p, sizeof(u32) * P, s);
    copy_h2d(d_lr.p, lr.data(), 64 * sum_k, s);
    copy_h2d(araw.p, a_commits, (size_t)P * C::kAbiGenBytes, s);
    copy_h2d(d_sc2.p, sc2.data(), 64 * (size_t)P, s);
    launch(IpaVerifyGensBody{gseg, d_rows, (const C::Gen*)ctx.builtin, gens.p, pairs}, starts[P], s);
    launch(IpaVerifyDecodeBody{lseg, d_rows, d_lr.p, gens.p, bad.p}, starts[2 * (P + 1) - 1], s);
    launch(IpaVerifyCommitsBody{araw.p, pairs}, P, s);
    // one engine pass: column 2p = <exponents, [Q, G, L, R]>, column 2p + 1 = product Q + a_commit
    std::vector<ColumnDesc> colv;
    for (uint32_t p = 0; p < P; ++p) {
      colv.push_back(column(e.p + rows[p].e_off, 1 + rows[p].np + 2 * rows[p].k, rows[p].g_off));
      colv.push_back(column(d_sc2.p + 64 * (size_t)p, 2, e_total + 2 * (u64)p));
    }
    DevBuf<C::Point> pts(2 * P, s);
    DevBuf<unsigned char> enc(64 * (size_t)P, s);
    Ops::run_columns(ctx, gens.p, colv, pts.p);
    launch_store_commit<C>(s, pts.p, enc.p, 2 * (u64)P, ctx.opt.lane_tail != 0);
    std::vector<uint8_t> enc_host(64 * (size_t)P);
    std::vector<u32> bad_host(P);
    copy_d2h(enc_host.data(), enc.p, 64 * (size_t)P, s);
    copy_d2h(bad_host.data(), bad.p, sizeof(u32) * P, s);
    stream_sync(s);
    dev_free((void*)d_rows, s);
    dev_free((void*)d_starts, s);
    uint32_t accepted = 0;
    for (uint32_t p = 0; p < P; ++p) {
      results[p] = bad_host[p] == 0 && std::memcmp(&enc_host[64 * (size_t)p],
                                                   &enc_host[64 * (size_t)p + 32], 32) == 0;
      accepted += (uint32_t)results[p];
    }
    return accepted;
  }
};

}  // namespace b200
