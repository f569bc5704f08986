// Batch-affine bucket accumulation for the short Weierstrass curves (bls12-381 G1, bn254 G1,
// Grumpkin): the first levels of the bucket sums are computed as AFFINE + AFFINE -> AFFINE additions
// whose field inversions are shared by Montgomery's trick over the whole level, ~6 field
// multiplications per addition against 11 multiplications + 2 multiplications by 3b of the complete
// projective mixed addition (Renes-Costello-Batina Alg. 8) the chunk walk uses.
//
// Replaces, for these curves, the bulk of the work of mtxbk::bucket_accumulate
// (sxt/multiexp/bucket_method/accumulation_kernel.h:38-75) / cg1o::add (sxt/curve_g1/operation/
// add.cc:37-72) — 32 projective additions per term there.
//
// Layout: the counting sort pads every bucket to a multiple of 2^L slots (pad slots = identity), so
// that level l+1 is simply out[j] = in[2j] + in[2j+1] with no compaction between levels: a pair never
// straddles two buckets, the key of slot j at level l is the key of slot j << l at level 0. After L
// levels (L from the mean bucket load: pads stay below a quarter of the slots) the surviving
// ~2^-L fraction goes through the ordinary chunk walk + cascade.
//
// Every kernel is an index-parallel body (no shared memory): thread t owns B consecutive pairs,
//   pass 1: den_i = x2 - x1 (2 y1 for a doubling, 1 when no addition is needed); prefix products are
//           written to HBM, the thread's total to A[t];
//   A is inverted in place by a 64-ary product tree (BatchUp / BatchTop / BatchDown bodies);
//   pass 2: walks the pairs backwards, peeling one inverse per pair off A[t]^-1, and writes the sum.
#pragma once
#include "curve.cuh"
#include "runtime.cuh"

namespace b200 {

constexpr u32 kPadIndex = 0x7fffffffu;  // generator index of a pad entry (identity)
constexpr u32 kBatchGroup = 8;          // arity of the inversion tree: short serial chains per thread, the
                                        // levels above the first are latency-bound either way
constexpr u32 kBatchTop = 4;            // at most this many values reach the top of the tree (their
                                        // data-dependent inversions diverge within a warp: 64 lanes take
                                        // several times as long as a handful)

// ---- in-place batch inversion of n non-zero field elements ----------------------------------------
template <class F> struct BatchUpBody {
  static constexpr int kBlock = 128;
  const typename F::E* vals;
  typename F::E* pre;
  typename F::E* prod;
  u64 n;
  B200_HD void operator()(u64 j) const {
    const u64 b = j * kBatchGroup, e = b + kBatchGroup < n ? b + kBatchGroup : n;
    typename F::E acc = F::one();
    for (u64 i = b; i < e; ++i) {
      pre[i] = acc;
      F::mul(acc, acc, vals[i]);
    }
    prod[j] = acc;
  }
};
template <class F> struct BatchDownBody {
  static constexpr int kBlock = 128;
  typename F::E* vals;
  const typename F::E* pre;
  const typename F::E* prod;  // inverses of the group products
  u64 n;
  B200_HD void operator()(u64 j) const {
    const u64 b = j * kBatchGroup, e = b + kBatchGroup < n ? b + kBatchGroup : n;
    typename F::E inv = prod[j];
    for (u64 i = e; i-- > b;) {
      typename F::E t, v = vals[i];
      F::mul(t, inv, pre[i]);
      F::mul(inv, inv, v);
      vals[i] = t;
    }
  }
};
// top of the tree: at most kBatchTop values, one inversion per thread (binary extended Euclid, all in
// parallel: the latency of ONE inversion, without a serial prefix / back-substitution pass around it)
template <class F> struct BatchTopBody {
  static constexpr int kBlock = 32;
  typename F::E* vals;
  B200_HD void operator()(u64 i) const {
    typename F::E inv;
    F::invert_eea(inv, vals[i]);  // at most kBatchTop threads: latency of one inversion
    vals[i] = inv;
  }
};
template <class F> inline void batch_invert(stream_t s, typename F::E* vals, u64 n) {
  typedef typename F::E E;
  if (n == 0)
    return;
  if (n <= kBatchTop) {
    launch(BatchTopBody<F>{vals}, n, s);
    return;
  }
  E* pre = (E*)dev_alloc(n * sizeof(E), s);
  const u64 m = (n + kBatchGroup - 1) / kBatchGroup;
  E* prod = (E*)dev_alloc(m * sizeof(E), s);
  launch(BatchUpBody<F>{vals, pre, prod, n}, m, s);
  batch_invert<F>(s, prod, m);
  launch(BatchDownBody<F>{vals, pre, prod, n}, m, s);
  dev_free(prod, s);
  dev_free(pre, s);
}

// ---- one pair level --------------------------------------------------------------------------------
template <class C> struct PairLevel {
  typedef typename C::F F;
  typedef typename F::E fe;
  typedef typename C::Gen Gen;
  // level 0 reads the sorted, padded entry list and gathers generators; later levels read the
  // previous level's points
  const u64* entries;
  const Gen* gens;
  const Gen* in;
  const u32* m_ptr;  // number of padded level-0 slots (device)
  u32 level;         // this level's inputs are slots of 2^level level-0 slots
  u32 B;             // pairs per thread

  B200_HD u64 valid_pairs() const { return (u64)(*m_ptr) >> (level + 1); }
  B200_HD void load(Gen& a, u64 slot) const {
    if (in) {
      a = in[slot];
      return;
    }
    const u64 ent = entries[slot];
    const u32 idx = (u32)ent >> 1;
    if (idx == kPadIndex) {
      a.x = F::zero();
      a.y = F::zero();
      return;
    }
    a = gens[idx];
    if (((u32)ent & 1u) && !C::gen_is_identity(a))
      F::neg(a.y, a.y);
  }
  // 0 = chord addition, 1 = result is a, 2 = result is b, 3 = tangent (doubling), 4 = identity
  B200_HD int classify(fe& den, const Gen& a, const Gen& b) const {
    den = F::one();
    if (C::gen_is_identity(b))
      return 1;
    if (C::gen_is_identity(a))
      return 2;
    if (F::equal(a.x, b.x)) {
      fe s;
      F::add(s, a.y, b.y);
      if (F::is_zero(s))
        return 4;
      den = s;  // = 2 y
      return 3;
    }
    F::sub(den, b.x, a.x);
    return 0;
  }
};

// Pass 1 of level 0 (later levels get theirs fused into the previous level's pass 2): only the x
// coordinates are gathered — half the bytes of this HBM-bound pass — and y is fetched for the rare
// pairs that need it (equal x, or x = 0 where (0,0) encodes the identity).
template <class C> struct PairPass1Body {
  static constexpr int kBlock = 128;
  typedef typename C::F F;
  typedef typename F::E fe;
  PairLevel<C> lv;
  fe* pre;     // one per pair
  fe* totals;  // one per thread
  u64 t0;      // first thread of this launch (the level is launched in two halves on two streams)
  B200_HD void operator()(u64 t) const {
    t += t0;
    const u64 np = lv.valid_pairs();
    const u64 b = t * lv.B, e = b + lv.B < np ? b + lv.B : np;
    fe acc = F::one();
    for (u64 p = b; p < e; ++p) {
      const u64 ea = lv.entries[2 * p], eb = lv.entries[2 * p + 1];
      const u32 ia = (u32)ea >> 1, ib = (u32)eb >> 1;
      fe den = F::one();
      if (ia != kPadIndex && ib != kPadIndex) {
        const fe xa = lv.gens[ia].x, xb = lv.gens[ib].x;
        if (F::equal(xa, xb) || F::is_zero(xa) || F::is_zero(xb)) {
          typename C::Gen ga, gb;  // rare: the full classification
          lv.load(ga, 2 * p);
          lv.load(gb, 2 * p + 1);
          lv.classify(den, ga, gb);
        } else {
          F::sub(den, xb, xa);
        }
      }
      pre[p] = acc;
      F::mul(acc, acc, den);
    }
    totals[t] = acc;
  }
};

// Pass 2 of level l, fused with pass 1 of level l+1: the sums a thread writes are exactly the inputs
// of its own pairs one level up (B halves per level), so their denominators and prefix products are
// formed on the spot — one heavy kernel per level and no second read of the points. The prefix of
// level l+1 is therefore built in the order level l is walked, and each level is walked against the
// order its own prefix was built in: `descending` alternates from level to level.
template <class C> struct PairPass2Body {
  static constexpr int kBlock = 128;
  static constexpr int kMinBlocks = C::F::N > 8 ? 2 : 3;  // 168-register cap for the 8-limb fields
  typedef typename C::F F;
  typedef typename F::E fe;
  typedef typename C::Gen Gen;
  PairLevel<C> lv;
  const fe* pre;
  const fe* totals;  // inverted
  Gen* out;
  fe* pre_next;     // null on the last level
  fe* totals_next;
  u32 descending;
  u64 t0;
  B200_HD void add_pair(Gen& r, const Gen& x, const Gen& y, int kind, const fe& inv) const {
    if (kind == 1) {
      r = x;
    } else if (kind == 2) {
      r = y;
    } else if (kind == 4) {
      r.x = F::zero();
      r.y = F::zero();
    } else {
      fe num, lam, l2, dx;
      if (kind == 3) {  // 3 x^2 / (2 y)
        fe xx;
        F::sqr(xx, x.x);
        F::add(num, xx, xx);
        F::add(num, num, xx);
      } else {
        F::sub(num, y.y, x.y);
      }
      F::mul(lam, num, inv);
      F::sqr(l2, lam);
      F::sub(l2, l2, x.x);
      F::sub(r.x, l2, y.x);
      F::sub(dx, x.x, r.x);
      F::mul(l2, lam, dx);
      F::sub(r.y, l2, x.y);
    }
  }
  B200_HD void operator()(u64 t) const {
    t += t0;
    const u64 np = lv.valid_pairs();
    const u64 b = t * lv.B, e = b + lv.B < np ? b + lv.B : np;
    if (b >= e) {
      if (pre_next)
        totals_next[t] = F::one();  // the inversion tree multiplies every thread's total
      return;
    }
    const u64 cnt = e - b;
    fe inv_acc = totals[t], acc_next = F::one();
    Gen held;
    // operands of the next pair are loaded before the current addition is computed
    u64 p = descending ? e - 1 : b;
    Gen xn, yn;
    fe pn;
    lv.load(xn, 2 * p);
    lv.load(yn, 2 * p + 1);
    pn = pre[p];
    for (u64 k = 0; k < cnt; ++k) {
      const Gen x = xn, y = yn;
      const fe pr = pn;
      const u64 cur = p;
      if (k + 1 < cnt) {
        p = descending ? p - 1 : p + 1;
        lv.load(xn, 2 * p);
        lv.load(yn, 2 * p + 1);
        pn = pre[p];
      }
      fe den, inv;
      Gen r;
      const int kind = lv.classify(den, x, y);
      F::mul(inv, inv_acc, pr);
      F::mul(inv_acc, inv_acc, den);
      add_pair(r, x, y, kind, inv);
      out[cur] = r;
      if (pre_next) {
        // the element reached first is the odd one when walking down, the even one when walking up
        const bool second = descending ? (cur & 1u) == 0 : (cur & 1u) != 0;
        if (!second) {
          held = r;
        } else {
          fe den2;
          if (descending)
            lv.classify(den2, r, held);
          else
            lv.classify(den2, held, r);
          pre_next[cur >> 1] = acc_next;
          F::mul(acc_next, acc_next, den2);
        }
      }
    }
    if (pre_next)
      totals_next[t] = acc_next;
  }
};

// counts -> counts rounded up to a multiple of 2^L (the scan of these gives the padded offsets)
struct PadCountsBody {
  static constexpr int kBlock = 256;
  u32* counts;
  u32 mask;  // 2^L - 1
  B200_HD void operator()(u64 k) const { counts[k] = (counts[k] + mask) & ~mask; }
};
// pad entries behind the real entries of every bucket: [cursor[k], starts[k+1])
struct FillPadsBody {
  static constexpr int kBlock = 128;
  const u32* starts;  // padded exclusive offsets, nkeys + 1
  const u32* cursor;  // end of the real entries of every bucket (scatter cursor)
  u64* entries;
  B200_HD void operator()(u64 k) const {
    const u64 pad = ((u64)k << 32) | ((u64)kPadIndex << 1);
    for (u32 i = cursor[k]; i < starts[k + 1]; ++i)
      entries[i] = pad;
  }
};
// entry list of the level the chunk walk starts from: slot j holds the point of 2^L level-0 slots,
// keyed like them
struct FinalEntriesBody {
  static constexpr int kBlock = 256;
  const u64* entries0;
  const u32* m_ptr;
  u32 L;
  u64* entries;
  u32* m_out;
  B200_HD void operator()(u64 j) const {
    const u64 m = (u64)(*m_ptr) >> L;
    if (j == 0)
      *m_out = (u32)m;
    if (j < m)
      entries[j] = (entries0[j << L] & 0xffffffff00000000ull) | (j << 1);
  }
};

}  // namespace b200
