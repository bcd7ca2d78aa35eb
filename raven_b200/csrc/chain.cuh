// raven_b200 — ram's per-band chain rules (ram::MinimizerEngine::Chain, SURVEY.md
// App. A.2): the one copy, called by the chain kernels of map.cu. A hit is a ram
// "Match" (seed.cuh): group = (rhs_id << 1 | same_strand) << 32 | diagonal, positions =
// lhs_pos << 32 | rhs_pos. It is compiled for the host as well (tests/test_chain_host.py
// runs ChainPairSerial against ram's Chain in the oracle).
#pragma once

#include <cstdint>

#include "../../include/raven_b200.h"

#ifndef RVN_HD
#if defined(__CUDACC__)
#define RVN_HD __host__ __device__ __forceinline__
#else
#define RVN_HD inline
#endif
#endif

namespace rvn {

struct ChainParams {
  uint32_t k, bandwidth, chain, matches, gap;
};

// ram's patience recurrence over the len hits of a band in position order: pos(t) is
// hit t's positions, lis.tail(n) the hit ending the best chain of n hits so far,
// lis.pred(t) hit t's predecessor. Returns the length of the longest chain and leaves
// that chain, as hit indices, in lis.chain(0 .. longest) - or returns 0 when it is
// shorter than min_chain.
template <typename Pos, typename Lis>
RVN_HD uint32_t BandLis(uint32_t len, bool strand, uint32_t min_chain, const Pos& pos,
                        const Lis& lis) {
  if (len < min_chain) return 0;
  // ram's "strand ? tr < cr : tr > cr" as (tr ^ flip) < (cr ^ flip): ~ reverses the order
  const uint32_t flip = strand ? 0u : ~0u;
  uint32_t longest = 0;
  for (uint32_t t = 0; t < len; ++t) {
    const uint64_t cur = pos(t);
    const uint32_t cl = static_cast<uint32_t>(cur >> 32);
    const uint32_t cr = static_cast<uint32_t>(cur) ^ flip;
    uint32_t lo = 1, hi = longest;
    while (lo <= hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      const uint64_t tail = pos(lis.tail(mid));
      const uint32_t tl = static_cast<uint32_t>(tail >> 32);
      const uint32_t tr = static_cast<uint32_t>(tail);
      if (tl < cl && (tr ^ flip) < cr) {
        lo = mid + 1;
      } else {
        hi = mid - 1;
      }
    }
    lis.set_pred(t, lo > 1 ? lis.tail(lo - 1) : 0u);
    lis.set_tail(lo, t);
    longest = longest < lo ? lo : longest;
  }
  if (longest < min_chain) return 0;
  uint32_t j = lis.tail(longest);
  for (uint32_t i = 0; i < longest; ++i) {
    const uint32_t pj = lis.pred(j);
    lis.set_chain(longest - 1 - i, j);
    j = pj;
  }
  return longest;
}

// The overlaps of one unrolled chain of `longest` hits, at(m) being the positions of
// its m-th hit: the chain is cut where the lhs position jumps by more than cp.gap, and
// every piece of at least cp.chain hits whose covered bases on both reads reach
// cp.matches calls emit(first, last, score) with the positions of its first and last
// hit and the smaller of the two covered-base counts.
template <typename At, typename Emit>
RVN_HD void ForEachChainOverlap(uint32_t longest, bool strand, const ChainParams& cp,
                                const At& at, Emit&& emit) {
  for (uint32_t kk = 1, l = 0; kk <= longest; ++kk) {
    const uint32_t prev = static_cast<uint32_t>(at(kk - 1) >> 32);
    const uint32_t cur = kk < longest ? static_cast<uint32_t>(at(kk) >> 32) : 0xFFFFFFFFu;
    if (cur - prev <= cp.gap) continue;
    if (kk - l >= cp.chain) {
      // covered bases m of one read: the union of the k-mers [b, e) begun so far
      uint32_t lm = 0, lb = 0, le = 0, rm = 0, rb = 0, re = 0;
      auto cover = [&](uint32_t p, uint32_t& m, uint32_t& b, uint32_t& e) {
        if (p > e) {
          m += e - b;
          b = p;
        }
        e = p + cp.k;
      };
      for (uint32_t m = l; m < kk; ++m) {
        const uint64_t pp = at(m);
        const uint32_t rp = static_cast<uint32_t>(pp);
        cover(static_cast<uint32_t>(pp >> 32), lm, lb, le);
        cover(strand ? rp : (1U << 31) - (rp + cp.k - 1), rm, rb, re);
      }
      lm += le - lb;
      rm += re - rb;
      const uint32_t score = lm < rm ? lm : rm;
      if (score >= cp.matches) emit(at(l), at(kk - 1), score);
    }
    l = kk;
  }
}

// the record of a chain piece from its first and last hit's positions
RVN_HD rvn_overlap MakeOverlap(uint32_t lhs_id, uint32_t rhs_id, bool strand, uint32_t k,
                               uint64_t first, uint64_t last, uint32_t score) {
  rvn_overlap o;
  o.lhs_id = lhs_id;
  o.lhs_begin = static_cast<uint32_t>(first >> 32);
  o.lhs_end = k + static_cast<uint32_t>(last >> 32);
  o.rhs_id = rhs_id;
  o.rhs_begin = strand ? static_cast<uint32_t>(first) : static_cast<uint32_t>(last);
  o.rhs_end = k + (strand ? static_cast<uint32_t>(last) : static_cast<uint32_t>(first));
  o.score = score;
  o.strand = strand;
  return o;
}

// one pair's hits, element i at P[i * T] and D[i * T] (columns interleaved by thread)
struct Column {
  uint64_t* P;  // positions
  uint32_t* D;  // diagonals; per band re-used as (minimal, predecessor) u16 pairs
  uint32_t T;   // stride
  RVN_HD uint64_t& p(uint32_t i) const { return P[i * T]; }
  RVN_HD uint32_t& d(uint32_t i) const { return D[i * T]; }
};

// BandLis storage of a band from column element jb on, in its diagonals (dead once the
// band is in position order): tail(n) then chain(n - 1) in the low, pred in the high half
struct ColumnLis {
  const Column& c;
  uint32_t jb;
  RVN_HD uint32_t chain(uint32_t x) const { return c.d(jb + x) & 0xFFFFu; }
  RVN_HD void set_chain(uint32_t x, uint32_t v) const {
    c.d(jb + x) = (c.d(jb + x) & 0xFFFF0000u) | v;
  }
  RVN_HD uint32_t tail(uint32_t n) const { return chain(n - 1); }
  RVN_HD void set_tail(uint32_t n, uint32_t v) const { set_chain(n - 1, v); }
  RVN_HD uint32_t pred(uint32_t x) const { return c.d(jb + x) >> 16; }
  RVN_HD void set_pred(uint32_t x, uint32_t v) const {
    c.d(jb + x) = (c.d(jb + x) & 0xFFFFu) | (v << 16);
  }
};

// Shell sort of elements [0, n) by operator<, get(i) reading element i and set(i, v)
// writing it (Ciura's gaps, then a plain insertion pass). Not stable: the callers' keys
// tie only on bitwise-equal hits. A pair's hits arrive in no order, and the gapped passes
// move each of them a few times where an insertion sort moves about n / 4 per element.
template <typename Get, typename Set>
RVN_HD void ShellSort(uint32_t n, const Get& get, const Set& set) {
  auto pass = [&](uint32_t gap) {
    for (uint32_t a = gap; a < n; ++a) {
      const auto v = get(a);
      uint32_t b = a;
      for (; b >= gap; b -= gap) {
        const auto u = get(b - gap);
        if (!(v < u)) break;
        set(b, u);
      }
      if (b != a) set(b, v);
    }
  };
  if (n > 1750) pass(1750);
  if (n > 701) pass(701);
  if (n > 301) pass(301);
  if (n > 132) pass(132);
  if (n > 57) pass(57);
  if (n > 23) pass(23);
  if (n > 10) pass(10);
  if (n > 4) pass(4);
  pass(1);
}

struct DiagPos {
  uint32_t d;
  uint64_t p;
  RVN_HD bool operator<(const DiagPos& o) const { return d < o.d || (d == o.d && p < o.p); }
};

// ram's Chain of the m hits of one (rhs_id, strand) pair `gid` by one thread: (diagonal,
// positions) order, ram's window loop over the diagonals, and per band the position
// order, BandLis and ForEachChainOverlap. emit(overlap) gets the overlaps in ram's order.
template <typename Emit>
RVN_HD void ChainPairSerial(const Column& c, uint32_t m, uint32_t gid, uint32_t lhs_id,
                            const ChainParams& cp, Emit&& emit) {
  // A pair whose diagonals all lie within the bandwidth is one window, hence one band of
  // all its hits, which the band step puts in position order anyway: the (diagonal,
  // positions) sort is only needed when the pair spans more than the bandwidth.
  uint32_t dmin = 0xFFFFFFFFu, dmax = 0;
  for (uint32_t i = 0; i < m; ++i) {
    const uint32_t d = c.d(i);
    dmin = d < dmin ? d : dmin;
    dmax = d > dmax ? d : dmax;
  }
  const bool one_band = m == 0 || dmax - dmin <= cp.bandwidth;
  if (!one_band) {
    ShellSort(m, [&](uint32_t i) { return DiagPos{c.d(i), c.p(i)}; },
                  [&](uint32_t i, DiagPos v) {
                    c.d(i) = v.d;
                    c.p(i) = v.p;
                  });
  }
  const bool strand = gid & 1;
  const uint32_t rhs_id = gid >> 1;
  // one band [jb, ie): position order, then the chain rules
  auto band = [&](uint32_t jb, uint32_t ie) {
    const uint32_t len = ie - jb;
    ShellSort(len, [&](uint32_t i) { return c.p(jb + i); },
                  [&](uint32_t i, uint64_t v) { c.p(jb + i) = v; });
    const ColumnLis lis{c, jb};
    const uint32_t longest =
        BandLis(len, strand, cp.chain, [&](uint32_t t) { return c.p(jb + t); }, lis);
    ForEachChainOverlap(longest, strand, cp, [&](uint32_t x) { return c.p(jb + lis.chain(x)); },
                        [&](uint64_t first, uint64_t last, uint32_t score) {
                          emit(MakeOverlap(lhs_id, rhs_id, strand, cp.k, first, last, score));
                        });
  };
  if (one_band) {  // (the window loop below would give the band [0, m) for m >= 4)
    if (m >= 4) band(0, m);
    return;
  }
  // the reference's window loop; index m plays the stop dummy
  bool open = false;
  uint32_t ob = 0, oe = 0;
  for (uint32_t i = 1, j = 0; i <= m; ++i) {
    if (i == m || c.d(i) - c.d(j) > cp.bandwidth) {
      if (i - j >= 4) {
        if (open && oe > j) {
          oe = i;
        } else {
          if (open) band(ob, oe);
          ob = j;
          oe = i;
          open = true;
        }
      }
      ++j;
      while (j < i && (i == m || c.d(i) - c.d(j) > cp.bandwidth)) ++j;
    }
  }
  if (open) band(ob, oe);
}

}  // namespace rvn
