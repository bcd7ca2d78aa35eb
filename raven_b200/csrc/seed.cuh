// raven_b200 — seed lookup and hit expansion shared by the single-GPU map (map.cu)
// and the multi-GPU owner path (dist.cu); the warp's slot search is also the bucket
// fill of the index table (index.cu).
//
// A seed hit is a ram "Match": group = (rhs_id << 1 | same_strand) << 32 | diagonal,
// the diagonal offset by 3 << 30 on the same strand, and positions = lhs_pos << 32 |
// rhs_pos. The chain kernels (map.cu) decode exactly this. An origin is
// read_id << 32 | position << 1 | strand, for queries and postings alike.
#pragma once
#include <cstdint>

#include "common.cuh"

namespace rvn {
namespace {

struct IndexView {
  ValView val;  // sorted values, u32 or u64
  const uint64_t* org;
  const uint32_t* bucket;
  uint64_t n;
  int shift;
  uint32_t occurrence;
  uint64_t limit;  // values beyond it are not indexed (tiered build)
};

// first record with value v and the run length capped at occurrence+1
__device__ __forceinline__ void Lookup(const IndexView& ix, uint64_t v,
                                       uint32_t* first, uint32_t* count) {
  if (v > ix.limit) {
    *first = 0;
    *count = 0;
    return;
  }
  const uint64_t b = v >> ix.shift;
  uint32_t lo = ix.bucket[b], hi = ix.bucket[b + 1];
  while (hi - lo > 8) {  // long buckets: bisect down to a short scan
    const uint32_t mid = lo + (hi - lo) / 2;
    if (ix.val[mid] < v) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  // here every record before lo is < v; the run (if any) starts in [lo, hi]
  const uint32_t end = ix.bucket[b + 1];
  while (lo < end && ix.val[lo] < v) ++lo;
  if (lo >= end || ix.val[lo] != v) {
    *first = 0;
    *count = 0;
    return;
  }
  *first = lo;
  if (ix.occurrence != 0xFFFFFFFFu &&
      static_cast<uint64_t>(lo) + ix.occurrence < ix.n &&
      ix.val[static_cast<uint64_t>(lo) + ix.occurrence] == v) {
    *count = ix.occurrence + 1;  // over the threshold, exact length not needed
    return;
  }
  uint32_t n = 1;
  while (static_cast<uint64_t>(lo) + n < ix.n && ix.val[lo + n] == v) ++n;
  *count = n;
}

__device__ __forceinline__ bool KeepPosting(uint32_t lhs_id, uint64_t origin,
                                            bool avoid_equal,
                                            bool avoid_symmetric) {
  const uint32_t rhs_id = static_cast<uint32_t>(origin >> 32);
  if (avoid_equal && lhs_id == rhs_id) return false;
  if (avoid_symmetric && lhs_id > rhs_id) return false;
  return true;
}

// Probe of one query (value v, read lhs_id) under any flags: the first posting of
// v's run and the number of its postings KeepPosting keeps, counted one by one. A
// run longer than the occurrence threshold keeps none and sets *over.
__device__ __forceinline__ void ProbeRun(const IndexView& ix, uint64_t v, uint32_t lhs_id,
                                         bool avoid_equal, bool avoid_symmetric,
                                         uint32_t* first, uint32_t* kept, uint8_t* over) {
  uint32_t f, n;
  Lookup(ix, v, &f, &n);
  const uint8_t o = n > ix.occurrence;
  uint32_t k = 0;
  if (!o) {
    for (uint32_t j = 0; j < n; ++j) {
      k += KeepPosting(lhs_id, ix.org[f + j], avoid_equal, avoid_symmetric);
    }
  }
  *kept = k;
  *first = f;
  *over = o;
}

// Probe of one query (value v) when the kept postings are a suffix of the run: the
// postings of a key are in read order (the index sort is stable over records in
// (read, position) order), so with avoid_equal && avoid_symmetric (strict_above) the
// kept postings are those with rhs_id > lhs_id, found by a binary search, and with
// both flags off they are the whole run. Gives the first kept posting and their
// number; a run longer than the occurrence threshold keeps none and sets *over.
// q_org[q], the query's origin, is read only when strict_above and the run is kept.
__device__ __forceinline__ void ProbeSuffix(const IndexView& ix, uint64_t v, bool strict_above,
                                            const uint64_t* q_org, uint64_t q, uint32_t* first,
                                            uint32_t* kept, uint8_t* over) {
  uint32_t f, n;
  Lookup(ix, v, &f, &n);
  uint8_t o = 0;
  uint32_t k = 0, fk = f;
  if (n > ix.occurrence) {
    o = 1;
  } else if (n > 0) {
    if (strict_above) {
      const uint32_t lhs_id = static_cast<uint32_t>(q_org[q] >> 32);
      uint32_t lo = f, hi = f + n;  // first posting with rhs_id > lhs_id
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (static_cast<uint32_t>(ix.org[mid] >> 32) <= lhs_id) lo = mid + 1; else hi = mid;
      }
      fk = lo;
    }
    k = f + n - fk;
  }
  *kept = k;
  *first = fk;
  *over = o;
}

// the seed hit of the query with origin lo and the posting with origin o
__device__ __forceinline__ void EncodeHit(uint64_t lo, uint64_t o, uint64_t* grp,
                                          uint64_t* pos) {
  const uint64_t lhs_pos = static_cast<uint32_t>(lo) >> 1;
  const uint64_t rhs_id = o >> 32;
  const uint64_t strand = (lo & 1) == (o & 1);
  const uint64_t rhs_pos = static_cast<uint32_t>(o) >> 1;
  const uint64_t diagonal =
      !strand ? rhs_pos + lhs_pos : rhs_pos - lhs_pos + (3ULL << 30);
  *grp = (((rhs_id << 1) | strand) << 32) | diagonal;
  *pos = (lhs_pos << 32) + rhs_pos;  // ('+', not '|': one register fewer in ExpandKernel)
}

// The hits of one query (value v, origin lo) by one thread: the first `left` postings
// KeepPosting keeps, walking v's run from posting `first`. Hit h goes to
// store(dst + h, group, positions, lhs_id).
template <typename Store>
__device__ __forceinline__ void ExpandRun(const IndexView& ix, uint64_t v, uint64_t lo,
                                          uint32_t first, uint32_t left, bool avoid_equal,
                                          bool avoid_symmetric, uint64_t dst, Store store) {
  const uint32_t lhs_id = static_cast<uint32_t>(lo >> 32);
  for (uint64_t j = first; left > 0 && j < ix.n && ix.val[j] == v; ++j) {
    const uint64_t o = ix.org[j];
    if (!KeepPosting(lhs_id, o, avoid_equal, avoid_symmetric)) continue;
    uint64_t grp, pos;
    EncodeHit(lo, o, &grp, &pos);
    store(dst, grp, pos, lhs_id);
    ++dst;
    --left;
  }
}

// Exclusive prefix of the 32 lanes' counts; *total = their sum.
__device__ __forceinline__ uint32_t WarpExclusiveSum(uint32_t cnt, uint32_t lane,
                                                     uint32_t* total) {
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if (lane >= static_cast<uint32_t>(d)) incl += o;
  }
  *total = __shfl_sync(0xFFFFFFFFu, incl, 31);
  return incl - cnt;
}

// The lane that owns slot t of the warp, lane q owning slots [rel_q, rel_q + count_q)
// (rel = WarpExclusiveSum of the counts): the largest q with rel_q <= t, found by a
// shuffle search over the 32 prefixes.
__device__ __forceinline__ uint32_t WarpSlotLane(uint32_t rel, uint32_t t) {
  uint32_t q = 0;
#pragma unroll
  for (uint32_t step = 16; step > 0; step >>= 1) {
    const uint32_t r = __shfl_sync(0xFFFFFFFFu, rel, q + step);
    if (r <= t) q += step;
  }
  return q;
}

// The hits of a warp's 32 queries by the whole warp, with coalesced stores: lane q's
// query (origin lo) has `cnt` hits, the postings org[first ..) of the run, and its hits
// go to dst, dst + 1, ... Each step takes the warp's next 32 hits and finds each one's
// query by WarpSlotLane. Hit h of a query goes to store(dst + h, group, positions,
// lhs_id). A lane without a query gives cnt = 0.
template <typename Store>
__device__ __forceinline__ void ExpandWarp(const uint64_t* __restrict__ org, uint32_t lane,
                                           uint32_t cnt, uint32_t first, uint64_t lo,
                                           uint64_t dst, Store store) {
  uint32_t total;
  const uint32_t rel = WarpExclusiveSum(cnt, lane, &total);
  for (uint32_t t0 = 0; t0 < total; t0 += 32) {
    const uint32_t t = t0 + lane;
    const uint32_t q = WarpSlotLane(rel, t);
    const uint32_t h = t - __shfl_sync(0xFFFFFFFFu, rel, q);
    const uint32_t qfirst = __shfl_sync(0xFFFFFFFFu, first, q);
    const uint64_t qlo = __shfl_sync(0xFFFFFFFFu, lo, q);
    const uint64_t qdst = __shfl_sync(0xFFFFFFFFu, dst, q);
    if (t < total) {
      uint64_t grp, pos;
      EncodeHit(qlo, org[qfirst + h], &grp, &pos);
      store(qdst + h, grp, pos, static_cast<uint32_t>(qlo >> 32));
    }
  }
}

}  // namespace
}  // namespace rvn
