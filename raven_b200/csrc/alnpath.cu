// raven_b200 — batched read-to-target alignment paths and window breaking points
// on sm_90a (SURVEY §8 f-1 / K10).
//
// Replaces, inside racon::Polisher::Polish (RavenLib/src/polish.cc:43-51), the
// per-read edlibAlign(query, target, NW, EDLIB_TASK_PATH) and the walk along its
// path that finds, for every 500-base window of the target, the first and the last
// aligned (target, query) position pair. The polished sequence depends on WHICH of
// the equally optimal paths is taken, so upstream edlib's two rules are kept
// exactly (they are restated on the host in raven_b200/host/edlib.cc, which the
// tests compare this file with):
//   * obtainAlignment: problems whose traceback data, (2*8+4)*ceil(|q|/64)*|t| +
//     8*|t| bytes, is 1 MiB or more are split at target column |t|/2, at the
//     SMALLEST query row r in [1,|q|-1] with forward[r] + backward[r] == distance
//     (then r = 0, then r = |q|), both halves recursively (Hirschberg);
//   * obtainAlignmentTraceback below that size: from the end cell, up (query symbol
//     alone) if optimal, else left (target symbol alone), else the diagonal.
// The path itself is never stored: a leaf's traceback updates the per-window
// first/last pairs directly (64-bit atomicMin/atomicMax, positions are monotone
// along a path).
//
// Formulation: the recursion is run level by level over ALL pairs of the batch.
// Every level computes the forward and the backward score column of each open
// problem (Myers/Hyyro bit-vector blocks inside the Ukkonen band of the KNOWN
// distance of the problem; the query's match masks are precomputed once per pair
// and funnel-shifted to the sub-problem's row offset) - one WARP per problem for
// wide bands (ColumnsWarpKernel: a wavefront over strips of 32 blocks, state in
// registers), one thread per problem for the small ones (ColumnsKernel: the band's
// vectors in a shared-memory ring) - and then the split rows (SplitRowKernel, one
// warp per problem).
// Leaves (one thread each) store their banded columns and walk back. Every value
// the rules compare is exact inside the band (cells of value <= distance), so the
// band changes nothing. The distances themselves come from the same column
// kernel with a doubling band.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <numeric>

#include "engine.cuh"
#include "myers.cuh"

namespace rvn {

namespace {

constexpr int32_t kFar = 1 << 29;

struct AlnPair {
  uint64_t q_word, t_word;  // first word of the reads in `words`
  uint32_t q_begin, q_len;  // query: bases [q_begin, +q_len) of its read, reverse
  uint32_t t_begin, t_len;  //   complemented as a whole when !strand
  uint32_t strand, pad;
  uint64_t arena;           // packed copies: query, reversed query, target, reversed target
  uint64_t peq;             // match masks of the query, then of the reversed query
  uint64_t bp;              // first breaking-point slot of the pair
};

__host__ __device__ inline uint64_t PackedWords(uint32_t len) { return (len + 31ULL) / 32 + 2; }
// (+1: funnel shift of the last block, +4: the grouped loads of ColumnsKernel read ahead)
__host__ __device__ inline uint32_t PeqWords(uint32_t len) { return (len + 63) / 64 + 5; }

struct ColTask {
  uint64_t peq;      // masks of this direction; symbol stride pb
  uint64_t tarr;     // packed target of this direction
  uint64_t scores;   // m + 1 entries in the score scratch, or ~0
  uint64_t carry;    // cols + 1 entries in the carry scratch (warp kernel)
  uint32_t pb;
  uint32_t q0, m;    // rows: bases [q0, q0 + m) of the (reversed) query
  uint32_t t0, cols; // columns: bases [t0, t0 + cols) of the (reversed) target
  int32_t k;
  uint32_t out;      // dist[out]
  uint32_t mode;     // 1: dist = min over the rows of the last column (prefix estimate)
};

struct PathTask {
  uint32_t pair, q0, m, t0, n;
  int32_t score;
};

struct SplitTask {
  PathTask t;
  uint64_t fw, bw;  // score scratch offsets
};

struct LeafTask {
  PathTask t;
  uint32_t w, pad;  // band slots per column
  uint64_t store;   // first 8-byte word of the leaf's columns
};

// ---- per-pair staging: oriented, reversed copies and the query's match masks ----
__global__ void __launch_bounds__(128)
PackPairsKernel(const uint64_t* __restrict__ words, const AlnPair* __restrict__ pairs,
                uint64_t* __restrict__ arena) {
  const AlnPair p = pairs[blockIdx.x];
  const uint64_t qw = PackedWords(p.q_len), tw = PackedWords(p.t_len);
  const uint64_t* qsrc = words + p.q_word;
  const uint64_t* tsrc = words + p.t_word;
  for (uint64_t w = threadIdx.x; w < 2 * qw + 2 * tw; w += blockDim.x) {
    const int which = w < qw ? 0 : w < 2 * qw ? 1 : w < 2 * qw + tw ? 2 : 3;
    const uint64_t idx = which == 0 ? w : which == 1 ? w - qw : which == 2 ? w - 2 * qw
                                                                          : w - 2 * qw - tw;
    const uint32_t len = which < 2 ? p.q_len : p.t_len;
    uint64_t word = 0;
    for (uint32_t x = 0; x < 32; ++x) {
      const uint64_t pos = idx * 32 + x;
      if (pos >= len) break;
      uint32_t base;
      if (which < 2) {
        const uint64_t f = which == 0 ? pos : len - 1 - pos;  // position in the oriented query
        base = p.strand ? BaseAt(qsrc, p.q_begin + f)
                        : 3u - BaseAt(qsrc, static_cast<uint64_t>(p.q_begin) + len - 1 - f);
      } else {
        const uint64_t f = which == 2 ? pos : len - 1 - pos;
        base = BaseAt(tsrc, p.t_begin + f);
      }
      word |= static_cast<uint64_t>(base) << (x << 1);
    }
    arena[p.arena + w] = word;
  }
}

__global__ void __launch_bounds__(128)
PairMasksKernel(const AlnPair* __restrict__ pairs, const uint64_t* __restrict__ arena,
                uint64_t* __restrict__ peq) {
  const AlnPair p = pairs[blockIdx.x];
  const uint64_t qw = PackedWords(p.q_len);
  const uint32_t pb = PeqWords(p.q_len);
  for (uint32_t x = threadIdx.x; x < 2 * pb; x += blockDim.x) {
    const uint32_t dir = x / pb, blk = x % pb;
    uint64_t w0 = 0, w1 = 0;
    uint32_t rows = 0;
    if (64ULL * blk < p.q_len) {
      rows = min(64u, p.q_len - 64u * blk);
      Bases64(arena + p.arena + dir * qw, 64ULL * blk, qw, &w0, &w1);
    }
    const uint64_t mask = rows == 64 ? ~0ULL : ((1ULL << rows) - 1ULL);
#pragma unroll
    for (uint32_t s = 0; s < 4; ++s) {
      const uint64_t eq = (EqMask32(w0, s) | (EqMask32(w1, s) << 32)) & mask;
      peq[p.peq + (dir * 4ULL + s) * pb + blk] = eq;
    }
  }
}

// match mask of the 64 rows starting at base `pos` of a query whose masks are P
__device__ __forceinline__ uint64_t RowsEq(const uint64_t* __restrict__ P, uint32_t pos,
                                           uint32_t rows) {
  const uint32_t w = pos >> 6, sh = pos & 63;
  uint64_t e = P[w] >> sh;
  if (sh) e |= P[w + 1] << (64 - sh);
  if (rows < 64) e &= (1ULL << rows) - 1ULL;
  return e;
}

__device__ __forceinline__ int BandLo(int j, int k) { return (max(1, j - k) - 1) >> 6; }
__device__ __forceinline__ int BandHi(int j, int k, int m) {
  return (min(m, max(1, j + k)) - 1) >> 6;
}

// D[r][cols], r = 0..m, of rows [q0, q0+m) x columns [t0, t0+cols) inside the band
// |row - column| <= k (block granularity); dist = D[m][cols] if the band reaches
// it and it is <= k, else -1. Entries <= k are exact.
template <bool SMEM>
__global__ void __launch_bounds__(64)
ColumnsKernel(const ColTask* __restrict__ tasks, uint32_t n_tasks, uint32_t ring,
              const uint64_t* __restrict__ arena, const uint64_t* __restrict__ peq,
              uint64_t* __restrict__ scratch, int32_t* __restrict__ scores,
              int32_t* __restrict__ dist) {
  extern __shared__ uint64_t sh_vec[];  // SMEM: [2][ring][64]
  const uint32_t tid = blockIdx.x * 64 + threadIdx.x;
  if (tid >= n_tasks) return;
  const ColTask t = tasks[tid];
  const int m = static_cast<int>(t.m), cols = static_cast<int>(t.cols), k = t.k;
  int32_t* S = t.scores == ~0ULL ? nullptr : scores + t.scores;
  if (m == 0) {
    if (S) S[0] = cols;
    dist[t.out] = cols <= k ? cols : -1;
    return;
  }
  // the band's vertical delta vectors: a ring of `ring` blocks, [slot][thread]
  const uint64_t stride = SMEM ? 64 : static_cast<uint64_t>(gridDim.x) * 64;
  uint64_t* pv = SMEM ? sh_vec + threadIdx.x : scratch + tid;
  uint64_t* mv = pv + static_cast<uint64_t>(ring) * stride;
  const uint64_t* P = peq + t.peq;
  const uint64_t* T = arena + t.tarr;
  const int blocks = (m + 63) >> 6;
  const uint64_t last_high = 1ULL << ((m - 1) & 63);
  const uint32_t sh = t.q0 & 63;  // every block of the task starts at the same bit of a mask word
  auto rows_of = [&](int b) { return min(64, m - (b << 6)); };

  int lo = 0;
  int hi = BandHi(0, k, m);
  for (int b = 0; b <= hi; ++b) {
    pv[(b % ring) * stride] = ~0ULL;
    mv[(b % ring) * stride] = 0;
  }
  int score = min(m, (hi + 1) << 6);  // D[bottom row of block hi][column]
  for (int j = 1; j <= cols; ++j) {
    const int want_hi = BandHi(j, k, m);
    if (hi < want_hi) {  // a block enters the band: vertical deltas all +1
      ++hi;
      pv[(hi % ring) * stride] = ~0ULL;
      mv[(hi % ring) * stride] = 0;
      score += rows_of(hi);
    }
    lo = max(lo, BandLo(j, k));
    const uint32_t sym = BaseAt(T, static_cast<uint64_t>(t.t0) + j - 1);
    // mask words of this column's symbol, four blocks per round of loads
    const uint64_t* Ps = P + static_cast<uint64_t>(sym) * t.pb + ((t.q0 + (lo << 6)) >> 6);
    int h = 1;  // row 0 for lo == 0; an upper bound once the band has left row 0
    uint32_t slot = static_cast<uint32_t>(lo) % ring;
    uint64_t x0 = Ps[0];
    for (int b = lo; b <= hi; b += 4, Ps += 4) {
      const uint64_t x1 = Ps[1], x2 = Ps[2], x3 = Ps[3], x4 = Ps[4];
      const uint64_t xs[5] = {x0, x1, x2, x3, x4};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (b + u <= hi) {
          uint64_t e = xs[u] >> sh;
          if (sh) e |= xs[u + 1] << (64 - sh);
          const int rows = rows_of(b + u);
          if (rows < 64) e &= (1ULL << rows) - 1ULL;
          const uint64_t at = slot * stride;
          uint64_t p = pv[at], q = mv[at];
          h = Step(e, h, b + u == blocks - 1 ? last_high : (1ULL << 63), p, q);
          pv[at] = p;
          mv[at] = q;
          slot = slot + 1 == ring ? 0 : slot + 1;
        }
      }
      x0 = x4;
    }
    score += h;
  }
  if (t.mode == 1) {  // smallest value of the column inside the band
    int best = (lo == 0 && cols <= k) ? cols : kFar;
    int v = score;
    for (int b = hi; b >= lo; --b) {
      const uint64_t p = pv[(b % ring) * stride], q = mv[(b % ring) * stride];
      for (int bit = rows_of(b) - 1; bit >= 0; --bit) {
        best = min(best, v);
        v -= static_cast<int>((p >> bit) & 1) - static_cast<int>((q >> bit) & 1);
      }
    }
    dist[t.out] = best <= k ? best : -1;
    return;
  }
  dist[t.out] = (hi == blocks - 1 && score <= k) ? score : -1;
  if (S) {
    for (int r = 0; r <= m; ++r) S[r] = kFar;
    if (lo == 0 && cols <= k) S[0] = cols;
    int v = score;
    for (int b = hi; b >= lo; --b) {
      const uint64_t p = pv[(b % ring) * stride], q = mv[(b % ring) * stride];
      for (int bit = rows_of(b) - 1; bit >= 0; --bit) {
        S[(b << 6) + bit + 1] = v;
        v -= static_cast<int>((p >> bit) & 1) - static_cast<int>((q >> bit) & 1);
      }
    }
  }
}

// The same columns for a WIDE band, one WARP per problem. The band is cut into
// strips of 32 consecutive blocks; inside a strip lane l owns block 32s + l (its
// vectors, its bottom value and its four match masks stay in registers) and the
// strip is swept as a wavefront: at step tau lane l computes column tau - l and
// hands its horizontal delta and bottom value to lane l + 1 by shuffle. The last
// lane of a strip leaves both, per column, in global scratch for lane 0 of the next
// strip. The serial chain of a 10 kb x 10 kb problem shrinks from ~1e6 dependent
// block steps to ~2.5e4 wavefront steps. Same recurrences as ColumnsKernel, same
// results: block b is in the band for columns [max(1, 64b+1-k), 64(b+1)+k].
__global__ void __launch_bounds__(128)
ColumnsWarpKernel(const ColTask* __restrict__ tasks, uint32_t n_tasks,
                  const uint64_t* __restrict__ arena, const uint64_t* __restrict__ peq,
                  int32_t* __restrict__ carry_scratch, int32_t* __restrict__ scores,
                  int32_t* __restrict__ dist) {
  const uint32_t wid = (blockIdx.x * 128 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= n_tasks) return;
  const ColTask t = tasks[wid];
  const int m = static_cast<int>(t.m), cols = static_cast<int>(t.cols), k = t.k;
  int32_t* S = t.scores == ~0ULL ? nullptr : scores + t.scores;
  if (m == 0) {
    if (lane == 0) {
      if (S) S[0] = cols;
      dist[t.out] = cols <= k ? cols : -1;
    }
    return;
  }
  const uint64_t* P = peq + t.peq;
  const uint64_t* T = arena + t.tarr;
  int32_t* carry = carry_scratch + t.carry;
  const int blocks = (m + 63) >> 6;
  const uint64_t last_high = 1ULL << ((m - 1) & 63);
  const uint32_t sh = t.q0 & 63;
  const int hi0 = BandHi(0, k, m);
  const int hi_fin = BandHi(cols, k, m);
  const int lo_fin = cols > 0 ? BandLo(cols, k) : 0;
  if (S) {
    for (int r = lane; r <= m; r += 32) S[r] = kFar;
  }
  if (lane == 0) dist[t.out] = -1;
  __syncwarp();
  if (S && lane == 0 && cols <= k) S[0] = cols;
  int best = (lane == 0 && cols <= k) ? cols : kFar;  // mode 1

  for (int s = 0; 32 * s <= hi_fin; ++s) {
    const int b = 32 * s + lane;
    const bool valid = b <= hi_fin;
    const int last_lane = min(31, hi_fin - 32 * s);
    const bool more = 32 * (s + 1) <= hi_fin;  // another strip follows
    const int jin = b <= hi0 ? 1 : 64 * b + 1 - k;
    const int jout = min(cols, 64 * (b + 1) + k);
    const int above_out = min(cols, 64 * b + k);  // last column with block b - 1 in the band
    const int rows = valid ? min(64, m - (b << 6)) : 0;
    const uint64_t high = b == blocks - 1 ? last_high : (1ULL << 63);
    uint64_t e0 = 0, e1 = 0, e2 = 0, e3 = 0;
    if (valid) {
      const uint32_t w = (t.q0 + (static_cast<uint32_t>(b) << 6)) >> 6;
      const uint64_t mask = rows < 64 ? (1ULL << rows) - 1ULL : ~0ULL;
      auto load = [&](uint32_t sym) {
        const uint64_t* Ps = P + static_cast<uint64_t>(sym) * t.pb + w;
        uint64_t e = Ps[0] >> sh;
        if (sh) e |= Ps[1] << (64 - sh);
        return e & mask;
      };
      e0 = load(0);
      e1 = load(1);
      e2 = load(2);
      e3 = load(3);
    }
    uint64_t pv = ~0ULL, mv = 0;
    int bottom = b <= hi0 ? min(m, (b + 1) << 6) : 0;
    int out_h = 0, out_b = 0;
    uint64_t tword = 0;
    const int first_jin = 32 * s <= hi0 ? 1 : 64 * (32 * s) + 1 - k;
    const int tau1 = min(cols, 64 * (32 * s + last_lane + 1) + k) + last_lane;
    // lane 0 of a later strip reads what the previous strip left, one step ahead
    int enc_next = 0;
    if (s > 0 && lane == 0 && first_jin <= cols) enc_next = carry[first_jin];
    for (int tau = first_jin; tau <= tau1; ++tau) {
      const int j = tau - lane;
      int in_h = __shfl_up_sync(0xFFFFFFFFu, out_h, 1);
      int in_b = __shfl_up_sync(0xFFFFFFFFu, out_b, 1);
      if (lane == 0 && s > 0) {
        in_h = (enc_next & 3) - 1;
        in_b = enc_next >> 2;
        if (j + 1 <= cols) enc_next = carry[j + 1];
      }
      if (valid && j >= jin && j <= jout) {
        const uint64_t pos = static_cast<uint64_t>(t.t0) + j - 1;
        if (j == jin || (pos & 31) == 0) tword = T[pos >> 5];
        const uint32_t sym = static_cast<uint32_t>(tword >> ((pos & 31) << 1)) & 3u;
        const uint64_t e = sym == 0 ? e0 : sym == 1 ? e1 : sym == 2 ? e2 : e3;
        const int h = (b > 0 && j <= above_out) ? in_h : 1;
        if (j == jin && b > hi0) bottom = in_b - in_h + rows;  // the block enters the band
        const int hout = Step(e, h, high, pv, mv);
        bottom += hout;
        out_h = hout;
        out_b = bottom;
        if (more && lane == last_lane) carry[j] = (bottom << 2) | (hout + 1);
      }
    }
    // the last column: rows of the blocks still in the band
    if (valid && b >= lo_fin) {
      if (b == blocks - 1) dist[t.out] = bottom <= k ? bottom : -1;
      if (S || t.mode == 1) {
        int v = bottom;
        for (int bit = rows - 1; bit >= 0; --bit) {
          if (S) S[(b << 6) + bit + 1] = v;
          best = min(best, v);
          v -= static_cast<int>((pv >> bit) & 1) - static_cast<int>((mv >> bit) & 1);
        }
      }
    }
    __syncwarp();
  }
  if (t.mode == 1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
    if (lane == 0) dist[t.out] = best <= k ? best : -1;
  }
}

// one warp per problem: the row where the path crosses the middle column
__global__ void __launch_bounds__(128)
SplitRowKernel(const SplitTask* __restrict__ tasks, uint32_t n_tasks,
               const int32_t* __restrict__ scores, PathTask* __restrict__ children,
               uint32_t* __restrict__ errors) {
  const uint32_t wid = (blockIdx.x * 128 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= n_tasks) return;
  const SplitTask s = tasks[wid];
  const int32_t* fw = scores + s.fw;
  const int32_t* bw = scores + s.bw;
  const int m = static_cast<int>(s.t.m), best = s.t.score;
  int split = -1;
  for (int r0 = 1; r0 <= m - 1 && split < 0; r0 += 32) {
    const int r = r0 + static_cast<int>(lane);
    const bool hit = r <= m - 1 && fw[r] + bw[m - r] == best;
    const uint32_t any = __ballot_sync(0xFFFFFFFFu, hit);
    if (any) split = r0 + __ffs(any) - 1;
  }
  if (split < 0 && fw[0] + bw[m] == best) split = 0;
  if (split < 0 && fw[m] + bw[0] == best) split = m;
  if (lane != 0) return;
  if (split < 0) {  // (unreachable: some row of the column lies on an optimal path)
    atomicAdd(errors, 1u);
    split = 0;
  }
  const uint32_t left = s.t.n / 2;
  children[2 * wid] = PathTask{s.t.pair, s.t.q0, static_cast<uint32_t>(split), s.t.t0, left,
                               fw[split]};
  children[2 * wid + 1] =
      PathTask{s.t.pair, s.t.q0 + split, static_cast<uint32_t>(m - split), s.t.t0 + left,
               s.t.n - left, bw[m - split]};
}

// A leaf: banded columns stored (vertical deltas and the value at the bottom of
// every block), edlib's traceback, per-window first / last (mis)match positions.
__global__ void __launch_bounds__(64)
LeafKernel(const LeafTask* __restrict__ leaves, uint32_t n_leaves,
           const AlnPair* __restrict__ pairs, const uint64_t* __restrict__ arena,
           const uint64_t* __restrict__ peq, uint64_t* __restrict__ store, uint32_t window,
           unsigned long long* __restrict__ bp_first, unsigned long long* __restrict__ bp_last) {
  const uint32_t tid = blockIdx.x * 64 + threadIdx.x;
  if (tid >= n_leaves) return;
  const LeafTask L = leaves[tid];
  const AlnPair pr = pairs[L.t.pair];
  const int m = static_cast<int>(L.t.m), n = static_cast<int>(L.t.n), k = L.t.score;
  const int W = static_cast<int>(L.w);
  const uint64_t qw = PackedWords(pr.q_len);
  const uint32_t pb = PeqWords(pr.q_len);
  const uint64_t* Q = arena + pr.arena;
  const uint64_t* T = arena + pr.arena + 2 * qw;
  const uint64_t* P = peq + pr.peq;
  uint64_t* PV = store + L.store;
  uint64_t* MV = PV + static_cast<uint64_t>(n) * W;
  int32_t* BT = reinterpret_cast<int32_t*>(MV + static_cast<uint64_t>(n) * W);
  const int blocks = (m + 63) >> 6;
  const uint64_t last_high = 1ULL << ((m - 1) & 63);
  auto rows_of = [&](int b) { return min(64, m - (b << 6)); };

  // forward: column j reads the stored column j - 1
  for (int j = 1; j <= n; ++j) {
    const int lo = BandLo(j, k), hi = BandHi(j, k, m);
    const int plo = BandLo(j - 1, k), phi = BandHi(j - 1, k, m);
    const uint32_t sym = BaseAt(T, static_cast<uint64_t>(L.t.t0) + j - 1);
    const uint64_t* Ps = P + static_cast<uint64_t>(sym) * pb;
    const uint64_t at = static_cast<uint64_t>(j - 1) * W, pat = static_cast<uint64_t>(j - 2) * W;
    int h = 1;
    int below = 0;  // D[bottom of block b - 1][j - 1] (set by the previous iteration)
    for (int b = lo; b <= hi; ++b) {
      uint64_t p, q;
      int bot;
      if (b > phi) {  // the block enters the band
        p = ~0ULL;
        q = 0;
        bot = below + rows_of(b);
      } else if (j == 1) {
        p = ~0ULL;
        q = 0;
        bot = min(m, (b + 1) << 6);
      } else {
        p = PV[pat + (b - plo)];
        q = MV[pat + (b - plo)];
        bot = BT[pat + (b - plo)];
      }
      below = bot;
      h = Step(RowsEq(Ps, L.t.q0 + (b << 6), rows_of(b)), h,
               b == blocks - 1 ? last_high : (1ULL << 63), p, q);
      PV[at + (b - lo)] = p;
      MV[at + (b - lo)] = q;
      BT[at + (b - lo)] = bot + h;
    }
  }

  auto cell = [&](int i, int j) -> int {  // D[i][j]
    if (j == 0) return i;
    if (i == 0) return j;
    const int b = (i - 1) >> 6;
    const int lo = BandLo(j, k), hi = BandHi(j, k, m);
    if (b < lo || b > hi) return kFar;
    const uint64_t at = static_cast<uint64_t>(j - 1) * W + (b - lo);
    const int last_row = min(m, (b + 1) << 6);
    const int below = last_row - i;
    int v = BT[at];
    if (below > 0) {
      const int lo_bit = ((i - 1) & 63) + 1;
      const uint64_t mask = (below >= 64 ? ~0ULL : ((1ULL << below) - 1ULL)) << lo_bit;
      v -= __popcll(PV[at] & mask);
      v += __popcll(MV[at] & mask);
    }
    return v;
  };

  const uint32_t w_first = pr.t_begin / window;
  long long cur_w = -1;
  unsigned long long first = 0, last = 0;
  auto flush = [&]() {
    if (cur_w < 0) return;
    const uint64_t slot = pr.bp + (static_cast<uint64_t>(cur_w) - w_first);
    atomicMin(bp_first + slot, first);
    atomicMax(bp_last + slot, last);
  };
  int i = m, j = n, cur = k;
  while (i > 0 || j > 0) {
    if (i > 0 && cell(i - 1, j) + 1 == cur) {
      --i;
      --cur;
    } else if (j > 0 && cell(i, j - 1) + 1 == cur) {
      --j;
      --cur;
    } else {
      const uint32_t tp = pr.t_begin + L.t.t0 + (j - 1), qp = L.t.q0 + (i - 1);
      const long long w = tp / window;
      if (w != cur_w) {
        flush();
        cur_w = w;
        last = (static_cast<unsigned long long>(tp + 1) << 32) | (qp + 1);
      }
      first = (static_cast<unsigned long long>(tp) << 32) | qp;
      const bool eq = BaseAt(Q, static_cast<uint64_t>(L.t.q0) + i - 1) ==
                      BaseAt(T, static_cast<uint64_t>(L.t.t0) + j - 1);
      --i;
      --j;
      if (!eq) --cur;
    }
  }
  flush();
}

}  // namespace

// Distances and window breaking points of n read-to-target alignments (see
// include/raven_b200.h, rvn_align_breaking_points).
void AlignBreakingPoints(Ctx& c, uint64_t n, const uint32_t* q_read, const uint32_t* q_begin,
                         const uint32_t* q_len, const uint8_t* strand, const uint32_t* t_read,
                         const uint32_t* t_begin, const uint32_t* t_len, uint32_t window,
                         const uint64_t* bp_off, int32_t* distance, uint32_t* bp) {
  if (n == 0) return;
  if (window == 0) throw InvalidArgument("window length 0");
  if (n >= 0x7FFFFFFFULL) throw LimitError("2^31 or more pairs");
  std::vector<AlnPair> h(n);
  uint64_t arena_words = 0, peq_words = 0;
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t a = q_read[i], b = t_read[i];
    if (a >= c.n_reads || b >= c.n_reads) throw InvalidArgument("read index out of bounds");
    if (a < c.res_first || a >= c.res_last || b < c.res_first || b >= c.res_last) {
      throw StateError("the bases of these reads were not uploaded (rvn_reads_upload_range)");
    }
    if (static_cast<uint64_t>(q_begin[i]) + q_len[i] > c.h_len[a] ||
        static_cast<uint64_t>(t_begin[i]) + t_len[i] > c.h_len[b]) {
      throw InvalidArgument("substring beyond the end of its read");
    }
    if (q_len[i] >= (1u << 28) || t_len[i] >= (1u << 28)) throw LimitError("substring of 2^28 bases");
    const uint64_t windows =
        t_len[i] ? (static_cast<uint64_t>(t_begin[i]) + t_len[i] - 1) / window - t_begin[i] / window + 1
                 : 0;
    if (bp_off[i + 1] - bp_off[i] != windows) {
      throw InvalidArgument("bp_off must count the windows every target substring touches");
    }
    h[i] = AlnPair{c.h_woff[a], c.h_woff[b], q_begin[i], q_len[i], t_begin[i], t_len[i],
                   strand[i] ? 1u : 0u, 0u, arena_words, peq_words, bp_off[i]};
    arena_words += 2 * PackedWords(q_len[i]) + 2 * PackedWords(t_len[i]);
    peq_words += 8ULL * PeqWords(q_len[i]);
  }
  const uint64_t n_slots = bp_off[n];
  TimerBegin(c, "align_path");
  DevBuf<AlnPair> d_pairs;
  DevBuf<uint64_t> d_arena, d_peq, d_first, d_last;
  DevBuf<int32_t> d_dist, d_scores, d_carry;
  DevBuf<ColTask> d_cols;
  DevBuf<SplitTask> d_splits;
  DevBuf<PathTask> d_children;
  DevBuf<LeafTask> d_leaves;
  DevBuf<uint32_t> d_err;
  d_pairs.reserve(n);
  d_arena.reserve(arena_words + 4);
  d_peq.reserve(peq_words + 8);
  d_first.reserve(n_slots + 1);
  d_last.reserve(n_slots + 1);
  d_err.reserve(1);
  RVN_CUDA(cudaMemcpyAsync(d_pairs.get(), h.data(), n * sizeof(AlnPair), cudaMemcpyHostToDevice,
                           c.stream));
  RVN_CUDA(cudaMemsetAsync(d_first.get(), 0xFF, (n_slots + 1) * 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_last.get(), 0, (n_slots + 1) * 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_err.get(), 0, 4, c.stream));
  PackPairsKernel<<<static_cast<uint32_t>(n), 128, 0, c.stream>>>(c.d_words.get(), d_pairs.get(),
                                                                d_arena.get());
  RVN_LAUNCH_CHECK();
  PairMasksKernel<<<static_cast<uint32_t>(n), 128, 0, c.stream>>>(d_pairs.get(), d_arena.get(),
                                                                d_peq.get());
  RVN_LAUNCH_CHECK();
  c.launches += 2;

  const bool trace = std::getenv("RVN_ALIGN_TRACE") != nullptr;
  auto t_trace = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!trace) return;
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    const auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[rvn::AlignBreakingPoints] %-28s %8.1f ms\n", what,
                 std::chrono::duration<double, std::milli>(now - t_trace).count());
    t_trace = now;
  };
  auto ring_of = [](uint32_t m, int32_t k) {
    const uint32_t blocks = (m + 63) / 64;
    return std::max<uint32_t>(1, std::min<uint32_t>(blocks, (2u * static_cast<uint32_t>(k) >> 6) + 2));
  };
  constexpr uint32_t kWarpRing = 24;   // bands of this many blocks or more: warp kernel,
  constexpr uint64_t kWarpSteps = 16384;  // and any problem of this many block steps
  constexpr uint32_t kSmemRing = 208;  // 208 KB of the 227 KB a CTA may use
  auto ring_class = [](uint32_t ring) {
    uint32_t c = 3;  // rings up to 8, 16, 32, ... slots
    while ((1u << c) < ring) ++c;
    return c;
  };
  // one launch of the column kernel over `tasks` (sorted by cost so that the lanes
  // of a warp carry similar work); results in h_dist[task.out]
  std::vector<int32_t> h_dist;
  auto run_columns = [&](std::vector<ColTask>& tasks, uint64_t score_entries, uint32_t n_out) {
    const auto t_enter = std::chrono::steady_clock::now();
    std::sort(tasks.begin(), tasks.end(), [&](const ColTask& a, const ColTask& b) {
      return static_cast<uint64_t>(a.cols) * ring_of(a.m, a.k) >
             static_cast<uint64_t>(b.cols) * ring_of(b.m, b.k);
    });
    const uint32_t nt = static_cast<uint32_t>(tasks.size());
    // wide bands: one warp per problem (ColumnsWarpKernel); the others one thread
    // per problem, launched by band size class - the vectors of a class live in
    // shared memory ([2][ring][64] per CTA)
    const auto wide = [&](const ColTask& t) {
      const uint32_t ring = ring_of(t.m, t.k);
      return ring >= kWarpRing || static_cast<uint64_t>(t.cols) * ring >= kWarpSteps;
    };
    const uint32_t nw = static_cast<uint32_t>(
        std::stable_partition(tasks.begin(), tasks.end(), wide) - tasks.begin());
    uint64_t carry_entries = 0;
    for (uint32_t x = 0; x < nw; ++x) {
      tasks[x].carry = carry_entries;
      carry_entries += tasks[x].cols + 1ULL;
    }
    std::stable_sort(tasks.begin() + nw, tasks.end(), [&](const ColTask& a, const ColTask& b) {
      return ring_class(ring_of(a.m, a.k)) > ring_class(ring_of(b.m, b.k));
    });
    d_cols.reserve(nt);
    d_dist.reserve(n_out + 1);
    if (score_entries) d_scores.reserve(score_entries + 1);
    if (carry_entries) d_carry.reserve(carry_entries + 1);
    RVN_CUDA(cudaMemcpyAsync(d_cols.get(), tasks.data(), nt * sizeof(ColTask),
                             cudaMemcpyHostToDevice, c.stream));
    if (nw) {
      ColumnsWarpKernel<<<CeilDiv(nw, 4), 128, 0, c.stream>>>(d_cols.get(), nw, d_arena.get(),
                                                             d_peq.get(), d_carry.get(),
                                                             d_scores.get(), d_dist.get());
      RVN_LAUNCH_CHECK();
      ++c.launches;
    }
    uint32_t ring = 1;
    for (uint32_t x0 = nw; x0 < nt;) {
      const uint32_t cls = ring_class(ring_of(tasks[x0].m, tasks[x0].k));
      uint32_t x1 = x0;
      ring = 1;
      while (x1 < nt && ring_class(ring_of(tasks[x1].m, tasks[x1].k)) == cls) {
        ring = std::max(ring, ring_of(tasks[x1].m, tasks[x1].k));
        ++x1;
      }
      const uint32_t cnt = x1 - x0;
      if (ring <= kSmemRing) {
        const size_t smem = 2ULL * ring * 64 * sizeof(uint64_t);
        RVN_CUDA(cudaFuncSetAttribute(ColumnsKernel<true>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(2ULL * kSmemRing * 64 * sizeof(uint64_t))));
        ColumnsKernel<true><<<CeilDiv(cnt, 64), 64, smem, c.stream>>>(
            d_cols.get() + x0, cnt, ring, d_arena.get(), d_peq.get(), nullptr, d_scores.get(),
            d_dist.get());
      } else {
        const uint64_t threads = static_cast<uint64_t>(CeilDiv(cnt, 64)) * 64;
        uint64_t* scratch = c.m_scratch64.reserve(2ULL * ring * threads + 16);
        ColumnsKernel<false><<<CeilDiv(cnt, 64), 64, 0, c.stream>>>(
            d_cols.get() + x0, cnt, ring, d_arena.get(), d_peq.get(), scratch, d_scores.get(),
            d_dist.get());
      }
      RVN_LAUNCH_CHECK();
      ++c.launches;
      x0 = x1;
    }
    if (trace) {
      const auto t0 = std::chrono::steady_clock::now();
      RVN_CUDA(cudaStreamSynchronize(c.stream));
      uint64_t steps = 0;
      for (const auto& t : tasks) steps += static_cast<uint64_t>(t.cols) * ring_of(t.m, t.k);
      std::fprintf(stderr, "[rvn::AlignBreakingPoints]   columns: %u tasks (%u wide), %.2f G block steps, host %.1f ms, kernels %.1f ms\n",
                   nt, nw, steps * 1e-9,
                   std::chrono::duration<double, std::milli>(t0 - t_enter).count(),
                   std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    }
  };

  lap("stage pairs");

  // ---- 1. distances. edlib doubles the band from k = 64 until the distance fits;
  // the distance is unique, so any schedule of k gives the same value. To skip the
  // rounds that cannot succeed, the first k of a long pair is extrapolated from the
  // error rate of its first kPrefix target columns (a banded, query-end-free run of
  // the same kernel); pairs whose distance exceeds it double from there. ----
  std::vector<int32_t> dist(n, -1);
  {
    constexpr uint32_t kPrefix = 384;
    constexpr int32_t kPrefixBand = 96;
    std::vector<uint32_t> todo;
    std::vector<int64_t> kk(n);
    std::vector<ColTask> probe;
    std::vector<uint32_t> probed;
    for (uint64_t i = 0; i < n; ++i) {
      const int64_t m = q_len[i], t = t_len[i];
      if (m == 0 || t == 0) {
        dist[i] = static_cast<int32_t>(m + t);
        continue;
      }
      kk[i] = std::max<int64_t>(64, std::llabs(m - t));
      todo.push_back(static_cast<uint32_t>(i));
      if (t >= 4 * kPrefix && m >= 4 * kPrefix) {
        probe.push_back(ColTask{h[i].peq, h[i].arena + 2 * PackedWords(q_len[i]), ~0ULL, 0,
                                PeqWords(q_len[i]), 0, q_len[i], 0, kPrefix, kPrefixBand,
                                static_cast<uint32_t>(probed.size()), 1});
        probed.push_back(static_cast<uint32_t>(i));
      }
    }
    if (!probe.empty()) {
      run_columns(probe, 0, static_cast<uint32_t>(probed.size()));
      h_dist.resize(probed.size());
      RVN_CUDA(cudaMemcpyAsync(h_dist.data(), d_dist.get(), probed.size() * 4,
                               cudaMemcpyDeviceToHost, c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));
      for (size_t x = 0; x < probed.size(); ++x) {
        const uint32_t i = probed[x];
        const int64_t longest = std::max(q_len[i], t_len[i]);
        const int64_t guess = h_dist[x] >= 0
                                  ? (longest * h_dist[x] * 5 / 4) / kPrefix + 48
                                  : longest / 4;
        kk[i] = std::max(kk[i], guess);
      }
    }
    lap("distance: prefix estimate");
    std::vector<ColTask> tasks;
    while (!todo.empty()) {
      tasks.clear();
      for (uint32_t x = 0; x < todo.size(); ++x) {
        const uint32_t i = todo[x];
        const int32_t k = static_cast<int32_t>(std::min<int64_t>(kk[i], static_cast<int64_t>(q_len[i]) + t_len[i]));
        tasks.push_back(ColTask{h[i].peq, h[i].arena + 2 * PackedWords(q_len[i]), ~0ULL, 0,
                                PeqWords(q_len[i]), 0, q_len[i], 0, t_len[i], k, x, 0});
      }
      run_columns(tasks, 0, static_cast<uint32_t>(todo.size()));
      h_dist.resize(todo.size());
      RVN_CUDA(cudaMemcpyAsync(h_dist.data(), d_dist.get(), todo.size() * 4, cudaMemcpyDeviceToHost,
                               c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));
      std::vector<uint32_t> next;
      for (uint32_t x = 0; x < todo.size(); ++x) {
        const uint32_t i = todo[x];
        if (h_dist[x] >= 0) {
          dist[i] = h_dist[x];
        } else {
          kk[i] *= 2;
          next.push_back(i);
        }
      }
      todo.swap(next);
    }
  }
  lap("distance: band rounds");

  // ---- 2. Hirschberg levels ----
  std::vector<PathTask> level, children;
  std::vector<LeafTask> leaves;
  for (uint64_t i = 0; i < n; ++i) {
    if (q_len[i] && t_len[i]) {
      level.push_back(PathTask{static_cast<uint32_t>(i), 0, q_len[i], 0, t_len[i], dist[i]});
    }
  }
  std::vector<SplitTask> splits;
  std::vector<ColTask> tasks;
  while (!level.empty()) {
    splits.clear();
    tasks.clear();
    uint64_t entries = 0;
    for (const PathTask& t : level) {
      if (t.m == 0 || t.n == 0) continue;  // only insertions / deletions: no aligned pair
      const uint64_t blocks = (t.m + 63) / 64;
      const uint64_t data = (2 * 8 + 4) * blocks * t.n + 2ULL * 4 * t.n;
      if (data < 1024 * 1024) {
        leaves.push_back(LeafTask{t, ring_of(t.m, t.score), 0, 0});
        continue;
      }
      const AlnPair& p = h[t.pair];
      const uint32_t pb = PeqWords(p.q_len);
      const uint64_t qw = PackedWords(p.q_len), tw = PackedWords(p.t_len);
      const uint32_t left = t.n / 2, right = t.n - left;
      SplitTask s{t, entries, entries + t.m + 1};
      entries += 2ULL * (t.m + 1);
      const uint32_t x = static_cast<uint32_t>(splits.size());
      tasks.push_back(ColTask{p.peq, p.arena + 2 * qw, s.fw, 0, pb, t.q0, t.m, t.t0, left, t.score,
                              2 * x, 0});
      tasks.push_back(ColTask{p.peq + 4ULL * pb, p.arena + 2 * qw + tw, s.bw, 0, pb,
                              p.q_len - t.q0 - t.m, t.m, p.t_len - t.t0 - t.n, right, t.score,
                              2 * x + 1, 0});
      splits.push_back(s);
    }
    level.clear();
    if (splits.empty()) break;
    if (entries >= (1ULL << 62)) throw LimitError("score scratch");
    lap("  level: tasks built");
    const uint32_t ns = static_cast<uint32_t>(splits.size());
    run_columns(tasks, entries, 2 * ns);
    d_splits.reserve(ns);
    d_children.reserve(2ULL * ns);
    RVN_CUDA(cudaMemcpyAsync(d_splits.get(), splits.data(), ns * sizeof(SplitTask),
                             cudaMemcpyHostToDevice, c.stream));
    SplitRowKernel<<<CeilDiv(ns, 4), 128, 0, c.stream>>>(d_splits.get(), ns, d_scores.get(),
                                                        d_children.get(), d_err.get());
    RVN_LAUNCH_CHECK();
    ++c.launches;
    level.resize(2ULL * ns);
    RVN_CUDA(cudaMemcpyAsync(level.data(), d_children.get(), 2ULL * ns * sizeof(PathTask),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    lap("  level: split rows + children");
  }

  lap("hirschberg levels");

  // ---- 3. leaves: stored columns + traceback, in chunks of bounded scratch ----
  std::sort(leaves.begin(), leaves.end(), [](const LeafTask& a, const LeafTask& b) {
    return static_cast<uint64_t>(a.t.n) * a.w > static_cast<uint64_t>(b.t.n) * b.w;
  });
  const uint64_t budget = 1ULL << 29;  // 8-byte words per chunk (4 GiB)
  for (size_t x0 = 0; x0 < leaves.size();) {
    size_t x1 = x0;
    uint64_t used = 0;
    while (x1 < leaves.size()) {
      const uint64_t cells = static_cast<uint64_t>(leaves[x1].t.n) * leaves[x1].w;
      const uint64_t need = 2 * cells + (cells + 1) / 2;
      if (x1 > x0 && used + need > budget) break;
      leaves[x1].store = used;
      used += need;
      ++x1;
    }
    const uint32_t nl = static_cast<uint32_t>(x1 - x0);
    if (trace) {
      std::fprintf(stderr, "[rvn::AlignBreakingPoints]   leaves: chunk of %u leaves, %.3f G words of scratch\n",
                   nl, used * 1e-9);
    }
    uint64_t* store = c.m_scratch64.reserve(used + 16);
    d_leaves.reserve(nl);
    RVN_CUDA(cudaMemcpyAsync(d_leaves.get(), leaves.data() + x0, nl * sizeof(LeafTask),
                             cudaMemcpyHostToDevice, c.stream));
    LeafKernel<<<CeilDiv(nl, 64), 64, 0, c.stream>>>(
        d_leaves.get(), nl, d_pairs.get(), d_arena.get(), d_peq.get(), store, window,
        reinterpret_cast<unsigned long long*>(d_first.get()),
        reinterpret_cast<unsigned long long*>(d_last.get()));
    RVN_LAUNCH_CHECK();
    ++c.launches;
    RVN_CUDA(cudaStreamSynchronize(c.stream));  // (the leaf array is reused by the next chunk)
    x0 = x1;
  }

  lap("leaves");

  // ---- 4. results ----
  std::vector<uint64_t> h_first(n_slots + 1), h_last(n_slots + 1);
  uint32_t h_err = 0;
  RVN_CUDA(cudaMemcpyAsync(h_first.data(), d_first.get(), n_slots * 8, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(h_last.data(), d_last.get(), n_slots * 8, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(&h_err, d_err.get(), 4, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  TimerEnd(c);
  lap("results");
  if (h_err) throw std::runtime_error("alignment path: no split row on an optimal path");
  for (uint64_t i = 0; i < n; ++i) distance[i] = dist[i];
  for (uint64_t s = 0; s < n_slots; ++s) {
    if (h_first[s] == ~0ULL) {
      bp[4 * s] = bp[4 * s + 1] = bp[4 * s + 2] = bp[4 * s + 3] = 0xFFFFFFFFu;
    } else {
      bp[4 * s] = static_cast<uint32_t>(h_first[s] >> 32);
      bp[4 * s + 1] = static_cast<uint32_t>(h_first[s]);
      bp[4 * s + 2] = static_cast<uint32_t>(h_last[s] >> 32);
      bp[4 * s + 3] = static_cast<uint32_t>(h_last[s]);
    }
  }
}

}  // namespace rvn
