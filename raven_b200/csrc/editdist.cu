// raven_b200 — batched global (NW) edit distance on sm_90a.
//
// Replaces the edlibAlign(lhs, rhs, edlibDefaultAlignConfig()) calls of the
// identity filter (RavenLib/src/construct.cc:162-217 ResolveContainedReads and
// :385-424 FindOverlapsAndRepetetiveRegions; score = 1 - ed / max(len)): up to
// 3e7 alignments of 10-15 kb substrings on the HiFi configuration. Only the
// integer distance is needed, so any exact method is bit-identical with edlib.
//
// Myers/Hyyro bit-vector blocks (64 query rows per u64) inside an Ukkonen band
// |row - column| <= k. One THREAD per pair: the band of a column spans at most
// NB blocks whose vertical delta vectors (pv, mv) live in registers as a window
// that slides down one block at a time; the match masks of the window's blocks
// sit in shared memory ([symbol][slot][thread], conflict free), built on the
// fly from the 2-bit packed reads (no inflated strings anywhere); the reverse
// complement of the rhs substring is read in place. A pair whose distance
// exceeds the band of one tier (k = 64, 192, 448, 960) moves to the next; what
// is left (or has no bound at all) runs the unbanded kernel with its vectors in
// global scratch. Integer ALU bound (about 40 instructions per block and
// column), no HBM pressure: 0.25 B per base once.
#include <algorithm>
#include <numeric>

#include "../../include/raven_b200/overlap_clip.hpp"
#include "engine.cuh"
#include "myers.cuh"

namespace rvn {

namespace {

// match mask of query block b (rows 64b .. 64b+63 of the lhs substring)
__device__ __forceinline__ uint64_t BlockEq(const uint64_t* __restrict__ qw, uint64_t q_words,
                                            uint32_t q_begin, uint32_t m, uint32_t b,
                                            uint32_t sym) {
  uint64_t w0, w1;
  Bases64(qw, static_cast<uint64_t>(q_begin) + 64ULL * b, q_words, &w0, &w1);
  uint64_t eq = EqMask32(w0, sym) | (EqMask32(w1, sym) << 32);
  const uint32_t rows = min(64u, m - 64u * b);
  if (rows < 64) eq &= (1ULL << rows) - 1ULL;
  return eq;
}

// target symbol of column j (1-based) of the rhs substring, reverse
// complemented in place when !strand
__device__ __forceinline__ uint32_t TargetSym(const uint64_t* __restrict__ tw, const PairDesc& d,
                                              uint32_t j) {
  if (d.strand) return BaseAt(tw, static_cast<uint64_t>(d.t_begin) + j - 1);
  return 3u - BaseAt(tw, static_cast<uint64_t>(d.t_begin) + d.t_len - j);
}

// Banded distance, window of NB blocks in registers. k <= 32 * (NB - 2).
// out[slot] = distance if it is <= k, else -1 ("beyond this tier").
template <int NB, int THREADS>
__global__ void __launch_bounds__(THREADS)
BandedMyersKernel(const uint64_t* __restrict__ words, const uint64_t* __restrict__ woff_unused,
                  const PairDesc* __restrict__ pairs, const uint32_t* __restrict__ list,
                  uint32_t n_list, int k, const int32_t* __restrict__ limit,
                  int32_t* __restrict__ out, uint64_t total_words) {
  extern __shared__ uint64_t sh_eq[];  // [4][NB][THREADS]
  (void)woff_unused;
  const uint32_t gi = blockIdx.x * THREADS + threadIdx.x;
  if (gi >= n_list) return;
  const PairDesc d = pairs[list[gi]];
  const int m = static_cast<int>(d.q_len), n = static_cast<int>(d.t_len);
  // the caller's bound for this pair (-1: none): never look beyond it
  const int lim = limit[d.slot];
  int kk = k;
  if (lim >= 0 && lim < kk) kk = lim;
  int result = -1;
  if (m == 0 || n == 0) {
    result = (m + n <= kk) ? m + n : -1;
    out[d.slot] = result;
    return;
  }
  if (abs(m - n) > kk) {
    out[d.slot] = -1;
    return;
  }
  const uint64_t* qw = words + d.q_word;
  const uint64_t* tw = words + d.t_word;
  const uint64_t q_words = total_words - d.q_word;  // reads beyond: zero bases, masked rows
  const int blocks = (m + 63) >> 6;
  const uint64_t last_high = 1ULL << ((m - 1) & 63);

  uint64_t pv[NB], mv[NB];
#pragma unroll
  for (int i = 0; i < NB; ++i) {
    pv[i] = ~0ULL;
    mv[i] = 0;
  }
  int wlo = 0;                                   // first block of the window
  int hi = (min(m, max(1, kk)) - 1) >> 6;        // last active block (column 0: rows 1..k)
  int score = min(m, (hi + 1) << 6);             // D[bottom row of block hi][column]
  auto eq_at = [&](uint32_t sym, int slot) -> uint64_t& {
    return sh_eq[(sym * NB + slot) * THREADS + threadIdx.x];
  };
  for (int b = 0; b <= hi; ++b) {
#pragma unroll
    for (uint32_t s = 0; s < 4; ++s) eq_at(s, b % NB) = BlockEq(qw, q_words, d.q_begin, m, b, s);
  }

  for (int j = 1; j <= n; ++j) {
    const int want_hi = (min(m, j + kk) - 1) >> 6;
    if (hi < want_hi) {  // a block enters the band: vertical deltas all +1
      ++hi;
      // (its register slot hi - wlo holds pv = ~0, mv = 0: set at start / when sliding)
      score += min(64, m - (hi << 6));
#pragma unroll
      for (uint32_t s = 0; s < 4; ++s) eq_at(s, hi % NB) = BlockEq(qw, q_words, d.q_begin, m, hi, s);
    }
    const int want_lo = (max(1, j - kk) - 1) >> 6;
    if (want_lo > wlo) {  // the window slides down one block
#pragma unroll
      for (int i = 0; i + 1 < NB; ++i) {
        pv[i] = pv[i + 1];
        mv[i] = mv[i + 1];
      }
      pv[NB - 1] = ~0ULL;
      mv[NB - 1] = 0;
      ++wlo;
    }
    const uint32_t sym = TargetSym(tw, d, j);
    int h = 1;  // row 0 for wlo == 0; an upper bound once the band has left row 0
    const int top = hi - wlo;  // last active register slot
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      if (i <= top) {
        const int b = wlo + i;
        h = Step(eq_at(sym, b % NB), h, b == blocks - 1 ? last_high : (1ULL << 63), pv[i], mv[i]);
      }
    }
    score += h;
  }
  if (hi == blocks - 1 && score <= kk) result = score;
  out[d.slot] = result;
}

// Unbanded distance for what the tiers left: vectors of all query blocks in
// global scratch, [block][thread of the launch] (coalesced across the warp).
__global__ void __launch_bounds__(64)
FullMyersKernel(const uint64_t* __restrict__ words, const PairDesc* __restrict__ pairs,
                const uint32_t* __restrict__ list, uint32_t n_list, uint32_t max_blocks,
                uint64_t* __restrict__ scratch, int32_t* __restrict__ out, uint64_t total_words) {
  const uint32_t gi = blockIdx.x * 64 + threadIdx.x;
  if (gi >= n_list) return;
  const PairDesc d = pairs[list[gi]];
  const int m = static_cast<int>(d.q_len), n = static_cast<int>(d.t_len);
  if (m == 0 || n == 0) {
    out[d.slot] = m + n;
    return;
  }
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * 64;
  uint64_t* pv = scratch + gi;                                // pv[b * stride]
  uint64_t* mv = scratch + static_cast<uint64_t>(max_blocks) * stride + gi;
  const uint64_t* qw = words + d.q_word;
  const uint64_t* tw = words + d.t_word;
  const uint64_t q_words = total_words - d.q_word;
  const int blocks = (m + 63) >> 6;
  const uint64_t last_high = 1ULL << ((m - 1) & 63);
  for (int b = 0; b < blocks; ++b) {
    pv[b * stride] = ~0ULL;
    mv[b * stride] = 0;
  }
  int score = m;
  for (int j = 1; j <= n; ++j) {
    const uint32_t sym = TargetSym(tw, d, j);
    int h = 1;
    for (int b = 0; b < blocks; ++b) {
      uint64_t p = pv[b * stride], q = mv[b * stride];
      h = Step(BlockEq(qw, q_words, d.q_begin, m, b, sym), h,
               b == blocks - 1 ? last_high : (1ULL << 63), p, q);
      pv[b * stride] = p;
      mv[b * stride] = q;
    }
    score += h;
  }
  out[d.slot] = score;
}

template <int NB, int THREADS>
void LaunchTier(Ctx& c, const PairDesc* d_pairs, const uint32_t* d_list, uint32_t n_list, int k,
                const int32_t* d_limit, int32_t* d_out) {
  auto kern = BandedMyersKernel<NB, THREADS>;
  const size_t smem = sizeof(uint64_t) * 4 * NB * THREADS;
  RVN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)));
  kern<<<CeilDiv(n_list, THREADS), THREADS, smem, c.stream>>>(
      c.d_words.get(), c.d_woff.get(), d_pairs, d_list, n_list, k, d_limit, d_out, c.n_words + 2);
  RVN_LAUNCH_CHECK();
  ++c.launches;
}

// tier cost of every listed pair (lhs + rhs bases): the list runs longest first, so
// the lanes of a warp carry similar work
__global__ void PairCostKernel(const PairDesc* __restrict__ pairs, const uint32_t* __restrict__ list,
                               uint32_t n, uint32_t* __restrict__ cost) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PairDesc d = pairs[list[i]];
  cost[i] = d.q_len + d.t_len;
}

// pairs of the list still open after a tier of band k: not found within the band and
// allowed to look further; the longest lhs of them into *max_q_len
__global__ void OpenPairsKernel(const PairDesc* __restrict__ pairs, const uint32_t* __restrict__ list,
                                uint32_t n, int k, const int32_t* __restrict__ limit,
                                const int32_t* __restrict__ out, uint32_t* __restrict__ flag,
                                uint32_t* __restrict__ max_q_len) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PairDesc d = pairs[list[i]];
  const int lim = limit[d.slot];
  const bool open = out[d.slot] < 0 && !(lim >= 0 && lim <= k);
  flag[i] = open ? 1u : 0u;
  if (open) atomicMax(max_q_len, d.q_len);
}

// dst[pos[i]] = src[i] where flag[i] (a stable compaction by an exclusive scan of flag)
template <typename T>
__global__ void CompactKernel(const T* __restrict__ src, const uint32_t* __restrict__ flag,
                              const uint64_t* __restrict__ pos, uint64_t n, T* __restrict__ dst) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) dst[pos[i]] = src[i];
}

}  // namespace

void MyersTiers(Ctx& c, const PairDesc* d_pairs, uint32_t* d_list, uint32_t n,
                const int32_t* d_limit, int32_t* d_out) {
  if (n == 0) return;
  uint32_t* key = c.e_key.reserve(n);
  uint32_t* key2 = c.e_key2.reserve(n);
  uint32_t* list2 = c.e_list2.reserve(n);
  uint32_t* flag = c.e_flag.reserve(n + 1ULL);
  uint64_t* pos = c.e_scan.reserve(n + 2ULL);
  PairCostKernel<<<CeilDiv(n, 256), 256, 0, c.stream>>>(d_pairs, d_list, n, key);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  // (the sort's sources may alias its buffers b)
  const int w = RadixSortPairs(c, key, key2, key, d_list, list2, d_list, n, 0, 32,
                               /*descending=*/true);
  uint32_t* list = w == 0 ? list2 : d_list;
  uint32_t* spare = w == 0 ? d_list : list2;
  static const int kTierK[4] = {64, 192, 448, 960};
  // one phase per tier that runs: the timings tell how far a call's pairs went
  static const char* const kTierPhase[5] = {"myers_k64", "myers_k192", "myers_k448",
                                            "myers_k960", "myers_full"};
  uint32_t m = n, max_q_len = 0;
  for (int tier = 0; tier <= 4 && m > 0; ++tier) {
    if (tier == 4) {
      // unbanded: scratch for the vectors of every query block of every pair in flight
      const uint32_t max_blocks = std::max(1u, (max_q_len + 63) / 64);
      const uint64_t threads = static_cast<uint64_t>(CeilDiv(m, 64)) * 64;
      uint64_t* scratch = c.m_scratch64.reserve(2ULL * max_blocks * threads + 16);
      TimerBegin(c, kTierPhase[4]);
      FullMyersKernel<<<CeilDiv(m, 64), 64, 0, c.stream>>>(c.d_words.get(), d_pairs, list, m,
                                                          max_blocks, scratch, d_out,
                                                          c.n_words + 2);
      RVN_LAUNCH_CHECK();
      ++c.launches;
      TimerEnd(c);
      break;
    }
    TimerBegin(c, kTierPhase[tier]);
    if (tier == 0) LaunchTier<4, 128>(c, d_pairs, list, m, kTierK[0], d_limit, d_out);
    if (tier == 1) LaunchTier<8, 128>(c, d_pairs, list, m, kTierK[1], d_limit, d_out);
    if (tier == 2) LaunchTier<16, 64>(c, d_pairs, list, m, kTierK[2], d_limit, d_out);
    if (tier == 3) LaunchTier<32, 64>(c, d_pairs, list, m, kTierK[3], d_limit, d_out);
    TimerEnd(c);
    RVN_CUDA(cudaMemsetAsync(flag + m, 0, sizeof(uint32_t), c.stream));  // (the max below)
    OpenPairsKernel<<<CeilDiv(m, 256), 256, 0, c.stream>>>(d_pairs, list, m, kTierK[tier],
                                                           d_limit, d_out, flag, flag + m);
    ExclusiveScanU32(c, flag, pos, m);
    CompactKernel<uint32_t><<<CeilDiv(m, 256), 256, 0, c.stream>>>(list, flag, pos, m, spare);
    RVN_LAUNCH_CHECK();
    c.launches += 2;
    uint64_t open = 0;
    RVN_CUDA(cudaMemcpyAsync(&max_q_len, flag + m, sizeof(uint32_t), cudaMemcpyDeviceToHost,
                             c.stream));
    open = ReadU64(c, pos + m);
    std::swap(list, spare);
    m = static_cast<uint32_t>(open);
  }
}

// Global edit distances of n substring pairs of the uploaded reads. limit[i] >= 0:
// distances above it are reported as -1 (the caller only needs "beyond").
void EditDistanceBatch(Ctx& c, uint64_t n, const uint32_t* lhs_read, const uint32_t* lhs_begin,
                       const uint32_t* lhs_len, const uint32_t* rhs_read,
                       const uint32_t* rhs_begin, const uint32_t* rhs_len,
                       const uint8_t* strand, const int32_t* limit, int32_t* out) {
  if (n == 0) return;
  if (n >= 0xFFFFFFFFULL) throw LimitError("2^32 or more pairs");
  std::vector<PairDesc> h(n);
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t a = lhs_read[i], b = rhs_read[i];
    if (a >= c.n_reads || b >= c.n_reads) throw InvalidArgument("read index out of bounds");
    if (a < c.res_first || a >= c.res_last || b < c.res_first || b >= c.res_last) {
      throw StateError("the bases of these reads were not uploaded (rvn_reads_upload_range)");
    }
    if (static_cast<uint64_t>(lhs_begin[i]) + lhs_len[i] > c.h_len[a] ||
        static_cast<uint64_t>(rhs_begin[i]) + rhs_len[i] > c.h_len[b]) {
      throw InvalidArgument("substring beyond the end of its read");
    }
    h[i] = PairDesc{c.h_woff[a], c.h_woff[b], lhs_begin[i], lhs_len[i], rhs_begin[i],
                    rhs_len[i], strand[i] ? 1u : 0u, static_cast<uint32_t>(i)};
  }
  TimerBegin(c, "edit_distance");
  PairDesc* d_pairs = c.e_pairs.reserve(n);
  uint32_t* d_list = c.e_list.reserve(n);
  int32_t* d_out = c.e_dist.reserve(n);
  int32_t* d_limit = c.e_limit.reserve(n);
  std::vector<int32_t> h_limit(n), h_out(n, -1);
  std::vector<uint32_t> h_list(n);
  for (uint64_t i = 0; i < n; ++i) {
    h_limit[i] = limit ? limit[i] : -1;
    h_list[i] = static_cast<uint32_t>(i);
  }
  RVN_CUDA(cudaMemcpyAsync(d_pairs, h.data(), n * sizeof(PairDesc), cudaMemcpyHostToDevice,
                           c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_limit, h_limit.data(), n * 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_list, h_list.data(), n * 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_out, 0xFF, n * 4, c.stream));
  MyersTiers(c, d_pairs, d_list, static_cast<uint32_t>(n), d_limit, d_out);
  RVN_CUDA(cudaMemcpyAsync(h_out.data(), d_out, n * 4, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  TimerEnd(c);
  for (uint64_t i = 0; i < n; ++i) {
    int32_t v = h_out[i];
    if (limit && limit[i] >= 0 && v > limit[i]) v = -1;
    out[i] = v;
  }
}

// ---------------------------------------------------------------------------
// Stage 2's clip and identity filter on the device (construct.cc:385-424): the map's
// overlaps of a flush never leave the device before they are final.
// ---------------------------------------------------------------------------
namespace {

// one thread per overlap: OverlapUpdate against the valid regions (reads by their
// position in the uploaded set, pos_of[id]), and the edit-distance pair of a clipped one
__global__ void ClipKernel(const rvn_overlap* __restrict__ ovl, uint64_t n,
                           const uint32_t* __restrict__ pos_of, const uint32_t* __restrict__ rbeg,
                           const uint32_t* __restrict__ rend, const uint64_t* __restrict__ woff,
                           double identity, rvn_overlap* __restrict__ clipped,
                           PairDesc* __restrict__ pairs, int32_t* __restrict__ limit,
                           int32_t* __restrict__ dist, uint32_t* __restrict__ flag) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rvn_overlap o = ovl[i];
  const uint32_t lp = pos_of[o.lhs_id], rp = pos_of[o.rhs_id];
  const bool ok = OverlapClip(o.lhs_begin, o.lhs_end, o.rhs_begin, o.rhs_end, o.strand != 0,
                              PileRegion{rbeg[lp], rend[lp], false},
                              PileRegion{rbeg[rp], rend[rp], false});
  clipped[i] = o;
  flag[i] = ok ? 1u : 0u;
  dist[i] = -1;
  if (!ok) return;
  const uint32_t ll = o.lhs_end - o.lhs_begin, rl = o.rhs_end - o.rhs_begin;
  pairs[i] = PairDesc{woff[lp], woff[rp], o.lhs_begin, ll, o.rhs_begin, rl,
                      o.strand ? 1u : 0u, static_cast<uint32_t>(i)};
  const int32_t b = IdentityBound(identity, ll > rl ? ll : rl);
  limit[i] = b < 0 ? 0 : b;  // (decided below; the search stays bounded)
}

// keep = clipped and 1 - ed / max(len) >= identity (construct.cc:407-413)
__global__ void KeepKernel(const rvn_overlap* __restrict__ clipped, uint64_t n,
                           const int32_t* __restrict__ dist, double identity,
                           uint32_t* __restrict__ flag) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const rvn_overlap o = clipped[i];
  const uint32_t ll = o.lhs_end - o.lhs_begin, rl = o.rhs_end - o.rhs_begin;
  const int32_t d = dist[i];
  const double score = 1. - static_cast<double>(d) / static_cast<double>(ll > rl ? ll : rl);
  flag[i] = (d >= 0 && !(score < identity)) ? 1u : 0u;
}

__global__ void IotaListKernel(const uint32_t* __restrict__ flag, const uint64_t* __restrict__ pos,
                               uint64_t n, uint32_t* __restrict__ list) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) list[pos[i]] = static_cast<uint32_t>(i);
}

// per read of the flush: the first kept overlap (the scan at its first overlap)
__global__ void KeptOffsetsKernel(const uint64_t* __restrict__ pos, const uint64_t* __restrict__ off,
                                  uint32_t nr, uint64_t* __restrict__ out_off) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r <= nr) out_off[r] = pos[off[r]];
}

}  // namespace

uint64_t Stage2ClipFilter(Ctx& c, const rvn_overlap* d_ovl, const uint64_t* d_off, uint32_t nr,
                          uint64_t n, double identity, rvn_overlap* d_out, uint64_t* d_out_off) {
  if (n >= 0xFFFFFFFFULL) throw LimitError("2^32 or more overlaps in one flush");
  TimerBegin(c, "stage2_filter");
  rvn_overlap* clipped = c.e_ovl.reserve(n + 1);
  PairDesc* pairs = c.e_pairs.reserve(n + 1);
  int32_t* limit = c.e_limit.reserve(n + 1);
  int32_t* dist = c.e_dist.reserve(n + 1);
  uint32_t* flag = c.e_sflag.reserve(n + 1);
  uint32_t* list = c.e_list.reserve(n + 1);
  uint64_t* pos = c.e_sscan.reserve(n + 2);
  uint64_t kept = 0;
  if (n > 0) {
    const uint32_t blocks = CeilDiv(n, 256);
    ClipKernel<<<blocks, 256, 0, c.stream>>>(d_ovl, n, c.s2_pos_of.get(), c.s2_rbeg.get(),
                                             c.s2_rend.get(), c.d_woff.get(), identity, clipped,
                                             pairs, limit, dist, flag);
    ExclusiveScanU32(c, flag, pos, n);
    IotaListKernel<<<blocks, 256, 0, c.stream>>>(flag, pos, n, list);
    RVN_LAUNCH_CHECK();
    c.launches += 2;
    const uint64_t m = ReadU64(c, pos + n);
    MyersTiers(c, pairs, list, static_cast<uint32_t>(m), limit, dist);
    KeepKernel<<<blocks, 256, 0, c.stream>>>(clipped, n, dist, identity, flag);
    ExclusiveScanU32(c, flag, pos, n);
    CompactKernel<rvn_overlap><<<blocks, 256, 0, c.stream>>>(clipped, flag, pos, n, d_out);
    RVN_LAUNCH_CHECK();
    c.launches += 3;
  } else {
    RVN_CUDA(cudaMemsetAsync(pos, 0, sizeof(uint64_t), c.stream));
  }
  KeptOffsetsKernel<<<CeilDiv(nr + 1ULL, 256), 256, 0, c.stream>>>(pos, d_off, nr, d_out_off);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  kept = n > 0 ? ReadU64(c, pos + n) : 0;
  TimerEnd(c);
  return kept;
}

}  // namespace rvn
