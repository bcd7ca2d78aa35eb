// raven_b200 — minimizer index build and frequency filter on sm_90a.
//
// Replaces the index half of ram::MinimizerEngine::Minimize(first,last,
// minhash) and ram::MinimizerEngine::Filter (un-vendored; call sites
// RavenLib/src/construct.cc:42-44,363,372; SURVEY.md App. A.2).
//
// The reference keeps 2^14 hash buckets, radix-sorts each bucket by value and
// fills an unordered_map per bucket. Here the whole batch is ONE stable
// radix sort (radix.cu) of the (value, origin) records by value — the input is already
// in (read, position) order, so equal values keep exactly the reference's
// posting order — plus a direct-address bucket table over the top bits of
// the (uniformly mixed) value: a probe is one table read and one short scan
// of a sorted run, no hashing, no pointer chasing.
#include <algorithm>
#include <cmath>

#include <cooperative_groups.h>

#include "engine.cuh"
#include "seed.cuh"

namespace rvn {

namespace {

constexpr int kThreads = 256;

constexpr uint32_t kHistBins = 1u << 16;
constexpr uint32_t kSmemBins = 1024;

// One pass over the sorted values:
//   bucket[b] = index of the first record whose (value >> shift) >= b;
//   hist[len] += 1 for every run of equal values (a key) of that many postings
//     (lengths >= kHistBins-1 land in the last bin; nearly every run has
//     length 1..3, so short lengths go through a shared-memory histogram);
//   hist[kHistBins] = number of keys.
// (minimizer values are minima of hashes: the top of the value range is nearly
// empty, so a few records own millions of buckets - those gaps are handed to
// FillLongGaps instead of being filled by one thread)
constexpr uint32_t kShortGap = 1024;
constexpr uint32_t kMaxLongGaps = 1u << 20;

template <typename ValT, bool kFill>
__global__ void __launch_bounds__(kThreads)
IndexTableKernel(const ValT* __restrict__ val, uint64_t n, int shift,
                 uint32_t n_buckets, uint32_t* __restrict__ bucket,
                 unsigned long long* __restrict__ hist, uint64_t* __restrict__ gaps) {
  __shared__ uint32_t sh[kSmemBins];
  __shared__ uint32_t keys;
  __shared__ uint32_t warp_first[kThreads / 32];
  for (uint32_t i = threadIdx.x; i < kSmemBins; i += kThreads) sh[i] = 0;
  if (threadIdx.x == 0) keys = 0;
  __syncthreads();
  // persistent CTAs: the shared histogram is set up and flushed once per CTA
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kThreads;
  for (uint64_t base = static_cast<uint64_t>(blockIdx.x) * kThreads; base <= n; base += stride) {
  const uint64_t i = base + threadIdx.x;
  bool start = false;
  uint32_t len = 0;
  uint64_t fill_lo = 0, mine = 0;
  uint32_t fill_cnt = 0;  // buckets (prev_bucket, this_bucket] this record owns
  if (i <= n) {
    const uint64_t prev = i == 0 ? 0 : val[i - 1];
    const uint64_t cur = i == n ? 0 : val[i];
    // record i is the first one of buckets (prev_bucket, this_bucket]
    const uint64_t lo = i == 0 ? 0 : (prev >> shift) + 1;
    const uint64_t hi = i == n ? n_buckets : (cur >> shift);
    if (kFill && hi >= lo) {
      if (hi + 1 - lo <= kShortGap) {
        fill_lo = lo;
        fill_cnt = static_cast<uint32_t>(hi + 1 - lo);
      } else {
        const unsigned long long g = atomicAdd(&hist[kHistBins + 1], 1ULL);
        if (g < kMaxLongGaps) {
          gaps[3 * g] = lo;
          gaps[3 * g + 1] = hi;
          gaps[3 * g + 2] = i;
        } else {  // (never seen: the list holds a million gaps)
          for (uint64_t b = lo; b <= hi; ++b) bucket[b] = static_cast<uint32_t>(i);
        }
      }
    }
    start = i < n && (i == 0 || cur != prev);  // a run starts here
    mine = cur;
  }
  // Run length = distance to the next run start: found in the warp's ballot, else
  // in the following warps of this tile (shared memory), else - the run crosses
  // the tile end - by scanning on from there. (A per-thread forward scan costs
  // every warp its longest run in dependent loads.) The virtual record n ends
  // the last run.
  {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t marks = __ballot_sync(0xFFFFFFFFu, start || i == n);
    if (lane == 0) warp_first[wid] = marks ? static_cast<uint32_t>(__ffs(marks) - 1) : 32u;
    __syncthreads();
    if (start) {
      const uint32_t above = lane == 31 ? 0u : (marks & ~((2u << lane) - 1u));
      if (above) {
        len = static_cast<uint32_t>(__ffs(above) - 1) - lane;
      } else {
        len = 32 - lane;
        uint32_t w2 = wid + 1;
        while (w2 < kThreads / 32 && warp_first[w2] == 32u) {
          len += 32;
          ++w2;
        }
        if (w2 < kThreads / 32) {
          len += warp_first[w2];
        } else {
          uint64_t pos = base + kThreads;
          while (len < kHistBins - 1 && pos < n && val[pos] == mine) {
            ++pos;
            ++len;
          }
        }
      }
      if (len > kHistBins - 1) len = kHistBins - 1;
    }
    __syncthreads();
  }
  // the warp fills its records' buckets together (a per-thread loop would run
  // as long as the widest gap among the 32 records): slot t of the warp's
  // total belongs to the lane found by a shuffle search over the prefixes
  {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t total;
    const uint32_t rel = WarpExclusiveSum(fill_cnt, lane, &total);
    for (uint32_t t0 = 0; t0 < total; t0 += 32) {
      const uint32_t t = t0 + lane;
      const uint32_t q = WarpSlotLane(rel, t);
      const uint32_t qrel = __shfl_sync(0xFFFFFFFFu, rel, q);
      const uint64_t qlo = __shfl_sync(0xFFFFFFFFu, fill_lo, q);
      if (kFill && t < total) bucket[qlo + (t - qrel)] = static_cast<uint32_t>(base + (threadIdx.x & ~31u) + q);
    }
  }
  // warp-aggregated: nearly all runs have the same few lengths
  const uint32_t starts = __ballot_sync(0xFFFFFFFFu, start);
  if (start) {
    const uint32_t same = __match_any_sync(starts, len);
    if ((threadIdx.x & 31) == static_cast<uint32_t>(__ffs(same) - 1)) {
      if (len < kSmemBins) {
        atomicAdd(&sh[len], static_cast<uint32_t>(__popc(same)));
      } else {
        atomicAdd(&hist[len], static_cast<unsigned long long>(__popc(same)));
      }
    }
  }
  if ((threadIdx.x & 31) == 0 && starts) atomicAdd(&keys, static_cast<uint32_t>(__popc(starts)));

  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < kSmemBins; b += kThreads) {
    if (sh[b]) atomicAdd(&hist[b], static_cast<unsigned long long>(sh[b]));
  }
  if (threadIdx.x == 0 && keys) atomicAdd(&hist[kHistBins], static_cast<unsigned long long>(keys));
}

__global__ void __launch_bounds__(kThreads)
FillLongGaps(const uint64_t* __restrict__ gaps, uint32_t* __restrict__ bucket) {
  const uint64_t lo = gaps[3ULL * blockIdx.x], hi = gaps[3ULL * blockIdx.x + 1];
  const uint32_t v = static_cast<uint32_t>(gaps[3ULL * blockIdx.x + 2]);
  for (uint64_t b = lo + threadIdx.x; b <= hi; b += kThreads) bucket[b] = v;
}

// exact lengths of the runs of kHistBins-1 or more postings (rare)
template <typename ValT>
__global__ void CollectLongRuns(const ValT* __restrict__ val, uint64_t n,
                                unsigned long long* __restrict__ counter,
                                uint32_t* __restrict__ out) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n || (i > 0 && val[i] == val[i - 1])) return;
  if (i + (kHistBins - 2) >= n || val[i + (kHistBins - 2)] != val[i]) return;
  uint64_t len = kHistBins - 1;
  while (i + len < n && val[i + len] == val[i]) ++len;
  out[atomicAdd(counter, 1ULL)] = static_cast<uint32_t>(len);
}

__global__ void NarrowValuesKernel(const uint64_t* __restrict__ in, uint64_t n,
                                   uint32_t* __restrict__ out) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<uint32_t>(in[i]);
}

// ---- tiers ------------------------------------------------------------------
// Stage 1 probes the index with micromizers only: with T = the largest micromizer
// value of every query read, a record whose value exceeds T can never be hit.
// Such records (about three in four at k = 15, w = 5) still count for the
// occurrence threshold, which ranks the multiplicities of ALL keys - so they are
// sorted as bare 4-byte keys, while only the probe-able tier carries its origins
// through the sort and into the table. Stable partition: count, scan, scatter.
constexpr uint32_t kTierTile = 4096;  // records per CTA (16 warp steps of 32 per warp x 8)

__global__ void __launch_bounds__(kThreads)
TierCountKernel(const uint32_t* __restrict__ val, uint64_t n, uint32_t limit,
                uint32_t* __restrict__ tile_cnt) {
  __shared__ uint32_t sm[34];
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * kTierTile;
  uint32_t mine = 0;
#pragma unroll
  for (uint32_t i = 0; i < kTierTile / kThreads; ++i) {
    const uint64_t idx = base + i * kThreads + threadIdx.x;
    mine += (idx < n && val[idx] <= limit) ? 1u : 0u;
  }
  uint32_t total;
  BlockExclusiveSum<uint32_t, kThreads>(mine, sm, &total);
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads, 4)
TierScatterKernel(const uint32_t* __restrict__ val, const uint64_t* __restrict__ org, uint64_t n,
                  uint32_t limit, const uint64_t* __restrict__ tile_off_a,
                  uint32_t* __restrict__ a_val, uint64_t* __restrict__ a_org,
                  uint32_t* __restrict__ b_val) {
  __shared__ uint32_t warp_a[kThreads / 32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr uint32_t kWarpSpan = kTierTile / (kThreads / 32);  // 512 consecutive records
  const uint64_t tile_base = static_cast<uint64_t>(blockIdx.x) * kTierTile;
  const uint64_t warp_base = tile_base + warp * kWarpSpan;
  uint32_t v[kWarpSpan / 32];
  uint32_t cnt = 0;
#pragma unroll
  for (uint32_t i = 0; i < kWarpSpan / 32; ++i) {
    const uint64_t idx = warp_base + i * 32 + lane;
    v[i] = idx < n ? val[idx] : 0xFFFFFFFFu;
  }
#pragma unroll
  for (uint32_t i = 0; i < kWarpSpan / 32; ++i) {
    const uint64_t idx = warp_base + i * 32 + lane;
    cnt += __popc(__ballot_sync(0xFFFFFFFFu, idx < n && v[i] <= limit));
  }
  if (lane == 0) warp_a[warp] = cnt;
  __syncthreads();
  uint64_t a_at = tile_off_a[blockIdx.x];
  for (uint32_t w = 0; w < warp; ++w) a_at += warp_a[w];
  uint64_t b_at = warp_base - a_at;  // records before this warp that are not in tier A
  // origins in batches of 8 independent loads (all 16 at once cost too many registers)
#pragma unroll
  for (uint32_t h = 0; h < kWarpSpan / 32; h += 8) {
    uint64_t o[8];
#pragma unroll
    for (uint32_t u = 0; u < 8; ++u) {
      const uint64_t idx = warp_base + (h + u) * 32 + lane;
      o[u] = (idx < n && v[h + u] <= limit) ? org[idx] : 0;
    }
#pragma unroll
    for (uint32_t u = 0; u < 8; ++u) {
      const uint32_t i = h + u;
      const uint64_t idx = warp_base + i * 32 + lane;
      const bool in = idx < n;
      const bool is_a = in && v[i] <= limit;
      const uint32_t ma = __ballot_sync(0xFFFFFFFFu, is_a);
      const uint32_t mb = __ballot_sync(0xFFFFFFFFu, in && !is_a);
      const uint32_t below = (1u << lane) - 1u;
      if (is_a) {
        const uint64_t d = a_at + __popc(ma & below);
        a_val[d] = v[i];
        a_org[d] = o[u];
      } else if (in) {
        b_val[b_at + __popc(mb & below)] = v[i];
      }
      a_at += __popc(ma);
      b_at += __popc(mb);
    }
  }
}

// Chunked build: a coarse histogram of the sketch values (top kCapBits key bits) bounds
// the sizes of both tiers before the limit is known to the chunks
constexpr int kCapBits = 10;
constexpr uint32_t kCapBins = 1u << kCapBits;

__global__ void __launch_bounds__(kThreads)
ValueHistKernel(const uint32_t* __restrict__ val, uint64_t n, int shift,
                unsigned long long* __restrict__ hist) {
  __shared__ uint32_t sh[kCapBins];
  for (uint32_t i = threadIdx.x; i < kCapBins; i += kThreads) sh[i] = 0;
  __syncthreads();
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kThreads;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x; i < n;
       i += stride) {
    atomicAdd(&sh[(val[i] >> shift) & (kCapBins - 1)], 1u);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kCapBins; i += kThreads) {
    if (sh[i]) atomicAdd(&hist[i], static_cast<unsigned long long>(sh[i]));
  }
}

__global__ void MaxU64Kernel(const uint64_t* __restrict__ v, uint64_t n,
                             unsigned long long* __restrict__ out) {
  unsigned long long m = 0;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    m = max(m, static_cast<unsigned long long>(v[i]));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, d));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// Multiplicities of bare keys that are sorted by their bits above `low` only (two
// radix passes instead of three at k = 15): the keys of one group (equal upper bits,
// ~600 keys at C2) are contiguous, a warp counts a group's low bits in 1024 shared
// counters and reads the run lengths off them - the histogram IndexTableKernel<.,
// false> takes from fully sorted keys, without the third pass. A warp owns the
// groups that START in its chunk.
constexpr uint32_t kGroupChunk = 4096;
constexpr int kGroupLowBits = 10;

__global__ void __launch_bounds__(kThreads)
GroupCountKernel(const uint32_t* __restrict__ key, uint64_t n, unsigned long long* __restrict__ hist) {
  __shared__ uint32_t sh[kSmemBins];
  __shared__ __align__(16) uint32_t cnt[kThreads / 32][1u << kGroupLowBits];
  __shared__ uint32_t keys_total;
  for (uint32_t i = threadIdx.x; i < kSmemBins; i += kThreads) sh[i] = 0;
  if (threadIdx.x == 0) keys_total = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t* my = cnt[wid];
  const uint32_t low_mask = (1u << kGroupLowBits) - 1;
  uint32_t h1 = 0, h2 = 0, h3 = 0, h4 = 0, nkeys = 0;
  const uint64_t n_chunks = (n + kGroupChunk - 1) / kGroupChunk;
  for (uint64_t chunk = static_cast<uint64_t>(blockIdx.x) * (kThreads / 32) + wid; chunk < n_chunks;
       chunk += static_cast<uint64_t>(gridDim.x) * (kThreads / 32)) {
    const uint64_t start = chunk * kGroupChunk;
    const uint64_t end = min(n, start + kGroupChunk);
    uint64_t pos = start;
    if (start > 0) {  // the group that began before the chunk is the previous warp's
      const uint32_t gprev = key[start - 1] >> kGroupLowBits;
      while (true) {
        const uint64_t idx = pos + lane;
        const bool in = idx < n && (key[idx] >> kGroupLowBits) == gprev;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, in);
        const uint32_t c = m == 0xFFFFFFFFu ? 32u : static_cast<uint32_t>(__ffs(~m) - 1);
        pos += c;
        if (c < 32) break;
      }
    }
    while (pos < end) {
      const uint32_t g = key[pos] >> kGroupLowBits;
      uint4* my4 = reinterpret_cast<uint4*>(my);
#pragma unroll
      for (uint32_t t = 0; t < (1u << kGroupLowBits) / 128; ++t) my4[t * 32 + lane] = make_uint4(0, 0, 0, 0);
      __syncwarp();
      bool open = true;
      while (open) {  // 128 keys per round: four independent loads per lane
        uint32_t k4[4];
#pragma unroll
        for (uint32_t u = 0; u < 4; ++u) {
          const uint64_t idx = pos + u * 32 + lane;
          k4[u] = idx < n ? key[idx] : ~(g << kGroupLowBits);
        }
#pragma unroll
        for (uint32_t u = 0; u < 4; ++u) {
          if (open) {
            const bool in = (k4[u] >> kGroupLowBits) == g;
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, in);
            if (in) atomicAdd(&my[k4[u] & low_mask], 1u);
            const uint32_t c = m == 0xFFFFFFFFu ? 32u : static_cast<uint32_t>(__ffs(~m) - 1);
            pos += c;
            open = c == 32;
          }
        }
      }
      __syncwarp();
#pragma unroll
      for (uint32_t t = 0; t < (1u << kGroupLowBits) / 128; ++t) {
        const uint4 q = my4[t * 32 + lane];
        if ((q.x | q.y | q.z | q.w) == 0) continue;
        const uint32_t cs[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const uint32_t c = cs[x];
          if (c == 0) continue;
          ++nkeys;
          if (c <= 4) {
            h1 += c == 1;
            h2 += c == 2;
            h3 += c == 3;
            h4 += c == 4;
          } else if (c < kSmemBins) {
            atomicAdd(&sh[c], 1u);
          } else {
            atomicAdd(&hist[min(c, kHistBins - 1)], 1ULL);
          }
        }
      }
      __syncwarp();
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    h1 += __shfl_xor_sync(0xFFFFFFFFu, h1, d);
    h2 += __shfl_xor_sync(0xFFFFFFFFu, h2, d);
    h3 += __shfl_xor_sync(0xFFFFFFFFu, h3, d);
    h4 += __shfl_xor_sync(0xFFFFFFFFu, h4, d);
    nkeys += __shfl_xor_sync(0xFFFFFFFFu, nkeys, d);
  }
  if (lane == 0) {
    atomicAdd(&sh[1], h1);
    atomicAdd(&sh[2], h2);
    atomicAdd(&sh[3], h3);
    atomicAdd(&sh[4], h4);
    atomicAdd(&keys_total, nkeys);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kSmemBins; i += kThreads) {
    if (sh[i]) atomicAdd(&hist[i], static_cast<unsigned long long>(sh[i]));
  }
  if (threadIdx.x == 0 && keys_total) {
    atomicAdd(&hist[kHistBins], static_cast<unsigned long long>(keys_total));
  }
}

// Multiplicities of bare keys that are only partitioned on their top kBareBucketBits
// bits (bucket = 2^span_bits consecutive values; one bucket of all values when the
// keys have 20 bits or fewer and were not partitioned at all). A cluster of C CTAs
// owns one bucket at a time and counts it in u32 counters spread over the CTAs'
// shared memory (distributed shared memory): value u of a sweep belongs to CTA
// u >> slot_bits, counter u & (2^slot_bits - 1). Every CTA streams its 1/C of the
// bucket's keys with coalesced loads and adds 1 to the owner's counter; after the
// cluster barrier every CTA reads its own counters off as runs (nonzero counter =
// one key, its value = the run length) - the histogram GroupCountKernel and
// IndexTableKernel<., false> take from sorted keys - and clears them. A bucket wider
// than the cluster's counters takes several sweeps over its keys (the repeats read
// the bucket from L2).
constexpr int kBareBucketBits = 10;
constexpr int kBareThreads = 1024;
constexpr int kBareSlotBits = 15;  // 32768 counters = 128 KB per CTA

__global__ void __launch_bounds__(kBareThreads, 1)
BareCountKernel(const uint32_t* __restrict__ key, uint64_t n, const uint32_t* __restrict__ bstart,
                uint32_t first_bucket, uint32_t n_buckets, int span_bits, int slot_bits,
                unsigned long long* __restrict__ hist) {
  extern __shared__ __align__(16) uint32_t bare_smem[];
  __shared__ uint32_t keys_total;
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t csize = cluster.num_blocks();
  const uint32_t crank = cluster.block_rank();
  const uint32_t n_slots = 1u << slot_bits;
  uint32_t* ctr = bare_smem;
  uint32_t* sh = bare_smem + n_slots;  // kSmemBins
  for (uint32_t i = threadIdx.x; i < n_slots; i += kBareThreads) ctr[i] = 0;
  for (uint32_t i = threadIdx.x; i < kSmemBins; i += kBareThreads) sh[i] = 0;
  if (threadIdx.x == 0) keys_total = 0;
  const uint32_t ctr_addr = static_cast<uint32_t>(__cvta_generic_to_shared(ctr));
  const uint32_t span_mask = (1u << span_bits) - 1u;
  const uint32_t sweep_span = n_slots * csize;  // (csize: a power of two)
  const uint32_t slot_mask = n_slots - 1u;
  uint32_t h1 = 0, h2 = 0, h3 = 0, h4 = 0, nkeys = 0;
  cluster.sync();  // every CTA's counters are zero before the first remote add
  const uint32_t n_clusters = gridDim.x / csize;
  for (uint32_t b = first_bucket + blockIdx.x / csize; b < n_buckets; b += n_clusters) {
    const uint64_t lo = bstart ? bstart[b] : 0;
    const uint64_t hi = bstart && b + 1 < n_buckets ? bstart[b + 1] : n;
    if (lo >= hi) continue;  // (the same for every CTA of the cluster)
    for (uint64_t s0 = 0; s0 <= span_mask; s0 += sweep_span) {
      constexpr int kUnroll = 4;
      const uint64_t stride = static_cast<uint64_t>(csize) * kBareThreads;
      for (uint64_t i0 = lo + crank * kBareThreads + threadIdx.x; i0 < hi; i0 += kUnroll * stride) {
        uint32_t k4[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint64_t i = i0 + u * stride;
          k4[u] = i < hi ? key[i] : 0u;
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint64_t v = static_cast<uint64_t>(k4[u] & span_mask) - s0;
          if (i0 + u * stride < hi && v < sweep_span) {
            const uint32_t owner = static_cast<uint32_t>(v) >> slot_bits;
            const uint32_t local = ctr_addr + 4u * (static_cast<uint32_t>(v) & slot_mask);
            uint32_t remote;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(owner));
            asm volatile("red.relaxed.cluster.shared::cluster.add.u32 [%0], 1;" ::"r"(remote) : "memory");
          }
        }
      }
      cluster.sync();  // every add of the sweep has landed
      for (uint32_t t = threadIdx.x; t < n_slots; t += kBareThreads) {
        const uint32_t c = ctr[t];
        if (c == 0) continue;
        ctr[t] = 0;
        ++nkeys;
        if (c <= 4) {
          h1 += c == 1;
          h2 += c == 2;
          h3 += c == 3;
          h4 += c == 4;
        } else if (c < kSmemBins) {
          atomicAdd(&sh[c], 1u);
        } else {
          atomicAdd(&hist[min(c, kHistBins - 1)], 1ULL);
        }
      }
      cluster.sync();  // every counter is clear before the next sweep's adds
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    h1 += __shfl_xor_sync(0xFFFFFFFFu, h1, d);
    h2 += __shfl_xor_sync(0xFFFFFFFFu, h2, d);
    h3 += __shfl_xor_sync(0xFFFFFFFFu, h3, d);
    h4 += __shfl_xor_sync(0xFFFFFFFFu, h4, d);
    nkeys += __shfl_xor_sync(0xFFFFFFFFu, nkeys, d);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&sh[1], h1);
    atomicAdd(&sh[2], h2);
    atomicAdd(&sh[3], h3);
    atomicAdd(&sh[4], h4);
    atomicAdd(&keys_total, nkeys);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kSmemBins; i += kBareThreads) {
    if (sh[i]) atomicAdd(&hist[i], static_cast<unsigned long long>(sh[i]));
  }
  if (threadIdx.x == 0 && keys_total) {
    atomicAdd(&hist[kHistBins], static_cast<unsigned long long>(keys_total));
  }
}

// run-length histogram + #keys of the n bare keys (all > limit) in `keys`, added to
// hist; bstart: first key of every bucket of the partition (nullptr: not partitioned,
// keys of at most 2 * kBareBucketBits bits)
void BareCount(Ctx& c, const uint32_t* keys, uint64_t n, int key_bits, uint32_t limit,
               const uint32_t* bstart, unsigned long long* hist) {
  const int span_bits = bstart ? key_bits - kBareBucketBits : key_bits;
  const uint32_t n_buckets = bstart ? (1u << kBareBucketBits) : 1u;
  const uint32_t first_bucket = bstart ? (limit >> span_bits) : 0u;
  if (c.bare_cluster == 0) {
    // cluster size: the option's, else 8 (portable; on an H100 it measured faster than
    // 16 with its half as many sweeps: the remote adds bound the kernel, not the reads)
    const int size = c.bare_count > 1 ? static_cast<int>(c.bare_count) : 8;
    const size_t smem = ((1u << kBareSlotBits) + kSmemBins) * sizeof(uint32_t);
    RVN_CUDA(cudaFuncSetAttribute(BareCountKernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem)));
    RVN_CUDA(cudaFuncSetAttribute(BareCountKernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(size));
    cfg.blockDim = dim3(kBareThreads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = static_cast<unsigned>(size);
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    RVN_CUDA(cudaOccupancyMaxActiveClusters(&clusters, BareCountKernel, &cfg));
    if (clusters < 1) throw CudaError("BareCountKernel: a cluster does not fit the device");
    c.bare_cluster = size;
    c.bare_clusters = clusters;
  }
  const int csize = c.bare_cluster;
  int log_c = 0;
  while ((1 << log_c) < csize) ++log_c;
  const int slot_bits = std::max(0, std::min(kBareSlotBits, span_bits - log_c));
  const unsigned clusters =
      static_cast<unsigned>(std::min<uint64_t>(n_buckets - first_bucket, c.bare_clusters));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(clusters * csize);
  cfg.blockDim = dim3(kBareThreads);
  cfg.dynamicSmemBytes = ((1u << slot_bits) + kSmemBins) * sizeof(uint32_t);
  cfg.stream = c.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = static_cast<unsigned>(csize);
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  RVN_CUDA(cudaLaunchKernelEx(&cfg, BareCountKernel, keys, n, bstart, first_bucket, n_buckets,
                              span_bits, slot_bits, hist));
  RVN_LAUNCH_CHECK();
  ++c.launches;
}

// largest micromizer value of the reads of t: the largest of their selection thresholds
uint64_t MaxThreshold(Ctx& c, const Thresholds& t) {
  uint64_t* w = c.m_counter.reserve(8);
  RVN_CUDA(cudaMemsetAsync(w, 0, sizeof(uint64_t), c.stream));
  const uint64_t n = t.last - t.first;
  MaxU64Kernel<<<std::min<unsigned>(CeilDiv(n, 256), c.sms * 8), 256, 0, c.stream>>>(
      t.val.get(), n, reinterpret_cast<unsigned long long*>(w));
  RVN_LAUNCH_CHECK();
  ++c.launches;
  return ReadU64(c, w);
}

}  // namespace

// largest micromizer value of reads [first, last) (c.qt)
uint64_t MaxMicromizerValue(Ctx& c, uint32_t first, uint32_t last) {
  EnsureThresholds(c, first, last);
  if (last <= first) return 0;
  if (!c.sk.is32) return ~0ULL;  // (tiers are only built over u32 values)
  return MaxThreshold(c, c.qt);
}

void BuildIndex(Ctx& c, uint32_t first, uint32_t last, bool minhash, uint64_t value_limit) {
  c.i_valid = false;
  c.occurrence = 0xFFFFFFFFu;
  EnsureSketch(c, first, last);
  if (minhash) EnsureMicromizers(c, first, last);
  const RecordSet& src = minhash ? c.mm : c.sk;
  c.i_first = first;
  c.i_last = last;
  BuildIndexFrom(c, src.Values(), src.org.get(), src.n, ReadBases(c, first, last),
                 minhash ? ~0ULL : value_limit, /*count_bare=*/true);
  c.i_sorted_ids = c.ids_ascending;
  c.i_from_sketch = !minhash;
}

namespace {

// the build splits a batch into tiers (index.cu, tiers): u32 values, a real limit and
// an input worth a partition pass
bool Tiered(const Ctx& c, bool is32, uint64_t value_limit, uint64_t n) {
  const int key_bits = static_cast<int>(2 * c.prm.k);
  const uint64_t value_mask = key_bits >= 64 ? ~0ULL : ((1ULL << key_bits) - 1);
  return is32 && value_limit < value_mask && n >= c.tier_min_records;
}

// The index of n records. pre_split < 0: the records are src_val / src_org. Otherwise
// the chunked build has laid them out already: tiered, tier A (pre_split records) in
// c.i_val_alt / c.i_org_alt and the n - pre_split bare keys in c.t_b0; untiered, all n
// in c.i_val_alt / c.i_org_alt (= src_val / src_org), the sort's second buffers.
void BuildIndexImpl(Ctx& c, ValView src_val, const uint64_t* src_org, uint64_t n,
                    uint64_t index_bases, uint64_t value_limit, bool count_bare,
                    int64_t pre_split);

}  // namespace

void BuildIndexFrom(Ctx& c, ValView src_val, const uint64_t* src_org, uint64_t n,
                    uint64_t index_bases, uint64_t value_limit, bool count_bare) {
  BuildIndexImpl(c, src_val, src_org, n, index_bases, value_limit, count_bare, -1);
}

namespace {

void BuildIndexImpl(Ctx& c, ValView src_val, const uint64_t* src_org, uint64_t n,
                    uint64_t index_bases, uint64_t value_limit, bool count_bare,
                    int64_t pre_split) {
  c.i_valid = false;
  c.i_sorted_ids = false;
  c.i_from_sketch = false;
  c.i_build_held = false;
  c.occurrence = 0xFFFFFFFFu;
  ++c.i_gen;  // (results derived from an earlier index are stale)
  if (n >= 0xFFFFFFFFULL) {
    throw LimitError("index batch holds 2^32 or more minimizers");
  }
  c.i_n = n;
  c.i_keys = 0;
  // 8-byte values that fit 30 bits (records of a partitioned run arrive in the
  // 16-byte exchange format): one narrowing copy, then the u32 path
  if (!src_val.is32 && 2 * c.prm.k <= 30 && n > 0) {
    uint32_t* narrow = reinterpret_cast<uint32_t*>(c.t_narrow.reserve(n / 2 + 2));
    NarrowValuesKernel<<<CeilDiv(n, kThreads), kThreads, 0, c.stream>>>(
        static_cast<const uint64_t*>(src_val.p), n, narrow);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    src_val = ValView{narrow, 1};
  }
  const bool is32 = src_val.is32 != 0;
  c.i_is32 = is32;

  const int key_bits = static_cast<int>(2 * c.prm.k);
  const uint64_t value_mask = key_bits >= 64 ? ~0ULL : ((1ULL << key_bits) - 1);
  const bool tiered = Tiered(c, is32, value_limit, n);
  const uint32_t limit32 = static_cast<uint32_t>(value_limit);
  c.i_limit = tiered ? value_limit : ~0ULL;
  uint64_t n_a = n, n_b = 0;
  const uint32_t* sorted_b = nullptr;
  const bool bare = tiered && count_bare && c.bare_count != 0;
  const uint32_t* bstart = nullptr;  // (bare: buckets of the partitioned keys)

  TimerBegin(c, "index_sort");
  // stable LSD radix sort on the value bits (radix.cu). The sketch arrays are
  // only read (they still serve the queries of this batch); values of up to 30
  // bits (k <= 15) are u32 keys straight from the sketch kernel: 12 instead of
  // 16 bytes per record and pass, three 10-bit passes at k = 15.
  if (tiered) {
    const uint32_t* a_val;
    const uint64_t* a_org;
    uint32_t* b_src;
    if (pre_split >= 0) {
      n_a = static_cast<uint64_t>(pre_split);
      n_b = n - n_a;
      a_val = reinterpret_cast<const uint32_t*>(c.i_val_alt.get());
      a_org = c.i_org_alt.get();
      b_src = reinterpret_cast<uint32_t*>(c.t_b0.get());
    } else {
      const uint32_t* src32 = static_cast<const uint32_t*>(src_val.p);
      const uint64_t tiles = (n + kTierTile - 1) / kTierTile;
      uint32_t* tcnt = c.t_cnt.reserve(tiles + 1);
      uint64_t* toff = c.t_off.reserve(tiles + 2);
      TierCountKernel<<<static_cast<unsigned>(tiles), kThreads, 0, c.stream>>>(src32, n, limit32,
                                                                            tcnt);
      ExclusiveScanU32(c, tcnt, toff, tiles);
      n_a = ReadU64(c, toff + tiles);
      n_b = n - n_a;
      uint32_t* av = reinterpret_cast<uint32_t*>(c.t_aval.reserve(n_a / 2 + 2));
      uint64_t* ao = c.t_aorg.reserve(n_a + 1);
      b_src = reinterpret_cast<uint32_t*>(c.t_b0.reserve(n_b / 2 + 2));
      TierScatterKernel<<<static_cast<unsigned>(tiles), kThreads, 0, c.stream>>>(
          src32, src_org, n, limit32, toff, av, ao, b_src);
      RVN_LAUNCH_CHECK();
      c.launches += 2;
      a_val = av;
      a_org = ao;
    }
    // the probe-able tier: values <= limit need fewer key bits
    int bits_a = 1;
    while (bits_a < key_bits && (value_limit >> bits_a) != 0) ++bits_a;
    c.i_val.reserve(n_a / 2 + 2);
    c.i_val_alt.reserve(n_a / 2 + 2);
    c.i_org.reserve(n_a + 1);
    c.i_org_alt.reserve(n_a + 1);
    if (n_a > 0) {
      const int where = RadixSortPairs(c, a_val, reinterpret_cast<uint32_t*>(c.i_val.get()),
                                       reinterpret_cast<uint32_t*>(c.i_val_alt.get()), a_org,
                                       c.i_org.get(), c.i_org_alt.get(), n_a, 0, bits_a);
      if (where == 1) {
        c.i_val.swap(c.i_val_alt);
        c.i_org.swap(c.i_org_alt);
      }
    }
    // the rest: bare keys, only their multiplicities matter
    uint32_t* b1 = reinterpret_cast<uint32_t*>(c.t_b1.reserve(n_b / 2 + 2));
    if (bare) {
      // one unstable partition on the top kBareBucketBits key bits (none when every
      // key fits one bucket), BareCountKernel counts inside the buckets
      c.t_b2.release();
      c.t_b_low = 0;
      c.t_b_sorted = false;
      sorted_b = n_b > 0 ? b_src : nullptr;
      if (n_b > 0 && key_bits > 2 * kBareBucketBits) {
        uint32_t* starts = c.t_bstart.reserve(1u << kBareBucketBits);
        RadixPartitionKeys(c, b_src, b1, n_b, key_bits - kBareBucketBits, key_bits, starts);
        sorted_b = b1;
        bstart = starts;
      }
    } else {
      uint32_t* b2 = reinterpret_cast<uint32_t*>(c.t_b2.reserve(n_b / 2 + 2));
      // (sorted above their low bits only: GroupCountKernel reads the multiplicities
      //  off groups of equal upper bits)
      // - while a group holds a few hundred keys: the rank of a partitioned run owns
      // 1/N of the keys of every group, and zeroing and reading 1024 counters per
      // group then costs more than the third pass
      const uint64_t n_groups = ((value_mask - value_limit) >> kGroupLowBits) + 1;
      c.t_b_low = (key_bits > 2 * kGroupLowBits && n_b / n_groups >= c.group_count_min)
                      ? kGroupLowBits
                      : 0;
      c.t_b_sorted = c.t_b_low == 0;
      if (n_b > 0) {
        const int where = RadixSortKeys(c, b_src, b1, b2, n_b, c.t_b_low, key_bits);
        sorted_b = where < 0 ? b_src : (where == 0 ? b1 : b2);
      }
    }
    c.t_sorted_b = sorted_b;
    c.t_nb = n_b;
  } else {
    const uint64_t val_elems = is32 ? n / 2 + 2 : n + 1;
    c.i_val.reserve(val_elems);
    c.i_val_alt.reserve(val_elems);
    c.i_org.reserve(n + 1);
    c.i_org_alt.reserve(n + 1);
    if (n > 0) {
      int where;
      if (is32) {
        where = RadixSortPairs(c, static_cast<const uint32_t*>(src_val.p),
                               reinterpret_cast<uint32_t*>(c.i_val.get()),
                               reinterpret_cast<uint32_t*>(c.i_val_alt.get()), src_org,
                               c.i_org.get(), c.i_org_alt.get(), n, 0, key_bits);
      } else {
        where = RadixSortPairs(c, static_cast<const uint64_t*>(src_val.p), c.i_val.get(),
                               c.i_val_alt.get(), src_org, c.i_org.get(), c.i_org_alt.get(), n, 0,
                               key_bits);
      }
      if (where == 1) {
        c.i_val.swap(c.i_val_alt);
        c.i_org.swap(c.i_org_alt);
      }
    }
    c.t_sorted_b = nullptr;
    c.t_nb = 0;
    c.t_b_sorted = true;
  }
  c.i_n = n_a;
  TimerEnd(c);
  const uint64_t* kv = c.i_val.get();

  TimerBegin(c, "index_table");
  // bucket table over the top bits of the (probe-able) value range + run-length
  // histogram + #keys
  int top_bits = key_bits;  // values are below 2^top_bits
  if (tiered) {
    top_bits = 1;
    while (top_bits < key_bits && (value_limit >> top_bits) != 0) ++top_bits;
  }
  int bits = 8;
  while (bits < 28 && (1ULL << (bits + 1)) <= n_a) ++bits;
  bits = std::min<int>(bits, top_bits);
  c.i_bucket_bits = bits;
  const int shift = top_bits - bits;
  c.i_shift = shift;
  const uint32_t n_buckets =
      tiered ? static_cast<uint32_t>((value_limit >> shift) + 1) : (1u << bits);
  uint32_t* bucket = c.i_bucket.reserve(n_buckets + 2ULL);
  static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "");
  uint64_t* hist = c.i_hist.reserve(kHistBins + 8);
  RVN_CUDA(cudaMemsetAsync(hist, 0, (kHistBins + 8) * sizeof(uint64_t), c.stream));
  uint64_t* gaps = c.i_gaps.reserve(3ULL * kMaxLongGaps);
  const unsigned grid = std::min<unsigned>(CeilDiv(n_a + 1, kThreads), c.sms * 8);
  if (is32) {
    IndexTableKernel<uint32_t, true><<<grid, kThreads, 0, c.stream>>>(
        reinterpret_cast<const uint32_t*>(kv), n_a, shift, n_buckets, bucket,
        reinterpret_cast<unsigned long long*>(hist), gaps);
    if (tiered && n_b > 0) {  // multiplicities of the keys beyond the limit
      if (bare) {
        BareCount(c, sorted_b, n_b, key_bits, limit32, bstart,
                  reinterpret_cast<unsigned long long*>(hist));
        --c.launches;  // (counted by BareCount)
      } else if (c.t_b_low) {
        GroupCountKernel<<<std::min<unsigned>(CeilDiv(n_b, kGroupChunk * (kThreads / 32)), c.sms * 6),
                           kThreads, 0, c.stream>>>(sorted_b, n_b,
                                                    reinterpret_cast<unsigned long long*>(hist));
      } else {
        IndexTableKernel<uint32_t, false>
            <<<std::min<unsigned>(CeilDiv(n_b + 1, kThreads), c.sms * 8), kThreads, 0, c.stream>>>(
                sorted_b, n_b, 0, 0, nullptr, reinterpret_cast<unsigned long long*>(hist), nullptr);
      }
      ++c.launches;
    }
  } else {
    IndexTableKernel<uint64_t, true><<<grid, kThreads, 0, c.stream>>>(
        kv, n_a, shift, n_buckets, bucket, reinterpret_cast<unsigned long long*>(hist), gaps);
  }
  RVN_LAUNCH_CHECK();
  ++c.launches;
  uint64_t* hk = c.pin64.reserve(8);
  RVN_CUDA(cudaMemcpyAsync(hk, hist + kHistBins, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                           c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  c.i_keys = hk[0];
  const uint64_t n_long = std::min<uint64_t>(hk[1], kMaxLongGaps);
  if (n_long) {
    FillLongGaps<<<static_cast<unsigned>(n_long), kThreads, 0, c.stream>>>(gaps, bucket);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  TimerEnd(c);

  c.stats.index_bases = index_bases;
  c.stats.index_records = n;
  c.stats.index_keys = c.i_keys;
  c.i_valid = true;
}

}  // namespace

uint64_t ReadBases(const Ctx& c, uint32_t first, uint32_t last) {
  uint64_t bases = 0;
  for (uint32_t r = first; r < last; ++r) bases += c.h_len[r];
  return bases;
}

std::vector<uint32_t> ChunkCuts(const Ctx& c, uint32_t first, uint32_t last, uint64_t chunk) {
  std::vector<uint32_t> cuts{first};
  uint64_t bases = 0;
  for (uint32_t r = first; r < last; ++r) {
    bases += c.h_len[r];
    if (r + 1 != last && bases < chunk) continue;
    bases = 0;
    cuts.push_back(r + 1);
  }
  if (cuts.back() != last) cuts.push_back(last);
  return cuts;
}

uint64_t BuildIndexChunked(Ctx& c, uint32_t first, uint32_t last, bool minhash, uint64_t chunk,
                           uint64_t tmax, bool tiers) {
  c.i_valid = false;
  c.occurrence = 0xFFFFFFFFu;
  CheckResident(c, first, last);
  // (an asynchronous upload: every chunk's bases are there before the first sketch)
  WaitUpload(c);
  const std::vector<uint32_t> cuts = ChunkCuts(c, first, last, chunk);
  // staged bases: each sketch is followed by the copy of the range sketched next - the next
  // chunk, after sweep 1 the first chunk again, after the last the range the caller named
  const uint32_t after_first = c.bases.next_first, after_last = c.bases.next_last;
  auto stage_next = [&](size_t i, bool sweep1) {
    if (i + 2 < cuts.size()) {
      BasesNext(c, cuts[i + 1], cuts[i + 2]);
    } else if (sweep1) {
      BasesNext(c, cuts[0], cuts[1]);
    } else {
      BasesNext(c, after_first, after_last);
    }
  };
  const uint32_t nr = last - first;
  const bool k32 = 2 * c.prm.k <= 30;
  const int key_bits = static_cast<int>(2 * c.prm.k);
  const int hist_shift = std::max(0, key_bits - kCapBits);
  unsigned long long* vhist = reinterpret_cast<unsigned long long*>(c.t_hist.reserve(kCapBins));
  RVN_CUDA(cudaMemsetAsync(vhist, 0, kCapBins * sizeof(uint64_t), c.stream));

  const uint64_t bases = ReadBases(c, first, last);
  if (minhash) {
    // one sweep: each chunk's micromizers are appended to the sort's second buffers,
    // sized by the len / k micromizers a read has at most
    uint64_t cap = 0;
    for (uint32_t r = first; r < last; ++r) cap += c.h_len[r] / c.prm.k;
    const size_t vb = k32 ? 4 : 8;
    uint64_t* q_val = c.i_val_alt.reserve(k32 ? cap / 2 + 2 : cap + 1);
    uint64_t* q_org = c.i_org_alt.reserve(cap + 1);
    uint64_t n = 0;
    for (size_t i = 0; i + 1 < cuts.size(); ++i) {
      stage_next(i, false);
      EnsureMicromizers(c, cuts[i], cuts[i + 1]);  // (sketches the chunk)
      TimerBegin(c, "sketch_tiers");
      if (c.mm.n) {
        RVN_CUDA(cudaMemcpyAsync(reinterpret_cast<uint8_t*>(q_val) + n * vb, c.mm.val.get(),
                                 c.mm.n * vb, cudaMemcpyDeviceToDevice, c.stream));
        RVN_CUDA(cudaMemcpyAsync(q_org + n, c.mm.org.get(), c.mm.n * sizeof(uint64_t),
                                 cudaMemcpyDeviceToDevice, c.stream));
      }
      TimerEnd(c);
      n += c.mm.n;
    }
    if (n >= 0xFFFFFFFFULL) throw LimitError("index batch holds 2^32 or more minimizers");
    c.i_first = first;
    c.i_last = last;
    BuildIndexImpl(c, ValView{q_val, k32 ? 1 : 0}, q_org, n, bases, ~0ULL, /*count_bare=*/true, 0);
    c.i_sorted_ids = c.ids_ascending;
    c.i_from_sketch = false;
    return tmax;
  }

  // ---- sweep 1: per chunk its sketch, its thresholds and micromizer counts (the
  // self-join's, for the whole batch), the record count and the coarse value histogram
  // that bounds the tiers ----
  uint64_t n = 0;
  std::vector<uint64_t> chunk_first{0};  // records before every chunk
  c.jt.Reset(first, nr);
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    const uint32_t r0 = cuts[i], r1 = cuts[i + 1];
    stage_next(i, true);
    EnsureSketch(c, r0, r1);  // (exactly the chunk: c.sk holds its records)
    EnsureThresholds(c, r0, r1);
    n += c.sk.n;
    chunk_first.push_back(n);
    c.jt.Append(c.qt, c.stream);
    if (tiers && k32 && c.sk.n > 0) {
      ValueHistKernel<<<std::min<unsigned>(CeilDiv(c.sk.n, kThreads), c.sms * 4), kThreads, 0,
                        c.stream>>>(reinterpret_cast<const uint32_t*>(c.sk.val.get()), c.sk.n,
                                    hist_shift, vhist);
      RVN_LAUNCH_CHECK();
      ++c.launches;
    }
  }
  if (n >= 0xFFFFFFFFULL) throw LimitError("index batch holds 2^32 or more minimizers");
  // the tier bound: the largest micromizer value of every read sketched so far
  if (tiers && nr > 0) tmax = k32 ? std::max(tmax, MaxThreshold(c, c.jt)) : ~0ULL;
  const uint64_t limit = tiers ? tmax : ~0ULL;
  const bool is32 = k32;
  const bool tiered = Tiered(c, is32, limit, n);
  // raven's stage-1 parameters: sweep 2 sketches straight into the tiers, or untiered into
  // the sort's second buffers, and the last chunk's sketch is not needed any more
  const bool fused = tiered && SketchTiersFused(c);
  const bool append = !tiered && SketchTiersFused(c);
  if (fused || append) {
    MarkStale(c, Stale::kRecords);
    c.sk.val.release();
    c.sk.org.release();
  }

  // ---- sweep 2: the chunks' records, appended in (read, position) order ----
  uint64_t n_a_cap = n, n_b_cap = 0;
  if (tiered) {  // tier capacities from the histogram (the bin of the limit counts in both)
    std::vector<uint64_t> h(kCapBins);
    RVN_CUDA(cudaMemcpyAsync(h.data(), vhist, kCapBins * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    const uint64_t lb = limit >> hist_shift;
    n_a_cap = 0;
    for (uint64_t b = 0; b < kCapBins; ++b) {
      if (b <= lb) n_a_cap += h[b];
      if (b >= lb) n_b_cap += h[b];
    }
  }
  const uint64_t val_elems = is32 ? n_a_cap / 2 + 2 : n_a_cap + 1;
  uint64_t* a_val = c.i_val_alt.reserve(val_elems);
  uint64_t* a_org = c.i_org_alt.reserve(n_a_cap + 1);
  uint32_t* b_val = tiered ? reinterpret_cast<uint32_t*>(c.t_b0.reserve(n_b_cap / 2 + 2)) : nullptr;
  const uint32_t limit32 = static_cast<uint32_t>(limit);
  uint64_t n_a = 0, n_b = 0;
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    const uint32_t r0 = cuts[i], r1 = cuts[i + 1];
    stage_next(i, false);
    if (fused) {
      TimerBegin(c, "sketch_tiers");
      uint64_t m_a = 0, m_b = 0;
      SketchTiers(c, r0, r1, limit32, reinterpret_cast<uint32_t*>(a_val) + n_a, a_org + n_a,
                  n_a_cap - n_a, b_val + n_b, n_b_cap - n_b, &m_a, &m_b);
      // (the capacities are the histogram's bound: never exceeded)
      if (n_a + m_a > n_a_cap || n_b + m_b > n_b_cap) {
        throw CudaError("chunked index build: tier capacity below the histogram's bound");
      }
      n_a += m_a;
      n_b += m_b;
      TimerEnd(c);
      continue;
    }
    if (append) {
      TimerBegin(c, "sketch_tiers");
      SketchAppend(c, r0, r1, reinterpret_cast<uint32_t*>(a_val), a_org, chunk_first[i], n);
      TimerEnd(c);
      continue;
    }
    EnsureSketch(c, r0, r1);  // (no-op for a batch of one chunk)
    const uint64_t* sv = c.sk.val.get();
    const uint64_t* so = c.sk.org.get();
    const uint64_t m = c.sk.n;
    TimerBegin(c, "sketch_tiers");
    if (m == 0) {
    } else if (tiered) {
      const uint32_t* sv32 = reinterpret_cast<const uint32_t*>(sv);
      const uint64_t tiles = (m + kTierTile - 1) / kTierTile;
      uint32_t* tcnt = c.t_cnt.reserve(tiles + 1);
      uint64_t* toff = c.t_off.reserve(tiles + 2);
      TierCountKernel<<<static_cast<unsigned>(tiles), kThreads, 0, c.stream>>>(sv32, m, limit32,
                                                                            tcnt);
      ExclusiveScanU32(c, tcnt, toff, tiles);
      const uint64_t m_a = ReadU64(c, toff + tiles);
      if (n_a + m_a > n_a_cap || n_b + (m - m_a) > n_b_cap) {
        throw CudaError("chunked index build: tier capacity below the histogram's bound");
      }
      TierScatterKernel<<<static_cast<unsigned>(tiles), kThreads, 0, c.stream>>>(
          sv32, so, m, limit32, toff, reinterpret_cast<uint32_t*>(a_val) + n_a, a_org + n_a,
          b_val + n_b);
      RVN_LAUNCH_CHECK();
      c.launches += 2;
      n_a += m_a;
      n_b += m - m_a;
    } else {
      const size_t vb = is32 ? 4 : 8;
      RVN_CUDA(cudaMemcpyAsync(reinterpret_cast<uint8_t*>(a_val) + n_a * vb, sv, m * vb,
                               cudaMemcpyDeviceToDevice, c.stream));
      RVN_CUDA(cudaMemcpyAsync(a_org + n_a, so, m * sizeof(uint64_t), cudaMemcpyDeviceToDevice,
                               c.stream));
      n_a += m;
    }
    TimerEnd(c);
  }
  // (sweep 1 counted the same records: the stream ends where its capacity does)
  if (append && nr > 0 && SketchAppendTotal(c) != n) {
    throw CudaError("chunked index build: the sweeps disagree on the batch's records");
  }
  c.i_first = first;
  c.i_last = last;
  BuildIndexImpl(c, ValView{a_val, is32 ? 1 : 0}, a_org, n, bases, limit, /*count_bare=*/true,
                 tiered ? static_cast<int64_t>(n_a) : 0);
  c.i_sorted_ids = c.ids_ascending;
  c.i_from_sketch = true;
  c.jt_gen = c.i_gen;
  return tmax;
}

void ReleaseIndexBuild(Ctx& c) {
  c.sk.valid = false;
  c.sk.val.release();
  c.sk.org.release();
  c.i_val_alt.release();
  c.i_org_alt.release();
  c.t_aval.release();
  c.t_aorg.release();
  c.t_b0.release();
  c.t_b1.release();
  c.t_b2.release();
  c.t_bstart.release();
  c.t_sorted_b = nullptr;  // (t_nb stays: FilterIndex refuses what would need the keys)
}

uint64_t* IndexHistogram(Ctx& c) {  // filled by the build
  return c.i_hist.get();
}

// same arithmetic as the reference engine: index = (1 - f) * #keys, truncated
// towards zero; the value at that ascending rank, plus one
uint32_t ThresholdFromHistogram(Ctx& c, const uint64_t* h, uint64_t n_keys,
                                double frequency, bool* needs_long_runs) {
  (void)c;
  *needs_long_runs = false;
  std::size_t rank = static_cast<std::size_t>((1 - frequency) * static_cast<double>(n_keys));
  if (rank >= n_keys) rank = n_keys - 1;
  uint64_t cum = 0;
  for (uint32_t len = 0; len + 1 < kHistBins; ++len) {
    cum += h[len];
    if (cum > rank) return len + 1;
  }
  *needs_long_runs = true;  // the rank falls among runs of >= 65535 postings
  return 0;
}

// occurrence_ = (run length at ascending rank (1-f)*#keys) + 1
uint32_t FilterIndex(Ctx& c, double frequency) {
  if (!(0 <= frequency && frequency <= 1)) {
    throw InvalidArgument(
        "[ram::MinimizerEngine::Filter] error: invalid frequency");
  }
  if (!c.i_valid) throw StateError("Filter before Minimize");
  if (frequency == 0 || c.i_keys == 0) {
    c.occurrence = 0xFFFFFFFFu;
    return c.occurrence;
  }
  uint64_t* hist = IndexHistogram(c);  // (filled by the index table pass)
  std::vector<uint64_t> h(kHistBins);
  RVN_CUDA(cudaMemcpyAsync(h.data(), hist, kHistBins * sizeof(uint64_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  bool long_runs = false;
  uint32_t occ = ThresholdFromHistogram(c, h.data(), c.i_keys, frequency, &long_runs);
  if (long_runs) {
    uint64_t cum = 0;
    for (uint32_t len = 0; len + 1 < kHistBins; ++len) cum += h[len];
    std::size_t rank = static_cast<std::size_t>((1 - frequency) * static_cast<double>(c.i_keys));
    if (rank >= c.i_keys) rank = c.i_keys - 1;
    if (c.i_is32 && c.t_nb && !c.t_sorted_b) {
      throw StateError(
          "the bare keys of this chunked index build were freed: runs of 65535 or more "
          "postings need them, build the index again to filter at this frequency");
    }
    const uint64_t n_long = h[kHistBins - 1];
    uint32_t* out = c.m_cnt.reserve(n_long + 1);
    uint64_t* counter = c.m_counter.reserve(8);
    RVN_CUDA(cudaMemsetAsync(counter, 0, sizeof(uint64_t), c.stream));
    if (c.i_is32) {
      CollectLongRuns<uint32_t><<<CeilDiv(c.i_n, kThreads), kThreads, 0, c.stream>>>(
          reinterpret_cast<const uint32_t*>(c.i_val.get()), c.i_n,
          reinterpret_cast<unsigned long long*>(counter), out);
      if (c.t_sorted_b && c.t_nb && !c.t_b_sorted) {  // (runs of >= 65535: sort the bare keys)
        // a full key sort is right from any order; the source buffer doubles as the
        // sort's second buffer (it is dead after the first pass)
        uint32_t* bufs[3] = {reinterpret_cast<uint32_t*>(c.t_b0.get()),
                             reinterpret_cast<uint32_t*>(c.t_b1.get()),
                             reinterpret_cast<uint32_t*>(c.t_b2.get())};
        uint32_t* src = nullptr;
        for (uint32_t* p : bufs) {
          if (p == c.t_sorted_b) src = p;
        }
        uint32_t* other = src == bufs[0] ? bufs[1] : bufs[0];
        const int where = RadixSortKeys(c, src, other, src, c.t_nb, 0,
                                        static_cast<int>(2 * c.prm.k));
        c.t_sorted_b = where == 0 ? other : src;
        c.t_b_low = 0;
        c.t_b_sorted = true;
      }
      if (c.t_sorted_b && c.t_nb) {  // tiered build: the keys beyond the limit too
        CollectLongRuns<uint32_t><<<CeilDiv(c.t_nb, kThreads), kThreads, 0, c.stream>>>(
            c.t_sorted_b, c.t_nb, reinterpret_cast<unsigned long long*>(counter), out);
      }
    } else {
      CollectLongRuns<uint64_t><<<CeilDiv(c.i_n, kThreads), kThreads, 0, c.stream>>>(
          c.i_val.get(), c.i_n, reinterpret_cast<unsigned long long*>(counter), out);
    }
    RVN_LAUNCH_CHECK();
    ++c.launches;
    std::vector<uint32_t> lens(n_long);
    RVN_CUDA(cudaMemcpyAsync(lens.data(), out, n_long * sizeof(uint32_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    std::sort(lens.begin(), lens.end());
    occ = lens[rank - cum] + 1;
  }
  c.occurrence = occ;
  c.stats.occurrence = c.occurrence;
  return c.occurrence;
}

}  // namespace rvn
