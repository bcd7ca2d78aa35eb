// raven_b200 — stable LSD radix sort for sm_90a, written for this engine
// ("onesweep": one pass over the data per digit, chained-scan of the tiles).
//
// Used for the minimizer index (ram::MinimizerEngine::Minimize, call site
// RavenLib/src/construct.cc:42-43: all (value, origin) records of an index batch
// ordered by value, equal values in (read, position) order = STABLE), for the
// value order of the query probes, the size order of the chain pairs and the
// emission order of the overlaps (map.cu) and the rhs order of the gather
// (gather.cu).
//
// Layout of one pass (digit = up to 10 bits, 1024 bins):
//   * an upfront kernel histograms the digits of ALL passes in one read of the
//     keys (global exclusive bin offsets per pass);
//   * OnesweepPass: a CTA of 256 threads takes the next tile of 8192 keys
//     (ticket), every warp ranks its 1024 consecutive keys 32 at a time
//     (__match_any_sync on the digit + a per-warp shared-memory counter: ranks
//     follow the input order, so the sort is stable), the per-bin counts of the
//     tile are chained to the tiles before it by decoupled look-back (one status
//     word per (tile, bin): aggregate or inclusive prefix), keys and payloads go
//     through shared memory so that every bin's run leaves the SM as one
//     contiguous, coalesced store.
// Per pass and record: one read + one write of key and payload (HBM bound);
// 30-bit minimizer values (k = 15) take three passes, values arrive as u32 from
// the sketch kernel (no narrowing / widening copies).
#include <algorithm>

#include "engine.cuh"

namespace rvn {

namespace {

constexpr int kRadixMaxBits = 10;
constexpr int kBins = 1 << kRadixMaxBits;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kBinsPerThread = kBins / kThreads; // 4
constexpr int kMaxPasses = 8;
// keys per thread: 32 for 4-byte keys (tile of 8192), 16 for 8-byte keys (4096):
// keys, staging slots and destinations of a tile live in registers
template <typename KeyT>
struct Items {
  static constexpr int value = sizeof(KeyT) == 4 ? 32 : 16;
};

// status word of (tile, bin): flag in the top two bits, count below
constexpr uint32_t kFlagAggregate = 1u << 30;
constexpr uint32_t kFlagPrefix = 2u << 30;
constexpr uint32_t kFlagMask = 3u << 30;
constexpr uint32_t kValueMask = ~kFlagMask;

struct PassPlan {
  int n_passes;
  int begin[kMaxPasses];
  int bits[kMaxPasses];
};

template <typename KeyT>
__device__ __forceinline__ uint32_t Digit(KeyT key, KeyT flip, int begin, uint32_t mask) {
  return static_cast<uint32_t>((key ^ flip) >> begin) & mask;
}

// histograms of the digits of every pass: hist[pass * kBins + digit]
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
RadixHistogramKernel(const KeyT* __restrict__ keys, uint64_t n, PassPlan plan, KeyT flip,
                     unsigned long long* __restrict__ hist) {
  extern __shared__ uint32_t sh_hist[];  // n_passes * kBins
  const int total = plan.n_passes * kBins;
  for (int i = threadIdx.x; i < total; i += kThreads) sh_hist[i] = 0;
  __syncthreads();
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kThreads;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x; i < n;
       i += stride) {
    const KeyT k = keys[i];
#pragma unroll
    for (int p = 0; p < kMaxPasses; ++p) {
      if (p < plan.n_passes) {
        atomicAdd(&sh_hist[p * kBins + Digit<KeyT>(k, flip, plan.begin[p],
                                                    (1u << plan.bits[p]) - 1u)], 1u);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < total; i += kThreads) {
    if (sh_hist[i]) atomicAdd(&hist[i], static_cast<unsigned long long>(sh_hist[i]));
  }
}

// exclusive scan over the bins of every pass (one CTA of kBins threads)
__global__ void __launch_bounds__(kBins)
RadixScanBinsKernel(const unsigned long long* __restrict__ hist, int n_passes,
                    uint32_t* __restrict__ bin_base) {
  __shared__ uint32_t sm[34];
  for (int p = 0; p < n_passes; ++p) {
    const uint32_t v = static_cast<uint32_t>(hist[p * kBins + threadIdx.x]);
    uint32_t total;
    const uint32_t ex = BlockExclusiveSum<uint32_t, kBins>(v, sm, &total);
    bin_base[p * kBins + threadIdx.x] = ex;
  }
}

// Decoupled look-back over the status words of one (tile, bin) grid: publishes the
// tile's counts of the thread's kBinsPerThread bins and returns in excl the counts
// of those bins in all tiles before it.
// A thread owns 4 neighbouring bins = ONE 16-byte status word per tile: all four
// aggregates are published in one store before any waiting, and one 16-byte load
// per step walks the four chains back together (a per-bin walk would put up to
// #resident-tiles dependent L2 round trips in series, four times over).
__device__ __forceinline__ void ChainTileCounts(uint32_t* __restrict__ status, uint32_t tile,
                                                const uint32_t (&cnt)[kBinsPerThread],
                                                uint32_t (&excl)[kBinsPerThread]) {
  uint4* st4 = reinterpret_cast<uint4*>(status);
  const uint64_t my4 = static_cast<uint64_t>(tile) * (kBins / 4) + threadIdx.x;
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) excl[j] = 0;
  static_assert(kBinsPerThread == 4, "one uint4 of status words per thread");
  if (tile > 0) {
    uint4 agg;
    agg.x = kFlagAggregate | cnt[0];
    agg.y = kFlagAggregate | cnt[1];
    agg.z = kFlagAggregate | cnt[2];
    agg.w = kFlagAggregate | cnt[3];
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(st4 + my4),
                 "r"(agg.x), "r"(agg.y), "r"(agg.z), "r"(agg.w)
                 : "memory");
    // kLook predecessors per round, their loads in flight together: one
    // dependent L2 round trip per tile would make the walk slower than the rate
    // at which tiles start, and the chain would grow to every tile in flight
    constexpr int kLook = 4;
    uint32_t open = 0xF;  // chains still walking
    int64_t p = static_cast<int64_t>(tile) - 1;
    while (open) {
      uint4 v[kLook];
#pragma unroll
      for (int u = 0; u < kLook; ++u) {
        const int64_t q = p - u;
        if (q >= 0) {
          const uint4* src = st4 + static_cast<uint64_t>(q) * (kBins / 4) + threadIdx.x;
          asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w)
                       : "l"(src)
                       : "memory");
        } else {  // before tile 0: empty prefixes
          v[u] = make_uint4(kFlagPrefix, kFlagPrefix, kFlagPrefix, kFlagPrefix);
        }
      }
      int used = 0;
#pragma unroll
      for (int u = 0; u < kLook; ++u) {
        const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
        const bool ready = (vv[0] & kFlagMask) && (vv[1] & kFlagMask) && (vv[2] & kFlagMask) &&
                           (vv[3] & kFlagMask);
        if (used == u && ready && open) {  // (in order; stop at the first unwritten tile)
#pragma unroll
          for (int j = 0; j < kBinsPerThread; ++j) {
            if (open & (1u << j)) {
              excl[j] += vv[j] & kValueMask;
              if ((vv[j] & kFlagMask) == kFlagPrefix) open &= ~(1u << j);
            }
          }
          used = u + 1;
        }
      }
      p -= used;  // (used == 0: the nearest tile has not published yet - poll again)
    }
  }
  uint4 pre;
  pre.x = kFlagPrefix | (excl[0] + cnt[0]);
  pre.y = kFlagPrefix | (excl[1] + cnt[1]);
  pre.z = kFlagPrefix | (excl[2] + cnt[2]);
  pre.w = kFlagPrefix | (excl[3] + cnt[3]);
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(st4 + my4), "r"(pre.x),
               "r"(pre.y), "r"(pre.z), "r"(pre.w)
               : "memory");
}

template <typename KeyT, typename ValT, bool HAS_VAL>
struct __align__(16) PassSmem {
  static constexpr int kTile = kThreads * Items<KeyT>::value;
  uint16_t warp_hist[kWarps][kBins];  // per-warp digit counts, later exclusive over warps
  uint32_t bin_off[kBins];            // first staging slot of the bin inside the tile
  uint32_t bin_dst[kBins];            // global index of staging slot s of bin d = bin_dst[d] + s
  uint32_t scan[34];
  uint32_t tile;
  uint16_t slot_digit[HAS_VAL ? kTile : 2];  // digit of the element staged at a slot
  union {
    KeyT keys[kTile];
    ValT vals[HAS_VAL ? kTile : 1];
  } stage;
};

template <typename KeyT, typename ValT, bool HAS_VAL>
__global__ void __launch_bounds__(kThreads, 2)
OnesweepPass(const KeyT* __restrict__ keys_in, KeyT* __restrict__ keys_out,
             const ValT* __restrict__ vals_in, ValT* __restrict__ vals_out, uint32_t n,
             KeyT flip, int begin_bit, int pass_bits, const uint32_t* __restrict__ bin_base,
             uint32_t* __restrict__ bin_next, uint32_t* __restrict__ status,
             unsigned int* __restrict__ ticket) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using Smem = PassSmem<KeyT, ValT, HAS_VAL>;
  constexpr int kItems = Items<KeyT>::value;
  constexpr int kTile = kThreads * kItems;
  constexpr int kWarpTile = 32 * kItems;
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lanemask_lt = (1u << lane) - 1u;
  const uint32_t dmask = (1u << pass_bits) - 1u;

  if (threadIdx.x == 0) sm.tile = atomicAdd(ticket, 1u);
  {  // zero the per-warp histograms (kWarps * kBins u16 = 4096 u32 words)
    uint32_t* w = reinterpret_cast<uint32_t*>(&sm.warp_hist[0][0]);
#pragma unroll
    for (int i = 0; i < kWarps * kBins / 2 / kThreads; ++i) w[i * kThreads + threadIdx.x] = 0;
  }
  __syncthreads();
  const uint32_t tile = sm.tile;
  const uint64_t tile_base = static_cast<uint64_t>(tile) * kTile;
  const uint32_t tile_count =
      static_cast<uint32_t>(min(static_cast<uint64_t>(kTile), static_cast<uint64_t>(n) - tile_base));

  // ---- load: warp-striped, item i of lane l = key tile_base + warp*1024 + i*32 + l ----
  KeyT key[kItems];
  const uint32_t warp_base = warp * kWarpTile;
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    key[i] = t < tile_count ? keys_in[tile_base + t] : static_cast<KeyT>(0);
  }

  // first half of the payloads: in flight while the keys are ranked
  constexpr int kHalf = kItems / 2;
  ValT early[HAS_VAL ? kHalf : 1];
  if (HAS_VAL) {
#pragma unroll
    for (int i = 0; i < kHalf; ++i) {
      const uint32_t t = warp_base + i * 32 + lane;
      early[i] = t < tile_count ? vals_in[tile_base + t] : ValT(0);
    }
  }

  // ---- rank inside the warp, in input order ----
  uint16_t rank[kItems];
  uint16_t* my_hist = sm.warp_hist[warp];
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    const bool valid = t < tile_count;
    // lanes with the same digit: one ballot per digit bit (the hardware MATCH.ANY
    // is several times slower than ten votes); invalid lanes stand alone
    const uint32_t d = valid ? Digit<KeyT>(key[i], flip, begin_bit, dmask) : 0u;
    uint32_t peers = __ballot_sync(0xFFFFFFFFu, valid);
#pragma unroll
    for (int bit = 0; bit < kRadixMaxBits; ++bit) {
      const bool one = (d >> bit) & 1u;
      const uint32_t vote = __ballot_sync(0xFFFFFFFFu, one);
      peers &= one ? vote : ~vote;
    }
    if (!valid) peers = 1u << lane;
    const uint32_t leader = __ffs(peers) - 1;
    uint32_t before = 0;
    if (lane == leader && valid) {
      before = my_hist[d];
      my_hist[d] = static_cast<uint16_t>(before + __popc(peers));
    }
    before = __shfl_sync(0xFFFFFFFFu, before, leader);
    rank[i] = static_cast<uint16_t>(before + __popc(peers & lanemask_lt));
    __syncwarp();  // the counter update is visible to the next step's leader
  }
  __syncthreads();

  // ---- per bin: exclusive over the warps, tile count, tile-exclusive offsets ----
  uint32_t cnt[kBinsPerThread];
  uint32_t mine = 0;
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) {
    const uint32_t b = threadIdx.x * kBinsPerThread + j;
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const uint32_t x = sm.warp_hist[w][b];
      sm.warp_hist[w][b] = static_cast<uint16_t>(c);
      c += x;
    }
    cnt[j] = c;
    mine += c;
  }
  uint32_t total;
  uint32_t ex = BlockExclusiveSum<uint32_t, kThreads>(mine, sm.scan, &total);
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) {
    sm.bin_off[threadIdx.x * kBinsPerThread + j] = ex;
    ex += cnt[j];
  }

  // ---- chain the tile's bin counts to the tiles before it (decoupled look-back) ----
  {
    uint32_t excl[kBinsPerThread];
    ChainTileCounts(status, tile, cnt, excl);
#pragma unroll
    for (int j = 0; j < kBinsPerThread; ++j) {
      const uint32_t b = threadIdx.x * kBinsPerThread + j;
      const uint32_t base = bin_base[b];  // (bins beyond the digit range: zero counts)
      sm.bin_dst[b] = base + excl[j] - sm.bin_off[b];
      // the last tile leaves the running end of every bin for the next portion
      if (tile == gridDim.x - 1) bin_next[b] = base + excl[j] + cnt[j];
    }
  }
  __syncthreads();

  // ---- staging slot of every item (kept packed in the rank registers) ----
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    if (t < tile_count) {
      const uint32_t d = Digit<KeyT>(key[i], flip, begin_bit, dmask);
      const uint32_t slot = sm.bin_off[d] + sm.warp_hist[warp][d] + rank[i];
      rank[i] = static_cast<uint16_t>(slot);
      if (HAS_VAL) sm.slot_digit[slot] = static_cast<uint16_t>(d);
    }
  }

  // ---- payloads first (the keys wait in registers): global -> staging slot,
  // then out in bin order. The first half was loaded before the ranking, the
  // second half goes out as one batch of independent loads. ----
  if (HAS_VAL) {
    ValT late[kHalf];
#pragma unroll
    for (int i = 0; i < kHalf; ++i) {
      const uint32_t t = warp_base + (kHalf + i) * 32 + lane;
      late[i] = t < tile_count ? vals_in[tile_base + t] : ValT(0);
    }
#pragma unroll
    for (int i = 0; i < kHalf; ++i) {
      const uint32_t t = warp_base + i * 32 + lane;
      if (t < tile_count) sm.stage.vals[rank[i]] = early[i];
    }
#pragma unroll
    for (int i = 0; i < kHalf; ++i) {
      const uint32_t t = warp_base + (kHalf + i) * 32 + lane;
      if (t < tile_count) sm.stage.vals[rank[kHalf + i]] = late[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
      const uint32_t s = i * kThreads + threadIdx.x;
      if (s < tile_count) vals_out[sm.bin_dst[sm.slot_digit[s]] + s] = sm.stage.vals[s];
    }
    __syncthreads();  // every payload has left the staging buffer
  }

  // ---- keys: the same two hops ----
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    if (t < tile_count) sm.stage.keys[rank[i]] = key[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t s = i * kThreads + threadIdx.x;
    if (s < tile_count) {
      const KeyT k = sm.stage.keys[s];
      keys_out[sm.bin_dst[Digit<KeyT>(k, flip, begin_bit, dmask)] + s] = k;
    }
  }
}

// One UNSTABLE key-only pass over a digit of up to kRadixMaxBits bits: same tiles,
// look-back and staging as OnesweepPass<u32, u32, false>, but every key takes its
// slot with one shared-memory atomicAdd on the tile's bin counter instead of the
// warp's ten ballots. Keys of a bin land in any order inside their tile's share of
// the bin; for callers that need only the multiset of every bin.
struct PartitionSmem {
  uint32_t bin_cnt[kBins];  // keys of the tile per bin
  uint32_t bin_off[kBins];  // first staging slot of the bin inside the tile
  uint32_t bin_dst[kBins];  // global index of staging slot s of bin d = bin_dst[d] + s
  uint32_t scan[34];
  uint32_t tile;
  uint32_t keys[kThreads * Items<uint32_t>::value];
};

__global__ void __launch_bounds__(kThreads, 2)
PartitionPass(const uint32_t* __restrict__ keys_in, uint32_t* __restrict__ keys_out, uint32_t n,
              int begin_bit, int pass_bits, const uint32_t* __restrict__ bin_base,
              uint32_t* __restrict__ bin_next, uint32_t* __restrict__ status,
              unsigned int* __restrict__ ticket) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PartitionSmem& sm = *reinterpret_cast<PartitionSmem*>(smem_raw);
  constexpr int kItems = Items<uint32_t>::value;
  constexpr int kTile = kThreads * kItems;
  constexpr int kWarpTile = 32 * kItems;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t dmask = (1u << pass_bits) - 1u;

  if (threadIdx.x == 0) sm.tile = atomicAdd(ticket, 1u);
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) sm.bin_cnt[j * kThreads + threadIdx.x] = 0;
  __syncthreads();
  const uint32_t tile = sm.tile;
  const uint64_t tile_base = static_cast<uint64_t>(tile) * kTile;
  const uint32_t tile_count =
      static_cast<uint32_t>(min(static_cast<uint64_t>(kTile), static_cast<uint64_t>(n) - tile_base));

  uint32_t key[kItems];
  const uint32_t warp_base = warp * kWarpTile;
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    key[i] = t < tile_count ? keys_in[tile_base + t] : 0u;
  }
  // rank inside the tile's bin: the counter's value before this key's increment
  uint16_t rank[kItems];
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    if (t < tile_count) {
      rank[i] = static_cast<uint16_t>(atomicAdd(&sm.bin_cnt[(key[i] >> begin_bit) & dmask], 1u));
    }
  }
  __syncthreads();

  uint32_t cnt[kBinsPerThread];
  uint32_t mine = 0;
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) {
    cnt[j] = sm.bin_cnt[threadIdx.x * kBinsPerThread + j];
    mine += cnt[j];
  }
  uint32_t total;
  uint32_t ex = BlockExclusiveSum<uint32_t, kThreads>(mine, sm.scan, &total);
#pragma unroll
  for (int j = 0; j < kBinsPerThread; ++j) {
    sm.bin_off[threadIdx.x * kBinsPerThread + j] = ex;
    ex += cnt[j];
  }
  {
    uint32_t excl[kBinsPerThread];
    ChainTileCounts(status, tile, cnt, excl);
#pragma unroll
    for (int j = 0; j < kBinsPerThread; ++j) {
      const uint32_t b = threadIdx.x * kBinsPerThread + j;
      const uint32_t base = bin_base[b];
      sm.bin_dst[b] = base + excl[j] - sm.bin_off[b];
      if (tile == gridDim.x - 1) bin_next[b] = base + excl[j] + cnt[j];
    }
  }
  __syncthreads();

  // staging in bin order, then every bin's run leaves the SM as one coalesced store
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t t = warp_base + i * 32 + lane;
    if (t < tile_count) sm.keys[sm.bin_off[(key[i] >> begin_bit) & dmask] + rank[i]] = key[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const uint32_t s = i * kThreads + threadIdx.x;
    if (s < tile_count) {
      const uint32_t k = sm.keys[s];
      keys_out[sm.bin_dst[(k >> begin_bit) & dmask] + s] = k;
    }
  }
}

PassPlan MakePlan(int begin_bit, int end_bit) {
  PassPlan plan{};
  const int total = std::max(0, end_bit - begin_bit);
  const int np = (total + kRadixMaxBits - 1) / kRadixMaxBits;
  if (np > kMaxPasses) throw InvalidArgument("radix sort: too many key bits");
  plan.n_passes = np;
  int at = begin_bit;
  for (int p = 0; p < np; ++p) {
    // spread the bits evenly over the passes (30 -> 10,10,10; 16 -> 8,8)
    const int b = (total - (at - begin_bit) + (np - p) - 1) / (np - p);
    plan.begin[p] = at;
    plan.bits[p] = b;
    at += b;
  }
  return plan;
}

template <typename KeyT, typename ValT, bool HAS_VAL>
int SortImpl(Ctx& c, const KeyT* src_keys, KeyT* keys_a, KeyT* keys_b, const ValT* src_vals,
             ValT* vals_a, ValT* vals_b, uint64_t n, int begin_bit, int end_bit,
             bool descending) {
  if (n >= 0xFFFFFFFFULL) throw LimitError("radix sort of 2^32 or more records");
  const PassPlan plan = MakePlan(begin_bit, end_bit);
  if (plan.n_passes == 0 || n == 0) return -1;  // nothing moves: the source is the result
  using Smem = PassSmem<KeyT, ValT, HAS_VAL>;
  constexpr uint64_t kTile = Smem::kTile;
  const KeyT flip = descending ? static_cast<KeyT>(~static_cast<KeyT>(0)) : static_cast<KeyT>(0);
  // a status word counts below 2^30: longer inputs go portion by portion, the
  // last tile of a portion hands the running bin ends to the next one
  const uint64_t portion = ((1ULL << 30) - 1) / kTile * kTile;
  const uint64_t n_portions = (n + portion - 1) / portion;
  const uint64_t max_tiles = (std::min(n, portion) + kTile - 1) / kTile;
  // scratch: [hist: passes*kBins u64][bin bases: 2 x passes*kBins u32][tickets][status]
  const size_t hist_bytes = sizeof(uint64_t) * plan.n_passes * kBins;
  const size_t base_bytes = sizeof(uint32_t) * plan.n_passes * kBins;
  const size_t ticket_bytes = sizeof(unsigned int) * kMaxPasses * 8;
  if (plan.n_passes * n_portions > kMaxPasses * 8) throw LimitError("radix sort: too many launches");
  const size_t status_bytes = sizeof(uint32_t) * max_tiles * kBins;
  const size_t head = hist_bytes + 2 * base_bytes + ticket_bytes;
  uint8_t* scratch = c.sort_tmp.reserve(head + status_bytes + 256);
  auto* hist = reinterpret_cast<unsigned long long*>(scratch);
  uint32_t* bases[2] = {reinterpret_cast<uint32_t*>(scratch + hist_bytes),
                        reinterpret_cast<uint32_t*>(scratch + hist_bytes + base_bytes)};
  auto* ticket = reinterpret_cast<unsigned int*>(scratch + hist_bytes + 2 * base_bytes);
  auto* status = reinterpret_cast<uint32_t*>(scratch + head);
  RVN_CUDA(cudaMemsetAsync(scratch, 0, head, c.stream));
  const unsigned hgrid =
      static_cast<unsigned>(std::min<uint64_t>((n + kThreads - 1) / kThreads, c.sms * 8));
  RadixHistogramKernel<KeyT><<<hgrid, kThreads, sizeof(uint32_t) * plan.n_passes * kBins,
                               c.stream>>>(src_keys, n, plan, flip, hist);
  RadixScanBinsKernel<<<1, kBins, 0, c.stream>>>(hist, plan.n_passes, bases[0]);
  RVN_LAUNCH_CHECK();
  c.launches += 2;

  auto kern = OnesweepPass<KeyT, ValT, HAS_VAL>;
  RVN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(Smem))));
  const KeyT* kin = src_keys;
  const ValT* vin = src_vals;
  int where = -1;
  unsigned launch = 0;
  for (int p = 0; p < plan.n_passes; ++p) {
    const int to = where == 0 ? 1 : 0;  // the first pass lands in buffer a
    KeyT* kout = to == 0 ? keys_a : keys_b;
    ValT* vout = to == 0 ? vals_a : vals_b;
    int cur = 0;  // bases[0] holds the scanned bin offsets of every pass
    for (uint64_t q = 0; q < n_portions; ++q) {
      const uint64_t first = q * portion;
      const uint64_t cnt = std::min(portion, n - first);
      const uint64_t tiles = (cnt + kTile - 1) / kTile;
      RVN_CUDA(cudaMemsetAsync(status, 0, sizeof(uint32_t) * tiles * kBins, c.stream));
      kern<<<static_cast<unsigned>(tiles), kThreads, sizeof(Smem), c.stream>>>(
          kin + first, kout, HAS_VAL ? vin + first : vin, vout, static_cast<uint32_t>(cnt), flip,
          plan.begin[p], plan.bits[p], bases[cur] + p * kBins, bases[cur ^ 1] + p * kBins, status,
          ticket + launch);
      RVN_LAUNCH_CHECK();
      ++c.launches;
      ++launch;
      cur ^= 1;
    }
    kin = kout;
    vin = vout;
    where = to;
  }
  return where;
}

}  // namespace

// Stable sort of (key, value) pairs on key bits [begin_bit, end_bit). The source
// arrays are only read; the result lands in buffer a (return 0) or b (return 1);
// -1: nothing to do (n == 0 or no bits), the source order is the result.
int RadixSortPairs(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b,
                   const uint64_t* src_vals, uint64_t* vals_a, uint64_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending) {
  return SortImpl<uint32_t, uint64_t, true>(c, src_keys, keys_a, keys_b, src_vals, vals_a, vals_b,
                                            n, begin_bit, end_bit, descending);
}
int RadixSortPairs(Ctx& c, const uint64_t* src_keys, uint64_t* keys_a, uint64_t* keys_b,
                   const uint64_t* src_vals, uint64_t* vals_a, uint64_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending) {
  return SortImpl<uint64_t, uint64_t, true>(c, src_keys, keys_a, keys_b, src_vals, vals_a, vals_b,
                                            n, begin_bit, end_bit, descending);
}
int RadixSortPairs(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b,
                   const uint32_t* src_vals, uint32_t* vals_a, uint32_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending) {
  return SortImpl<uint32_t, uint32_t, true>(c, src_keys, keys_a, keys_b, src_vals, vals_a, vals_b,
                                            n, begin_bit, end_bit, descending);
}
int RadixSortPairs(Ctx& c, const uint64_t* src_keys, uint64_t* keys_a, uint64_t* keys_b,
                   const uint32_t* src_vals, uint32_t* vals_a, uint32_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending) {
  return SortImpl<uint64_t, uint32_t, true>(c, src_keys, keys_a, keys_b, src_vals, vals_a, vals_b,
                                            n, begin_bit, end_bit, descending);
}
int RadixSortKeys(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b, uint64_t n,
                  int begin_bit, int end_bit) {
  return SortImpl<uint32_t, uint32_t, false>(c, src_keys, keys_a, keys_b, nullptr, nullptr, nullptr,
                                             n, begin_bit, end_bit, false);
}

// Unstable partition of u32 keys on their bits [begin_bit, end_bit) (at most 10):
// the keys of digit d land in dst[bin_start[d], bin_start[d + 1]) in no particular
// order (bin_start[d + 1] = n past the last digit). bin_start: 1024 entries, left on
// the device for the caller.
void RadixPartitionKeys(Ctx& c, const uint32_t* src, uint32_t* dst, uint64_t n, int begin_bit,
                        int end_bit, uint32_t* bin_start) {
  if (n >= 0xFFFFFFFFULL) throw LimitError("radix partition of 2^32 or more records");
  if (end_bit - begin_bit < 1 || end_bit - begin_bit > kRadixMaxBits) {
    throw InvalidArgument("radix partition: 1 to 10 key bits");
  }
  PassPlan plan{};
  plan.n_passes = 1;
  plan.begin[0] = begin_bit;
  plan.bits[0] = end_bit - begin_bit;
  constexpr uint64_t kTile = kThreads * Items<uint32_t>::value;
  // status words count below 2^30: portion by portion, as in SortImpl
  const uint64_t portion = ((1ULL << 30) - 1) / kTile * kTile;
  const uint64_t n_portions = (n + portion - 1) / portion;
  const uint64_t max_tiles = (std::min(n, portion) + kTile - 1) / kTile;
  const size_t hist_bytes = sizeof(uint64_t) * kBins;
  const size_t base_bytes = sizeof(uint32_t) * kBins;
  const size_t ticket_bytes = sizeof(unsigned int) * kMaxPasses * 8;
  if (n_portions > kMaxPasses * 8) throw LimitError("radix partition: too many launches");
  const size_t head = hist_bytes + 2 * base_bytes + ticket_bytes;
  const size_t status_bytes = sizeof(uint32_t) * max_tiles * kBins;
  uint8_t* scratch = c.sort_tmp.reserve(head + status_bytes + 256);
  auto* hist = reinterpret_cast<unsigned long long*>(scratch);
  uint32_t* bases[2] = {reinterpret_cast<uint32_t*>(scratch + hist_bytes),
                        reinterpret_cast<uint32_t*>(scratch + hist_bytes + base_bytes)};
  auto* ticket = reinterpret_cast<unsigned int*>(scratch + hist_bytes + 2 * base_bytes);
  auto* status = reinterpret_cast<uint32_t*>(scratch + head);
  RVN_CUDA(cudaMemsetAsync(scratch, 0, head, c.stream));
  if (n == 0) {
    RVN_CUDA(cudaMemsetAsync(bin_start, 0, base_bytes, c.stream));
    return;
  }
  const unsigned hgrid =
      static_cast<unsigned>(std::min<uint64_t>((n + kThreads - 1) / kThreads, c.sms * 8));
  RadixHistogramKernel<uint32_t><<<hgrid, kThreads, sizeof(uint32_t) * kBins, c.stream>>>(
      src, n, plan, 0u, hist);
  RadixScanBinsKernel<<<1, kBins, 0, c.stream>>>(hist, 1, bases[0]);
  RVN_LAUNCH_CHECK();
  c.launches += 2;
  // (bases[0] is overwritten from the third portion on)
  RVN_CUDA(cudaMemcpyAsync(bin_start, bases[0], base_bytes, cudaMemcpyDeviceToDevice, c.stream));
  RVN_CUDA(cudaFuncSetAttribute(PartitionPass, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(PartitionSmem))));
  int cur = 0;
  for (uint64_t q = 0; q < n_portions; ++q) {
    const uint64_t first = q * portion;
    const uint64_t cnt = std::min(portion, n - first);
    const uint64_t tiles = (cnt + kTile - 1) / kTile;
    RVN_CUDA(cudaMemsetAsync(status, 0, sizeof(uint32_t) * tiles * kBins, c.stream));
    PartitionPass<<<static_cast<unsigned>(tiles), kThreads, sizeof(PartitionSmem), c.stream>>>(
        src + first, dst, static_cast<uint32_t>(cnt), plan.begin[0], plan.bits[0], bases[cur],
        bases[cur ^ 1], status, ticket + q);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    cur ^= 1;
  }
}

}  // namespace rvn
