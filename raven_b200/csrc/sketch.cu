// raven_b200 — minimizer sketching on sm_90a.
//
// Replaces ram::MinimizerEngine::Minimize(sequence, minhash) (un-vendored;
// call sites RavenLib/src/construct.cc:42-43,62,363,377-381; algorithm
// SURVEY.md App. A.2). The reference walks each read with a rolling k-mer and
// a monotone deque. Here every k-mer position is independent:
//   * the 2k-bit k-mer is cut straight out of the 2-bit packed words (staged
//     in shared memory), the reverse complement is ~lo & mask and the forward
//     k-mer the 2-bit-group reversal of lo — no rolling state;
//   * position q is a minimizer iff its hash is <= every valid hash in at
//     least one of the w-wide windows that contain it, i.e. iff
//     left_run(q) + right_run(q) >= w - 1 where *_run counts consecutive
//     neighbours with hash >= hash(q) (capped at w-1 and at the read ends).
//     This is exactly the deque's "emit every tie of the window minimum
//     once" rule, and emission order equals position order (DESIGN.md).
// One CTA sketches kSketchTile positions of one read (+ w-1 halo each side).
// Pass 1 counts, a device scan places tiles, pass 2 writes (value, origin)
// records in (read, position) order — the order the index build relies on.
#include <algorithm>

#include "engine.cuh"

namespace rvn {

namespace {


__device__ __forceinline__ uint64_t MixHash(uint64_t key, uint64_t mask) {
  key = ((~key) + (key << 21)) & mask;
  key = key ^ (key >> 24);
  key = ((key + (key << 3)) + (key << 8)) & mask;
  key = key ^ (key >> 14);
  key = ((key + (key << 2)) + (key << 4)) & mask;
  key = key ^ (key >> 28);
  key = (key + (key << 31)) & mask;
  return key;
}

// reverse the order of the 32 two-bit groups of x
__device__ __forceinline__ uint64_t ReverseGroups(uint64_t x) {
  x = __brevll(x);
  return ((x >> 1) & 0x5555555555555555ULL) | ((x & 0x5555555555555555ULL) << 1);
}

__device__ __forceinline__ uint32_t MixHash32(uint32_t key, uint32_t mask) {
  // the same mix on 32-bit registers; exact for 2k <= 30 bits because every
  // step is masked to 2k bits and wrap-around above bit 31 never reaches them
  key = ((~key) + (key << 21)) & mask;
  key = key ^ (key >> 24);
  key = ((key + (key << 3)) + (key << 8)) & mask;
  key = key ^ (key >> 14);
  key = ((key + (key << 2)) + (key << 4)) & mask;
  key = key ^ (key >> 28);
  // (key << 31) has no bit below 31: the last step is the identity here
  return key & mask;
}

__device__ __forceinline__ uint32_t ReverseGroups32(uint32_t x) {
  x = __brev(x);
  return ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
}

// Window-minimum selection for a compile-time w <= 8, branch-free and in
// registers: the 8 positions of a thread need the hashes of 8 + 2(w-1)
// positions. Window minima come from a sparse table (widths 1, 2, 4, 8);
// position q is a minimizer iff it equals the minimum of one of the (valid)
// windows that contain it - the same set as "left run + right run >= w-1",
// ties included.
template <typename HashT, int W>
__device__ __forceinline__ uint32_t SelectFixedW(const HashT* __restrict__ sh_hash,
                                                 uint32_t hs, uint32_t he, uint32_t qa,
                                                 uint32_t q1, uint32_t L) {
  constexpr HashT kBad = static_cast<HashT>(~static_cast<HashT>(0));
  constexpr int H = W - 1;        // halo
  constexpr int N = 8 + 2 * H;    // slots; slot j = position qa - H + j
  constexpr int P = W >= 8 ? 8 : W >= 4 ? 4 : W >= 2 ? 2 : 1;  // largest power of two <= W
  const int64_t origin = static_cast<int64_t>(qa) - H;
  HashT h[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const int64_t p = origin + j;
    h[j] = (p >= static_cast<int64_t>(hs) && p < static_cast<int64_t>(he)) ? sh_hash[p - hs] : kBad;
  }
  // m[j] = min of slots j .. j + P - 1
  HashT m[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    HashT v = h[j];
#pragma unroll
    for (int t = 1; t < P; ++t) {
      if (j + t < N) v = h[j + t] < v ? h[j + t] : v;
    }
    m[j] = v;
  }
  // minimum of the window starting at slot j, j = 0 .. 7 + H; kBad if the window
  // leaves the read's k-mer positions [0, L)
  HashT wm[8 + H];
#pragma unroll
  for (int j = 0; j < 8 + H; ++j) {
    HashT v = m[j];
    if (W > P) v = m[j + W - P] < v ? m[j + W - P] : v;
    const int64_t p = origin + j;
    wm[j] = (p >= 0 && p + W <= static_cast<int64_t>(L)) ? v : kBad;
  }
  uint32_t flags = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const HashT hq = h[H + i];
    bool is_min = false;
#pragma unroll
    for (int d = 0; d <= H; ++d) is_min = is_min || wm[i + d] == hq;
    if (is_min && hq != kBad && qa + i < q1) flags |= 1u << i;
  }
  return flags;
}

// decoupled look-back status word: state in the top two bits
constexpr uint64_t kStAggregate = 1ULL << 62;
constexpr uint64_t kStPrefix = 2ULL << 62;
constexpr uint64_t kStMask = 3ULL << 62;

// Single pass: every CTA takes the next tile (ticket), selects its minimizers
// and obtains its output offset from the running prefix of the tiles before it
// (decoupled look-back on a status array), so records land in (read,
// position) order without a counting pass. HashT = u32 when 2k <= 30.
template <typename HashT>
__global__ void __launch_bounds__(kSketchThreads)
SketchKernel(const uint64_t* __restrict__ words,
             const uint64_t* __restrict__ woff,
             const uint32_t* __restrict__ lens,
             const uint32_t* __restrict__ ids,
             const uint64_t* __restrict__ tile_off, uint32_t first_read,
             uint32_t last_read, uint32_t k, uint32_t w,
             unsigned int* __restrict__ ticket, uint64_t* __restrict__ status,
             uint64_t* __restrict__ tile_out, uint64_t n_tiles, uint64_t out_cap,
             HashT* __restrict__ out_val, uint64_t* __restrict__ out_org) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr HashT kBad = static_cast<HashT>(~static_cast<HashT>(0));
  const uint32_t halo = w - 1;
  const uint32_t span = kSketchTile + 2 * halo;
  // layout: packed words | hash values | scan scratch | strand bytes
  const uint32_t max_words = (span + 31 + 31) / 32 + 2;
  uint64_t* sh_words = reinterpret_cast<uint64_t*>(smem_raw);
  HashT* sh_hash = reinterpret_cast<HashT*>(sh_words + max_words);
  uint32_t* sh_scan = reinterpret_cast<uint32_t*>(
      (reinterpret_cast<uintptr_t>(sh_hash + span) + 3) & ~uintptr_t(3));
  unsigned char* sh_strand = reinterpret_cast<unsigned char*>(sh_scan + 34);
  __shared__ uint32_t sh_read, sh_tile;
  __shared__ uint64_t sh_excl;

  if (threadIdx.x < 32) {
    // ticket, then the read of this tile by a 32-ary search of the first warp
    // (4 rounds of one load instead of 17 dependent ones)
    uint32_t tk = 0;
    if (threadIdx.x == 0) tk = atomicAdd(ticket, 1u);
    tk = __shfl_sync(0xFFFFFFFFu, tk, 0);
    const uint64_t want = tile_off[first_read] + tk;
    uint32_t lo = first_read, hi = last_read;  // tile_off[lo] <= want < tile_off[hi]
    while (hi - lo > 1) {
      const uint32_t step = (hi - lo + 31) / 32;
      const uint64_t probe = static_cast<uint64_t>(lo) + (threadIdx.x + 1ULL) * step;
      const bool le = probe < hi && tile_off[probe] <= want;
      const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, le));
      const uint64_t nlo = static_cast<uint64_t>(lo) + static_cast<uint64_t>(cnt) * step;
      const uint64_t nhi = nlo + step;
      lo = static_cast<uint32_t>(nlo);
      if (nhi < hi) hi = static_cast<uint32_t>(nhi);
    }
    if (threadIdx.x == 0) {
      sh_tile = tk;
      sh_read = lo;
    }
  }
  __syncthreads();
  const uint32_t tile = sh_tile;
  const uint64_t t = tile_off[first_read] + tile;
  const uint32_t r = sh_read;
  const uint32_t len = lens[r];
  const uint32_t L = len - k + 1;  // k-mer positions (tiles exist only if L >= w)
  const uint32_t q0 = static_cast<uint32_t>(t - tile_off[r]) * kSketchTile;
  const uint32_t q1 = min(q0 + kSketchTile, L);
  const uint32_t hs = q0 >= halo ? q0 - halo : 0;  // hashed range incl. halo
  const uint32_t he = min(q1 + halo, L);

  // ---- stage the packed words this tile touches ----
  const uint64_t* rw = words + woff[r];
  const uint32_t nwords = static_cast<uint32_t>(woff[r + 1] - woff[r]);
  const uint32_t w_lo = hs >> 5;
  const uint32_t w_hi = ((he - 1 + k - 1) >> 5) + 2;  // one spare for the funnel
  for (uint32_t i = w_lo + threadIdx.x; i < w_hi; i += kSketchThreads) {
    sh_words[i - w_lo] = i < nwords ? __ldg(rw + i) : 0ULL;
  }
  __syncthreads();

  // ---- canonical k-mer hash of every position in [hs, he) ----
  for (uint32_t p = hs + threadIdx.x; p < he; p += kSketchThreads) {
    const uint32_t wi = (p >> 5) - w_lo;
    const uint32_t sh = (p & 31) << 1;
    uint64_t lo = sh_words[wi] >> sh;
    if (sh) lo |= sh_words[wi + 1] << (64 - sh);
    HashT h = kBad;  // palindromic k-mers never enter a window
    unsigned char strand = 0;
    if (sizeof(HashT) == 4) {
      const uint32_t mask = (1u << (2 * k)) - 1;
      const uint32_t l32 = static_cast<uint32_t>(lo) & mask;
      const uint32_t rv = (~l32) & mask;
      const uint32_t fw = ReverseGroups32(l32) >> (32 - 2 * k);
      if (fw < rv) {
        h = static_cast<HashT>(MixHash32(fw, mask));
      } else if (fw > rv) {
        h = static_cast<HashT>(MixHash32(rv, mask));
        strand = 1;
      }
    } else {
      const uint64_t mask = (1ULL << (2 * k)) - 1;
      lo &= mask;
      const uint64_t rv = (~lo) & mask;
      const uint64_t fw = ReverseGroups(lo) >> (64 - 2 * k);
      if (fw < rv) {
        h = static_cast<HashT>(MixHash(fw, mask));
      } else if (fw > rv) {
        h = static_cast<HashT>(MixHash(rv, mask));
        strand = 1;
      }
    }
    sh_hash[p - hs] = h;
    sh_strand[p - hs] = strand;
  }
  __syncthreads();

  // ---- select: each thread owns ITEMS consecutive positions ----
  constexpr uint32_t ITEMS = kSketchTile / kSketchThreads;
  static_assert(ITEMS == 8, "SelectFixedW handles 8 positions per thread");
  uint32_t flags = 0;
  const uint32_t qa = q0 + threadIdx.x * ITEMS;
  if (w == 5) {  // raven's default window
    if (qa < q1) flags = SelectFixedW<HashT, 5>(sh_hash, hs, he, qa, q1, L);
  }
#pragma unroll
  for (uint32_t i = 0; i < ITEMS; ++i) {
    const uint32_t q = qa + i;
    if (q >= q1 || w == 5) break;
    const HashT h = sh_hash[q - hs];
    if (h == kBad) continue;
    // consecutive left neighbours with hash >= h (capped)
    const uint32_t lcap = min(halo, q);
    uint32_t ra = 0;
    while (ra < lcap && sh_hash[q - hs - ra - 1] >= h) ++ra;
    const uint32_t rcap = min(halo, L - 1 - q);
    if (ra + rcap < halo) continue;
    uint32_t rb = 0;
    const uint32_t need = halo - ra;
    while (rb < rcap && rb < need && sh_hash[q - hs + rb + 1] >= h) ++rb;
    if (ra + rb >= halo) flags |= 1u << i;
  }

  uint32_t total;
  const uint32_t ex = BlockExclusiveSum<uint32_t, kSketchThreads>(
      __popc(flags), sh_scan, &total);

  // ---- output offset: running prefix of the tiles before this one ----
  // decoupled look-back by the first warp: 32 predecessors per step
  if (threadIdx.x < 32) {
    const uint32_t lane = threadIdx.x;
    uint64_t excl = 0;
    volatile uint64_t* st = status;
    if (tile > 0) {
      if (lane == 0) {
        st[tile] = kStAggregate | total;
        __threadfence();
      }
      __syncwarp();
      int64_t idx = static_cast<int64_t>(tile) - 1;  // lane 0 looks at the nearest tile
      while (true) {
        const int64_t mine = idx - lane;
        uint64_t v = kStPrefix;  // before tile 0: an empty prefix
        if (mine >= 0) {
          do {
            v = st[mine];
          } while ((v & kStMask) == 0);
        }
        const uint32_t pm = __ballot_sync(0xFFFFFFFFu, (v & kStMask) == kStPrefix);
        const int firstp = __ffs(pm) - 1;  // nearest tile that already knows its prefix
        uint64_t part = (firstp < 0 || static_cast<int>(lane) <= firstp) ? (v & ~kStMask) : 0;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, d);
        excl += part;
        if (firstp >= 0) break;
        idx -= 32;
      }
    }
    if (lane == 0) {
      st[tile] = kStPrefix | (excl + total);
      tile_out[tile] = excl;
      if (tile + 1 == n_tiles) tile_out[n_tiles] = excl + total;
      sh_excl = excl;
    }
  }
  __syncthreads();
  uint64_t dst = sh_excl + ex;
  const uint64_t id = static_cast<uint64_t>(ids[r]) << 32;
  while (flags) {
    const uint32_t i = __ffs(flags) - 1;
    flags &= flags - 1;
    const uint32_t q = qa + i;
    if (dst < out_cap) {
      out_val[dst] = sh_hash[q - hs];  // u32 values when 2k <= 30: no narrowing pass later
      out_org[dst] = id | (static_cast<uint64_t>(q) << 1) | sh_strand[q - hs];
    }
    ++dst;
  }
}

// ---------------------------------------------------------------------------
// Fast path: 2k <= 30 (u32 hashes) and a compile-time window W <= 8.
// A thread owns 8 CONSECUTIVE k-mer positions: their 2-bit codes come out of one
// 64-bit funnel of the staged words (8 + k - 1 <= 22 bases), the eight k-mers
// are shifts of it, canonical strand and hash are branch-free, and the window
// minima are two sparse tables in registers over the thread's 8 + 2(W-1)
// neighbouring hashes (shared memory, padded with "no k-mer" outside the read).
// Position q is a minimizer iff its hash equals the LARGEST of the minima of the
// valid windows that contain it (every such minimum is <= hash(q)). About a
// quarter of the instructions of the generic kernel; same tiles, same look-back,
// same output order.
// The records of a tile are compacted in shared memory in output order (values in
// place over the tile's hashes, origins as 16-bit (q - q0) << 1 | strand) and the
// whole CTA writes them with aligned 16-byte stores: each warp store fills whole
// 32-byte sectors instead of a third of ten.
// ---------------------------------------------------------------------------
constexpr int kFastGroup = 4;  // consecutive tiles per CTA: one look-back for all

// the n records of one tile, compacted in shared memory in output order, by the CTA
__device__ __forceinline__ void StoreTileRecords(const uint32_t* __restrict__ sh_val,
                                                 const uint16_t* __restrict__ sh_org,
                                                 uint32_t n, uint64_t org_base,
                                                 uint32_t* __restrict__ out_val,
                                                 uint64_t* __restrict__ out_org) {
  {  // values: 4 a store; a head up to the first 16-byte boundary and a tail
    const uint32_t head =
        min(n, static_cast<uint32_t>((16 - (reinterpret_cast<uintptr_t>(out_val) & 15)) & 15) / 4);
    const uint32_t nvec = (n - head) / 4;
    uint4* vp = reinterpret_cast<uint4*>(out_val + head);
    for (uint32_t i = threadIdx.x; i < nvec; i += kSketchThreads) {
      const uint32_t* s = sh_val + head + 4 * i;
      vp[i] = make_uint4(s[0], s[1], s[2], s[3]);
    }
    const uint32_t tail = head + 4 * nvec;
    if (threadIdx.x < head) out_val[threadIdx.x] = sh_val[threadIdx.x];
    if (threadIdx.x < n - tail) out_val[tail + threadIdx.x] = sh_val[tail + threadIdx.x];
  }
  {  // origins: 2 a store
    const uint32_t head = min(n, (reinterpret_cast<uintptr_t>(out_org) & 15) ? 1u : 0u);
    const uint32_t nvec = (n - head) / 2;
    ulonglong2* op = reinterpret_cast<ulonglong2*>(out_org + head);
    for (uint32_t i = threadIdx.x; i < nvec; i += kSketchThreads) {
      const uint16_t* s = sh_org + head + 2 * i;
      op[i] = make_ulonglong2(org_base + s[0], org_base + s[1]);
    }
    const uint32_t tail = head + 2 * nvec;
    if (threadIdx.x < head) out_org[0] = org_base + sh_org[0];
    if (threadIdx.x < n - tail) out_org[tail + threadIdx.x] = org_base + sh_org[tail + threadIdx.x];
  }
}

template <int W>
__global__ void __launch_bounds__(kSketchThreads, 4)
SketchFastKernel(const uint64_t* __restrict__ words, const uint64_t* __restrict__ woff,
                 const uint32_t* __restrict__ lens, const uint32_t* __restrict__ ids,
                 const uint64_t* __restrict__ tile_off,
                 const uint32_t* __restrict__ tile_read, uint32_t first_read,
                 uint32_t last_read, uint32_t k, unsigned int* __restrict__ ticket,
                 uint64_t* __restrict__ status, uint64_t* __restrict__ tile_out,
                 uint64_t n_tiles, uint64_t out_cap, uint32_t* __restrict__ out_val,
                 uint64_t* __restrict__ out_org) {
  constexpr uint32_t kBad = 0xFFFFFFFFu;
  constexpr int H = W - 1;
  constexpr int ITEMS = 8;
  constexpr int N = ITEMS + 2 * H;  // hashes a thread looks at
  constexpr int kSlots = kSketchTile + 2 * H;
  constexpr int G = kFastGroup;
  constexpr uint32_t kTileWords = (kSlots + 31 + 31) / 32 + 3;
  static_assert(kSketchTile == ITEMS * kSketchThreads, "8 positions per thread");
  static_assert(W >= 2 && W <= 8, "window of 2..8 k-mers");
  static_assert(kSketchTile <= 1u << 15, "16-bit staged origins");
  // packed words of every tile of the group, staged together up front
  __shared__ uint64_t sh_words[G][kTileWords];
  // hashes of every tile of the group (they are the output values; a register copy
  // would cost occupancy): slot j of tile g = position q0 - H + j. At the write-out
  // slot e holds the value of the tile's e-th record.
  __shared__ __align__(16) uint32_t sh_hash_all[kFastGroup][kSlots + 8];
  __shared__ uint16_t sh_org[kSketchTile];  // origins of one tile's records, in order
  __shared__ uint64_t sh_scan[34];
  // per tile of the group: read length in k-mers, first position, read id, staged words
  __shared__ int32_t sh_L[G], sh_q0[G];
  __shared__ uint32_t sh_id[G], sh_wlo[G], sh_wn[G], sh_wvalid[G];
  __shared__ const uint64_t* sh_wsrc[G];
  __shared__ uint32_t sh_group;
  __shared__ uint64_t sh_excl;

  // ticket: the group of G consecutive tiles this CTA sketches (tiles of one launch
  // are ordered by (read, position), so a group may span reads). One lane per tile
  // then looks up its read, so the G chains of dependent loads overlap.
  if (threadIdx.x < 32) {
    uint32_t grp = 0;
    if (threadIdx.x == 0) grp = atomicAdd(ticket, 1u);
    grp = __shfl_sync(0xFFFFFFFFu, grp, 0);
    const uint64_t t = static_cast<uint64_t>(grp) * G + threadIdx.x;
    if (threadIdx.x < G && t < n_tiles) {
      const uint64_t tile_base = tile_off[first_read];
      const bool one_read = last_read - first_read == 1;  // e.g. an external query: no table
      const uint32_t r = one_read ? first_read : tile_read[tile_base + t];
      const int32_t L = static_cast<int32_t>(lens[r] - k + 1);  // k-mer positions, >= W
      const int32_t q0 = static_cast<int32_t>((tile_base + t - tile_off[r]) * kSketchTile);
      const int32_t q1 = min(q0 + static_cast<int32_t>(kSketchTile), L);
      const uint64_t wb = woff[r];
      const uint32_t nwords = static_cast<uint32_t>(woff[r + 1] - wb);
      // words of positions [q0 - H, q1 + H) (+ k - 1 bases), one spare for the funnel
      const uint32_t w_lo = static_cast<uint32_t>(max(q0 - H, 0)) >> 5;
      const uint32_t w_hi = ((static_cast<uint32_t>(min(q1 + H, L)) - 1 + k - 1) >> 5) + 2;
      sh_L[threadIdx.x] = L;
      sh_q0[threadIdx.x] = q0;
      sh_id[threadIdx.x] = ids[r];
      sh_wlo[threadIdx.x] = w_lo;
      sh_wn[threadIdx.x] = w_hi - w_lo;
      sh_wvalid[threadIdx.x] = nwords > w_lo ? nwords - w_lo : 0;
      sh_wsrc[threadIdx.x] = words + wb + w_lo;
    }
    if (threadIdx.x == 0) sh_group = grp;
  }
  __syncthreads();
  const uint32_t group = sh_group;
  const uint64_t t_first = static_cast<uint64_t>(group) * G;
  const int g_count = static_cast<int>(min(static_cast<uint64_t>(G), n_tiles - t_first));

  // ---- stage the packed words of all tiles at once ----
  constexpr uint32_t kStageIters = (G * kTileWords + kSketchThreads - 1) / kSketchThreads;
#pragma unroll
  for (uint32_t it = 0; it < kStageIters; ++it) {
    const uint32_t idx = it * kSketchThreads + threadIdx.x;
    const uint32_t g = idx / kTileWords, j = idx - g * kTileWords;
    if (g < static_cast<uint32_t>(g_count) && j < sh_wn[g]) {
      sh_words[g][j] = j < sh_wvalid[g] ? __ldg(sh_wsrc[g] + j) : 0ULL;
    }
  }
  __syncthreads();

  const uint32_t mask = (1u << (2 * k)) - 1u;
  const uint32_t rshift = 32 - 2 * k;
  // canonical hash of the k-mer whose 2-bit codes start at bit 0 of kb
  auto hash_of = [&](uint32_t kb, uint32_t* strand) -> uint32_t {
    kb &= mask;
    const uint32_t rv = (~kb) & mask;
    const uint32_t fw = ReverseGroups32(kb) >> rshift;
    *strand = rv < fw ? 1u : 0u;
    const uint32_t h = MixHash32(min(fw, rv), mask);
    return fw == rv ? kBad : h;  // palindromic k-mers never enter a window
  };

  uint32_t flags[G], strands[G];

  // ---- canonical hashes of every tile ----
#pragma unroll
  for (int g = 0; g < G; ++g) {
    strands[g] = 0;
    if (g < g_count) {  // (uniform over the CTA)
      const int32_t L = sh_L[g];
      const int32_t q0 = sh_q0[g];
      const int32_t q1 = min(q0 + static_cast<int32_t>(kSketchTile), L);
      const uint32_t w_lo = sh_wlo[g];
      const uint64_t* sh_w = sh_words[g];
      uint32_t* sh_hash = sh_hash_all[g];

      // ---- own positions: 8 consecutive k-mers out of one 64-bit funnel ----
      const int32_t qa = q0 + static_cast<int32_t>(threadIdx.x) * ITEMS;
      {
        const uint32_t wi = (static_cast<uint32_t>(qa) >> 5) - w_lo;
        const uint32_t sh = (static_cast<uint32_t>(qa) & 31) << 1;
        uint64_t lo = 0;
        if (qa < q1) {
          lo = sh_w[wi] >> sh;
          if (sh) lo |= sh_w[wi + 1] << (64 - sh);
        }
        const uint32_t lo_lo = static_cast<uint32_t>(lo), lo_hi = static_cast<uint32_t>(lo >> 32);
        uint32_t st_bits = 0;
        uint32_t* dst = sh_hash + H + threadIdx.x * ITEMS;  // slot of position qa
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
          uint32_t st;
          const uint32_t h = hash_of(__funnelshift_r(lo_lo, lo_hi, 2 * i), &st);
          dst[i] = qa + i < q1 ? h : kBad;
          st_bits |= st << i;
        }
        strands[g] = st_bits;
      }
      // ---- halo positions of the tile: H on each side, one thread each ----
      if (threadIdx.x < 2 * H) {
        const bool left = threadIdx.x < H;
        const int32_t p = left ? q0 - H + static_cast<int32_t>(threadIdx.x)
                               : q0 + static_cast<int32_t>(kSketchTile) +
                                     static_cast<int32_t>(threadIdx.x) - H;
        uint32_t h = kBad;
        if (p >= 0 && p < L) {
          const uint32_t wi = (static_cast<uint32_t>(p) >> 5) - w_lo;
          const uint32_t sh = (static_cast<uint32_t>(p) & 31) << 1;
          uint64_t lo = sh_w[wi] >> sh;
          if (sh) lo |= sh_w[wi + 1] << (64 - sh);
          uint32_t st;
          h = hash_of(static_cast<uint32_t>(lo), &st);
        }
        sh_hash[left ? threadIdx.x : H + kSketchTile + threadIdx.x - H] = h;
      }
    }
  }
  __syncthreads();

  // ---- select; one scan counts the records of all tiles (16 bits a tile) ----
  static_assert(kSketchTile < (1u << 16) && G <= 4, "tile counts packed in a u64");
  uint64_t packed = 0;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    flags[g] = 0;
    if (g < g_count) {
      const int32_t L = sh_L[g];
      const int32_t q0 = sh_q0[g];
      const int32_t q1 = min(q0 + static_cast<int32_t>(kSketchTile), L);
      const int32_t qa = q0 + static_cast<int32_t>(threadIdx.x) * ITEMS;
      // (every window of an interior tile lies inside the read: no bounds tests)
      const bool interior = q0 >= H && q0 + static_cast<int32_t>(kSketchTile) + H <= L;
      uint32_t fl = 0;
      if (qa < q1) {
        uint32_t h[N];
        const uint32_t* src = sh_hash_all[g] + threadIdx.x * ITEMS;  // slot of position qa - H
#pragma unroll
        for (int j = 0; j < N; ++j) h[j] = src[j];
        // minimum of the window starting at slot j (positions qa - H + j .. + W - 1),
        // 0 if the window leaves [0, L)
        uint32_t wm[ITEMS + H];
#pragma unroll
        for (int j = 0; j < ITEMS + H; ++j) {
          uint32_t v = h[j];
#pragma unroll
          for (int t2 = 1; t2 < W; ++t2) v = min(v, h[j + t2]);
          const int32_t s0 = qa - H + j;
          wm[j] = (interior || (s0 >= 0 && s0 + W <= L)) ? v : 0u;
        }
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
          uint32_t best = wm[i];
#pragma unroll
          for (int d = 1; d <= H; ++d) best = max(best, wm[i + d]);
          const uint32_t hq = h[H + i];
          if (best == hq && hq != kBad) fl |= 1u << i;
        }
      }
      flags[g] = fl;
      packed |= static_cast<uint64_t>(__popc(fl)) << (16 * g);
    }
  }
  uint64_t totals;
  const uint64_t ex_packed = BlockExclusiveSum<uint64_t, kSketchThreads>(packed, sh_scan, &totals);
  uint32_t group_total = 0;
#pragma unroll
  for (int g = 0; g < G; ++g) group_total += static_cast<uint32_t>(totals >> (16 * g)) & 0xFFFFu;

  // ---- output offset of the group: decoupled look-back by the first warp ----
  if (threadIdx.x < 32) {
    const uint32_t lane = threadIdx.x;
    uint64_t excl = 0;
    volatile uint64_t* st = status;
    if (group > 0) {
      if (lane == 0) {
        st[group] = kStAggregate | group_total;
        __threadfence();
      }
      __syncwarp();
      int64_t idx = static_cast<int64_t>(group) - 1;
      while (true) {
        const int64_t mine = idx - lane;
        uint64_t v = kStPrefix;  // before group 0: an empty prefix
        if (mine >= 0) {
          do {
            v = st[mine];
          } while ((v & kStMask) == 0);
        }
        const uint32_t pm = __ballot_sync(0xFFFFFFFFu, (v & kStMask) == kStPrefix);
        const int firstp = __ffs(pm) - 1;
        uint64_t part = (firstp < 0 || static_cast<int>(lane) <= firstp) ? (v & ~kStMask) : 0;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, d);
        excl += part;
        if (firstp >= 0) break;
        idx -= 32;
      }
    }
    if (lane == 0) {
      st[group] = kStPrefix | (excl + group_total);
      uint64_t run = excl;
      for (int g = 0; g < g_count; ++g) {
        tile_out[t_first + g] = run;
        run += static_cast<uint32_t>(totals >> (16 * g)) & 0xFFFFu;
      }
      if (t_first + g_count == n_tiles) tile_out[n_tiles] = run;
      sh_excl = excl;
    }
  }
  __syncthreads();

  // ---- write-out, tile by tile: compact in shared memory, then store coalesced ----
  uint64_t base = sh_excl;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (g < g_count) {
      const uint32_t n = static_cast<uint32_t>(totals >> (16 * g)) & 0xFFFFu;
      uint32_t* sh_val = sh_hash_all[g];
      // the value of record e moves to slot e <= its own slot: every thread reads its
      // values before any is overwritten (the barrier also ends the previous tile's
      // stores, which read sh_org)
      uint32_t v[ITEMS];
      const uint32_t* own = sh_val + H + threadIdx.x * ITEMS;
#pragma unroll
      for (int i = 0; i < ITEMS; ++i) v[i] = own[i];
      __syncthreads();
      uint32_t e = static_cast<uint32_t>(ex_packed >> (16 * g)) & 0xFFFFu;
#pragma unroll
      for (int i = 0; i < ITEMS; ++i) {
        if ((flags[g] >> i) & 1u) {
          sh_val[e] = v[i];
          sh_org[e] =
              static_cast<uint16_t>((threadIdx.x * ITEMS + i) << 1 | ((strands[g] >> i) & 1u));
          ++e;
        }
      }
      __syncthreads();
      // past out_cap the pass only counts (the host repeats it with the exact size)
      const uint64_t room = base < out_cap ? out_cap - base : 0;
      const uint32_t n_out = static_cast<uint32_t>(min(static_cast<uint64_t>(n), room));
      if (n_out > 0) {
        // origin = id << 32 | q << 1 | strand = (id << 32 | q0 << 1) + staged origin
        const uint64_t org_base = (static_cast<uint64_t>(sh_id[g]) << 32) |
                                  (static_cast<uint64_t>(static_cast<uint32_t>(sh_q0[g])) << 1);
        StoreTileRecords(sh_val, sh_org, n_out, org_base, out_val + base, out_org + base);
      }
      base += n;
    }
  }
}

__global__ void GatherReadOffsets(const uint64_t* __restrict__ tile_off,
                                  const uint64_t* __restrict__ tile_out,
                                  uint32_t first_read, uint32_t n_reads,
                                  uint64_t* __restrict__ read_off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_reads) return;
  // tile_out has (#tiles + 1) entries, so i == n_reads lands on the total
  read_off[i] = tile_out[tile_off[first_read + i] - tile_off[first_read]];
}

// ---- micromizers: the len/k smallest values of a read's sketch, ties by
// position, back in position order ("minhash", SURVEY.md App. A.2) ----
constexpr int kMicroThreads = 256;
constexpr int kMicroBits = 10;                          // radix digit of the selection
constexpr uint32_t kMicroBins = 1u << kMicroBits;
constexpr size_t kMicroStageBytes = 40 << 10;           // largest on-chip copy of a sketch

// The micromizers of one read whose sketch has more than m records, by the CTA.
// src: the read's values, in shared memory or (a sketch too long for it) in global
// memory; each is its own inlined copy, so on-chip reads compile to shared loads.
template <typename ValT, bool kWrite>
__device__ __forceinline__ void SelectMicromizers(
    const ValT* __restrict__ src, const uint64_t* __restrict__ org, uint32_t cnt, uint32_t m,
    uint32_t k, uint64_t ob, ValT* __restrict__ q_val, uint64_t* __restrict__ q_org,
    uint64_t* __restrict__ thr_val, uint32_t* __restrict__ thr_pos, uint32_t* hist,
    uint32_t* sh_scan, uint64_t* sh_scan64, uint32_t* sh_pick) {
  // ---- radix select of the value with ascending rank m-1 ----
  // (every thread owns 4 consecutive digits of the histogram's scan)
  static_assert(kMicroBins == 4 * kMicroThreads, "4 digits a thread");
  uint64_t prefix = 0, prefix_mask = 0;
  uint32_t want = m - 1;
  for (int shift = static_cast<int>((2 * k + kMicroBits - 1) / kMicroBits - 1) * kMicroBits;
       shift >= 0; shift -= kMicroBits) {
    reinterpret_cast<uint4*>(hist)[threadIdx.x] = make_uint4(0, 0, 0, 0);
    __syncthreads();  // (the first: the values are on chip)
    for (uint32_t i = threadIdx.x; i < cnt; i += kMicroThreads) {
      const uint64_t v = src[i];
      if ((v & prefix_mask) == prefix) {
        atomicAdd(&hist[(v >> shift) & (kMicroBins - 1)], 1u);
      }
    }
    __syncthreads();
    {  // the digit whose cumulative count first exceeds `want`: one block scan
      const uint4 h = reinterpret_cast<const uint4*>(hist)[threadIdx.x];
      uint32_t tot;
      uint32_t run = BlockExclusiveSum<uint32_t, kMicroThreads>(h.x + h.y + h.z + h.w, sh_scan,
                                                                &tot);
      const uint32_t hc[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (run <= want && want < run + hc[j]) {
          sh_pick[0] = 4 * threadIdx.x + j;
          sh_pick[1] = want - run;
        }
        run += hc[j];
      }
    }
    __syncthreads();
    prefix |= static_cast<uint64_t>(sh_pick[0]) << shift;
    prefix_mask |= static_cast<uint64_t>(kMicroBins - 1) << shift;
    want = sh_pick[1];
  }
  const uint64_t T = prefix;
  const uint32_t need_eq = want + 1;  // first need_eq records equal to T

  // ---- ordered compaction: every thread walks its own run of records ----
  // (an odd run length keeps the shared-memory reads of a warp free of conflicts)
  const uint32_t run_len = ((cnt + kMicroThreads - 1) / kMicroThreads) | 1u;
  const uint32_t lo = min(threadIdx.x * run_len, cnt), hi = min(lo + run_len, cnt);
  uint32_t n_eq = 0, n_lt = 0;
  for (uint32_t i = lo; i < hi; ++i) {
    const uint64_t v = src[i];
    n_eq += v == T;
    n_lt += v < T;
  }
  uint64_t tot;
  const uint64_t before = BlockExclusiveSum<uint64_t, kMicroThreads>(
      static_cast<uint64_t>(n_eq) << 32 | n_lt, sh_scan64, &tot);
  uint32_t eq_run = static_cast<uint32_t>(before >> 32);
  uint32_t lt_run = static_cast<uint32_t>(before);
  // (thresholds only: just the thread that holds the last kept tie walks again)
  if (kWrite || (eq_run < need_eq && need_eq <= eq_run + n_eq)) {
    for (uint32_t i = lo; i < hi; ++i) {
      const uint64_t v = src[i];
      const bool is_eq = v == T, is_lt = v < T;
      if (kWrite && (is_lt || (is_eq && eq_run < need_eq))) {
        const uint64_t d = ob + lt_run + min(eq_run, need_eq);
        q_val[d] = static_cast<ValT>(v);
        q_org[d] = org[i];
      }
      if (is_eq && eq_run + 1 == need_eq) {  // the last tie that is kept
        *thr_val = T;
        *thr_pos = (static_cast<uint32_t>(org[i]) >> 1) + 1;
      }
      lt_run += is_lt;
      eq_run += is_eq;
    }
  }
}

// Besides (kWrite) the micromizers themselves, the selection rule of every read is
// left behind as a pair (thr_val, thr_pos): record (value, position) of the read is
// one of its micromizers iff value < thr_val || (value == thr_val && position <
// thr_pos) - what the stage-1 self-join over the index asks of every posting.
// A read's values are copied to shared memory once (dynamic, stage_cap of them) and
// selected there; a sketch longer than that is selected from global memory.
template <typename ValT, bool kWrite>
__global__ void __launch_bounds__(kMicroThreads)
MicromizeKernel(const ValT* __restrict__ s_val,
                const uint64_t* __restrict__ s_org,
                const uint64_t* __restrict__ s_off,  // per read of the sketch
                uint32_t s_first, const uint64_t* __restrict__ q_off,
                uint32_t q_first, uint32_t k, uint32_t stage_cap,
                ValT* __restrict__ q_val, uint64_t* __restrict__ q_org,
                uint64_t* __restrict__ thr_val, uint32_t* __restrict__ thr_pos) {
  extern __shared__ __align__(16) unsigned char micro_smem[];
  __shared__ __align__(16) uint32_t hist[kMicroBins];
  __shared__ uint32_t sh_scan[34];
  __shared__ uint64_t sh_scan64[34];
  __shared__ uint32_t sh_pick[2];  // digit and remaining rank of a radix round
  __shared__ unsigned long long sh_max;

  const uint32_t r = q_first + blockIdx.x;
  const uint64_t b = s_off[r - s_first];
  const uint32_t cnt = static_cast<uint32_t>(s_off[r - s_first + 1] - b);
  const uint64_t ob = q_off[blockIdx.x];
  const uint32_t m = static_cast<uint32_t>(q_off[blockIdx.x + 1] - ob);
  const ValT* val = s_val + b;
  const uint64_t* org = s_org + b;
  if (m == 0) {
    if (threadIdx.x == 0) {
      thr_val[blockIdx.x] = 0;
      thr_pos[blockIdx.x] = 0;
    }
    return;
  }
  if (m >= cnt) {  // keep everything
    if (threadIdx.x == 0) sh_max = 0;
    __syncthreads();
    unsigned long long mx = 0;
    for (uint32_t i = threadIdx.x; i < cnt; i += kMicroThreads) {
      const ValT v = val[i];
      mx = max(mx, static_cast<unsigned long long>(v));
      if (kWrite) {
        q_val[ob + i] = v;
        q_org[ob + i] = org[i];
      }
    }
    atomicMax(&sh_max, mx);
    __syncthreads();
    if (threadIdx.x == 0) {
      thr_val[blockIdx.x] = sh_max;
      thr_pos[blockIdx.x] = 0xFFFFFFFFu;
    }
    return;
  }

  if (cnt <= stage_cap) {
    // the values on chip: 16-byte loads after a head up to the first boundary
    ValT* sh = reinterpret_cast<ValT*>(micro_smem);
    constexpr uint32_t V = 16 / sizeof(ValT);
    const uint32_t head = min(
        cnt, static_cast<uint32_t>((16 - (reinterpret_cast<uintptr_t>(val) & 15)) & 15) /
                 static_cast<uint32_t>(sizeof(ValT)));
    const uint32_t nvec = (cnt - head) / V;
    const uint4* vp = reinterpret_cast<const uint4*>(val + head);
    for (uint32_t i = threadIdx.x; i < nvec; i += kMicroThreads) {
      const uint4 x = __ldg(vp + i);
      if (sizeof(ValT) == 4) {
        sh[head + 4 * i] = x.x;
        sh[head + 4 * i + 1] = x.y;
        sh[head + 4 * i + 2] = x.z;
        sh[head + 4 * i + 3] = x.w;
      } else {
        sh[head + 2 * i] = static_cast<ValT>(static_cast<uint64_t>(x.y) << 32 | x.x);
        sh[head + 2 * i + 1] = static_cast<ValT>(static_cast<uint64_t>(x.w) << 32 | x.z);
      }
    }
    if (threadIdx.x < head) sh[threadIdx.x] = val[threadIdx.x];
    for (uint32_t i = head + V * nvec + threadIdx.x; i < cnt; i += kMicroThreads) sh[i] = val[i];
    SelectMicromizers<ValT, kWrite>(sh, org, cnt, m, k, ob, q_val, q_org, thr_val + blockIdx.x,
                                    thr_pos + blockIdx.x, hist, sh_scan, sh_scan64, sh_pick);
  } else {
    SelectMicromizers<ValT, kWrite>(val, org, cnt, m, k, ob, q_val, q_org, thr_val + blockIdx.x,
                                    thr_pos + blockIdx.x, hist, sh_scan, sh_scan64, sh_pick);
  }
}

size_t SketchSmemBytes(uint32_t w, size_t hash_bytes) {
  const uint32_t halo = w - 1;
  const uint32_t span = kSketchTile + 2 * halo;
  const uint32_t max_words = (span + 31 + 31) / 32 + 2;
  return max_words * 8 + span * hash_bytes + 4 + 34 * 4 + span + 16;
}

}  // namespace

void EnsureTiles(Ctx& c) {
  if (c.tiles_k == c.prm.k && c.h_tile_off.size() == c.n_reads + 1ULL) return;
  c.h_tile_off.assign(c.n_reads + 1ULL, 0);
  for (uint32_t r = 0; r < c.n_reads; ++r) {
    const uint32_t len = c.h_len[r];
    uint64_t tiles = 0;
    if (len >= c.prm.k) {
      const uint32_t L = len - c.prm.k + 1;
      if (L >= c.prm.w) tiles = (L + kSketchTile - 1) / kSketchTile;
    }
    c.h_tile_off[r + 1] = c.h_tile_off[r] + tiles;
  }
  // read of every tile (the fast kernel's lookup)
  {
    const uint64_t nt = c.h_tile_off[c.n_reads];
    if (nt >= 0xFFFFFFFFULL) throw LimitError("too many sketch tiles");
    std::vector<uint32_t> tr(nt);
    for (uint32_t r = 0; r < c.n_reads; ++r) {
      for (uint64_t t = c.h_tile_off[r]; t < c.h_tile_off[r + 1]; ++t) tr[t] = r;
    }
    uint32_t* dtr = c.d_tile_read.reserve(nt + 1);
    if (nt) {
      RVN_CUDA(cudaMemcpyAsync(dtr, tr.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice,
                               c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));  // tr goes out of scope
    }
  }
  // one spare slot: an external query read rides at index n_reads
  uint64_t* d = c.d_tile_off.reserve(c.n_reads + 2ULL);
  RVN_CUDA(cudaMemcpyAsync(d, c.h_tile_off.data(),
                           (c.n_reads + 1ULL) * sizeof(uint64_t),
                           cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  c.tiles_k = c.prm.k;
  c.s_valid = c.q_valid = false;
}

void EnsureSketch(Ctx& c, uint32_t first, uint32_t last) {
  if (c.s_valid && c.s_first == first && c.s_last == last) return;
  if (first < last && (first < c.res_first || last > c.res_last)) {
    throw StateError("the bases of these reads were not uploaded (rvn_reads_upload_range)");
  }
  EnsureTiles(c);
  c.s_valid = false;
  c.q_valid = false;
  const uint32_t nr = last - first;
  const uint64_t n_tiles = c.h_tile_off[last] - c.h_tile_off[first];
  if (n_tiles >= (1ULL << 31)) throw LimitError("too many sketch tiles");

  uint64_t* read_off = c.s_off.reserve(nr + 1ULL);
  c.h_s_off.assign(nr + 1ULL, 0);
  uint64_t total = 0;
  if (n_tiles > 0) {
    TimerBegin(c, "sketch");
    const bool k32 = 2 * c.prm.k <= 30;
    const size_t smem = SketchSmemBytes(c.prm.w, k32 ? 4 : 8);
    // status words + ticket; output capacity from the expected density (all
    // ties of a window minimum are emitted, so a repetitive read can exceed it:
    // the kernel then only counts and the pass is repeated with the exact size)
    uint64_t positions = 0;
    for (uint32_t r = first; r < last; ++r) {
      if (c.h_len[r] >= c.prm.k) positions += c.h_len[r] - c.prm.k + 1;
    }
    uint64_t cap = static_cast<uint64_t>(
                       static_cast<double>(positions) *
                       std::min(1.0, 2.2 / (c.prm.w + 1.0))) + 4096;
    // (u32 values: two per element of the u64-typed buffer)
    cap = std::max<uint64_t>(cap, std::min<uint64_t>(c.s_val.cap * (k32 ? 2 : 1), c.s_org.cap));
    uint64_t* tout = c.tile_out.reserve(n_tiles + 1);
    uint64_t* status = c.tile_status.reserve(n_tiles + 2);
    unsigned int* ticket = reinterpret_cast<unsigned int*>(status + n_tiles);
    for (int attempt = 0; attempt < 2; ++attempt) {
      uint64_t* val = c.s_val.reserve(k32 ? cap / 2 + 1 : cap);
      uint64_t* org = c.s_org.reserve(cap);
      RVN_CUDA(cudaMemsetAsync(status, 0, (n_tiles + 2) * sizeof(uint64_t), c.stream));
      if (!(k32 && c.prm.w == 5)) WaitUpload(c);
      if (k32 && c.prm.w == 5) {  // raven's default window: the fast kernel
        // (status words of this kernel: one per group of kFastGroup tiles)
        const uint64_t n_groups = (n_tiles + kFastGroup - 1) / kFastGroup;
        // An asynchronous upload still in flight: the groups of the reads a chunk
        // completes are launched behind that chunk's event (groups take tickets, and
        // the look-back chain runs on across launches)
        uint64_t launched = 0;
        const uint32_t pieces = c.up_pending ? c.up_chunks : 1;
        for (uint32_t p = 0; p < pieces; ++p) {
          uint64_t upto = n_groups;
          if (c.up_pending) {
            RVN_CUDA(cudaStreamWaitEvent(c.stream, c.up_events[p], 0));
            if (p + 1 < pieces) {
              const uint32_t r = std::min(std::max(c.up_read_end[p], first), last);
              upto = (c.h_tile_off[r] - c.h_tile_off[first]) / kFastGroup;
            }
          }
          if (upto <= launched) continue;
          SketchFastKernel<5><<<static_cast<unsigned>(upto - launched), kSketchThreads, 0,
                                c.stream>>>(
              c.d_words.get(), c.d_woff.get(), c.d_len.get(), c.d_ids.get(),
              c.d_tile_off.get(), c.d_tile_read.get(), first, last, c.prm.k, ticket, status, tout,
              n_tiles, cap, reinterpret_cast<uint32_t*>(val), org);
          launched = upto;
          ++c.launches;
        }
        --c.launches;  // (counted once more below)
        c.up_pending = false;
      } else if (k32) {
        SketchKernel<uint32_t><<<static_cast<unsigned>(n_tiles), kSketchThreads, smem,
                                 c.stream>>>(
            c.d_words.get(), c.d_woff.get(), c.d_len.get(), c.d_ids.get(),
            c.d_tile_off.get(), first, last, c.prm.k, c.prm.w, ticket, status, tout,
            n_tiles, cap, reinterpret_cast<uint32_t*>(val), org);
      } else {
        SketchKernel<uint64_t><<<static_cast<unsigned>(n_tiles), kSketchThreads, smem,
                                 c.stream>>>(
            c.d_words.get(), c.d_woff.get(), c.d_len.get(), c.d_ids.get(),
            c.d_tile_off.get(), first, last, c.prm.k, c.prm.w, ticket, status, tout,
            n_tiles, cap, val, org);
      }
      RVN_LAUNCH_CHECK();
      ++c.launches;
      total = ReadU64(c, tout + n_tiles);
      if (total <= cap) break;
      cap = total;  // denser than expected: once more with the exact size
    }
    GatherReadOffsets<<<CeilDiv(nr + 1ULL, 256), 256, 0, c.stream>>>(
        c.d_tile_off.get(), tout, first, nr, read_off);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    TimerEnd(c);
    RVN_CUDA(cudaMemcpyAsync(c.h_s_off.data(), read_off,
                             (nr + 1ULL) * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  } else {
    WaitUpload(c);
    RVN_CUDA(cudaMemsetAsync(read_off, 0, (nr + 1ULL) * sizeof(uint64_t),
                             c.stream));
  }
  c.s_first = first;
  c.s_last = last;
  c.s_n = total;
  c.s_is32 = 2 * c.prm.k <= 30;
  c.s_valid = true;
}

namespace {

// write == true: micromizers (c.q_*) and thresholds (c.qt_*); false: thresholds only
void Micromize(Ctx& c, uint32_t first, uint32_t last, bool write) {
  if (!c.s_valid || first < c.s_first || last > c.s_last) {
    EnsureSketch(c, first, last);
  }
  if (write) c.q_valid = false;
  c.qt_valid = false;
  const uint32_t nr = last - first;
  c.h_q_off.assign(nr + 1ULL, 0);
  for (uint32_t i = 0; i < nr; ++i) {
    const uint32_t r = first + i;
    const uint64_t cnt = c.h_s_off[r - c.s_first + 1] - c.h_s_off[r - c.s_first];
    const uint64_t m = c.h_len[r] / c.prm.k;
    c.h_q_off[i + 1] = c.h_q_off[i] + (m < cnt ? m : cnt);
  }
  const uint64_t total = c.h_q_off[nr];
  // shared memory for the longest sketch that is selected (len/k < its length), up to
  // kMicroStageBytes; longer ones are selected from global memory
  const size_t val_bytes = c.s_is32 ? 4 : 8;
  uint64_t longest = 0;
  for (uint32_t i = 0; i < nr; ++i) {
    const uint32_t r = first + i;
    const uint64_t cnt = c.h_s_off[r - c.s_first + 1] - c.h_s_off[r - c.s_first];
    if (c.h_q_off[i + 1] - c.h_q_off[i] < cnt) longest = std::max(longest, cnt);
  }
  const uint32_t stage_cap =
      static_cast<uint32_t>(std::min<uint64_t>(longest, kMicroStageBytes / val_bytes));
  const size_t smem = stage_cap * val_bytes;
  uint64_t* qoff = c.q_off.reserve(nr + 1ULL);
  RVN_CUDA(cudaMemcpyAsync(qoff, c.h_q_off.data(),
                           (nr + 1ULL) * sizeof(uint64_t),
                           cudaMemcpyHostToDevice, c.stream));
  uint64_t* qv = write ? c.q_val.reserve(total) : c.q_val.get();
  uint64_t* qo = write ? c.q_org.reserve(total) : c.q_org.get();
  uint64_t* tv = c.qt_val.reserve(nr + 1ULL);
  uint32_t* tp = c.qt_pos.reserve(nr + 1ULL);
  if (nr > 0) {
    TimerBegin(c, "micromize");
    RVN_CUDA(cudaMemsetAsync(tv, 0, (nr + 1ULL) * sizeof(uint64_t), c.stream));
    RVN_CUDA(cudaMemsetAsync(tp, 0, (nr + 1ULL) * sizeof(uint32_t), c.stream));
    if (c.s_is32) {  // micromizer values stay u32 like the sketch's
      auto* sv = reinterpret_cast<const uint32_t*>(c.s_val.get());
      auto* q32 = reinterpret_cast<uint32_t*>(qv);
      if (write) {
        MicromizeKernel<uint32_t, true><<<nr, kMicroThreads, smem, c.stream>>>(
            sv, c.s_org.get(), c.s_off.get(), c.s_first, qoff, first, c.prm.k, stage_cap, q32, qo,
            tv, tp);
      } else {
        MicromizeKernel<uint32_t, false><<<nr, kMicroThreads, smem, c.stream>>>(
            sv, c.s_org.get(), c.s_off.get(), c.s_first, qoff, first, c.prm.k, stage_cap, q32, qo,
            tv, tp);
      }
    } else if (write) {
      MicromizeKernel<uint64_t, true><<<nr, kMicroThreads, smem, c.stream>>>(
          c.s_val.get(), c.s_org.get(), c.s_off.get(), c.s_first, qoff, first, c.prm.k, stage_cap,
          qv, qo, tv, tp);
    } else {
      MicromizeKernel<uint64_t, false><<<nr, kMicroThreads, smem, c.stream>>>(
          c.s_val.get(), c.s_org.get(), c.s_off.get(), c.s_first, qoff, first, c.prm.k, stage_cap,
          qv, qo, tv, tp);
    }
    RVN_LAUNCH_CHECK();
    ++c.launches;
    TimerEnd(c);
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));  // h_q_off staging is reusable
  if (write) {
    c.q_first = first;
    c.q_last = last;
    c.q_n = total;
    c.q_is32 = c.s_is32;
    c.q_valid = true;
  } else if (c.q_valid) {
    // (q_off / h_q_off now describe [first, last): an older micromizer set is gone)
    c.q_valid = c.q_first == first && c.q_last == last;
  }
  c.qt_first = first;
  c.qt_last = last;
  c.qt_valid = true;
}

}  // namespace

void EnsureMicromizers(Ctx& c, uint32_t first, uint32_t last) {
  if (c.q_valid && c.q_first == first && c.q_last == last) return;
  Micromize(c, first, last, true);
}

// only the per-read selection rule (c.qt_*) and the counts (c.h_q_off)
void EnsureThresholds(Ctx& c, uint32_t first, uint32_t last) {
  if (c.qt_valid && c.qt_first == first && c.qt_last == last) return;
  Micromize(c, first, last, false);
}

}  // namespace rvn
