// raven_b200 — seed lookup, hit expansion and chaining on sm_90a.
//
// Replaces ram::MinimizerEngine::Map + Chain (un-vendored; call sites
// RavenLib/src/construct.cc:59-64 -> Map(seq,1,1,1) and :377-381 ->
// Map(seq,1,1,0,&filtered); algorithm SURVEY.md App. A.2).
//
//   probe   one thread per query minimizer: bucket table -> sorted run ->
//           (first posting, count) or "filtered" if count > occurrence
//   expand  hits (ram "Match": group = (rhs_id<<1|same_strand)<<32|diagonal,
//           positions = lhs_pos<<32|rhs_pos) written per query read
//   chain   each read's hits split by (rhs_id, strand) pair, each pair chained
//           on chip by one thread or one CTA by its size, large reads whole by a
//           CTA over global memory; ram's per-band rules are chain.cuh's. The
//           overlaps are re-ordered into the reference's output order.
//
// The chain result is a pure function of the MULTISET of hits of a query
// (both reference sorts are total orders here: equal (group, positions)
// pairs cannot occur), so hit generation order is free (DESIGN.md).
#include <algorithm>

#include "chain.cuh"
#include "engine.cuh"
#include "seed.cuh"

namespace rvn {

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads)
ProbeKernel(IndexView ix, ValView q_val,
            const uint64_t* __restrict__ q_org, uint64_t q_begin, uint64_t n_q,
            bool avoid_equal, bool avoid_symmetric,
            uint32_t* __restrict__ cnt, uint32_t* __restrict__ first,
            uint8_t* __restrict__ filt) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= n_q) return;
  const uint32_t lhs_id = static_cast<uint32_t>(q_org[q_begin + i] >> 32);
  ProbeRun(ix, q_val[q_begin + i], lhs_id, avoid_equal, avoid_symmetric, first + i, cnt + i,
           filt + i);
  // the posting count is re-derived in ExpandKernel from the run itself
}

// hit stores of the single-GPU map: one array of groups, one of positions
struct HitStore {
  uint64_t* grp;
  uint64_t* pos;
  __device__ __forceinline__ void operator()(uint64_t d, uint64_t g, uint64_t p,
                                             uint32_t) const {
    grp[d] = g;
    pos[d] = p;
  }
};

__global__ void __launch_bounds__(kThreads)
ExpandKernel(IndexView ix, ValView q_val,
             const uint64_t* __restrict__ q_org, uint64_t q_begin, uint64_t n_q,
             bool avoid_equal, bool avoid_symmetric,
             const uint32_t* __restrict__ cnt,
             const uint32_t* __restrict__ first,
             const uint64_t* __restrict__ hit_off, uint64_t* __restrict__ h_grp,
             uint64_t* __restrict__ h_pos) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= n_q) return;
  const uint32_t left = cnt[i];
  if (left == 0) return;
  const uint64_t v = q_val[q_begin + i];
  const uint64_t lo = q_org[q_begin + i];
  const uint64_t dst = hit_off[i];
  ExpandRun(ix, v, lo, first[i], left, avoid_equal, avoid_symmetric, dst,
            HitStore{h_grp, h_pos});
}

// ---- fast path of probe + expand -------------------------------------------
// With avoid_equal && avoid_symmetric over an index sorted by read, or with both
// flags off, the kept postings are a SUFFIX of the run (seed.cuh: ProbeSuffix). The
// probe then only needs the first kept posting, and the expansion can be done by
// whole warps with fully coalesced stores (seed.cuh: ExpandWarp).
__global__ void __launch_bounds__(kThreads)
ProbeSuffixKernel(IndexView ix, ValView q_val,
                  const uint64_t* __restrict__ q_org, uint64_t q_begin, uint64_t n_q,
                  bool strict_above, uint32_t* __restrict__ cnt,
                  uint32_t* __restrict__ first, uint8_t* __restrict__ filt) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= n_q) return;
  ProbeSuffix(ix, q_val[q_begin + i], strict_above, q_org + q_begin, i, first + i, cnt + i,
              filt + i);
}

// the same probe over queries sorted by value: neighbouring threads walk
// neighbouring parts of the bucket table and of the postings (coalesced,
// TLB-friendly) instead of 67 M independent random probes into 12 GB
__global__ void __launch_bounds__(kThreads)
ProbeSortedKernel(IndexView ix, ValView sorted_val,
                  const uint32_t* __restrict__ sorted_idx,
                  const uint64_t* __restrict__ q_org, uint64_t q_begin, uint64_t n_q,
                  bool strict_above, uint64_t* __restrict__ packed) {
  const uint64_t t = static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (t >= n_q) return;
  const uint64_t v = sorted_val[t];
  const uint32_t i = sorted_idx[t];
  uint32_t fk, kept;
  uint8_t over;
  ProbeSuffix(ix, v, strict_above, q_org + q_begin, i, &fk, &kept, &over);
  // ONE scattered store per query (a partial-sector write costs a read-modify-
  // write in HBM): first kept posting | over-threshold flag | kept count
  packed[i] = (static_cast<uint64_t>(fk) << 32) | (static_cast<uint64_t>(over) << 31) | kept;
}

__global__ void UnpackProbe(const uint64_t* __restrict__ packed, uint64_t n,
                            uint32_t* __restrict__ cnt, uint32_t* __restrict__ first,
                            uint8_t* __restrict__ filt) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t p = packed[i];
  cnt[i] = static_cast<uint32_t>(p) & 0x7FFFFFFFu;
  first[i] = static_cast<uint32_t>(p >> 32);
  filt[i] = static_cast<uint8_t>((p >> 31) & 1);
}


__global__ void __launch_bounds__(kThreads)
ExpandWarpKernel(IndexView ix, const uint64_t* __restrict__ q_org, uint64_t q_begin,
                 uint64_t n_q, const uint32_t* __restrict__ cnt,
                 const uint32_t* __restrict__ first, const uint64_t* __restrict__ hit_off,
                 uint64_t* __restrict__ h_grp, uint64_t* __restrict__ h_pos) {
  const uint64_t i = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x);
  const bool valid = i < n_q;
  ExpandWarp(ix.org, threadIdx.x & 31, valid ? cnt[i] : 0, valid ? first[i] : 0,
             valid ? q_org[q_begin + i] : 0, valid ? hit_off[i] : 0, HitStore{h_grp, h_pos});
}

// ---- stage-1 hits by a self-join over the index ----
// In stage 1 (construct.cc:59-64) the queries of a flush are the micromizers of reads
// that are themselves in the index, so every query IS a posting of the run of its
// value: a posting (value v, read r, position p) is a query iff it passes r's
// selection rule (thr_val, thr_pos; sketch.cu), and its hits are the postings of the
// same run with a larger read id - the ones that follow it, the run being in read
// order. No query sort and no table probe: one sweep over the sorted postings fills
// the slots of the index batch's reads from its first join flush on, and each flush expands
// its own reads' slots (the order of the hits inside a read is free, see the
// header). Runs longer than `occurrence` give no hits.
struct JoinView {
  ValView val;
  const uint64_t* org;
  uint64_t n;
  uint32_t occurrence;
  const uint64_t* thr_val;  // of reads [first, last)
  const uint32_t* thr_pos;
  uint32_t first, last;     // query reads: the index batch's reads from the first join flush on
};

__device__ __forceinline__ bool JoinIsQuery(const JoinView& jv, uint64_t v, uint64_t o) {
  const uint32_t r = static_cast<uint32_t>(o >> 32);
  if (r < jv.first || r >= jv.last) return false;
  const uint64_t t = jv.thr_val[r - jv.first];
  return v < t || (v == t && (static_cast<uint32_t>(o) >> 1) < jv.thr_pos[r - jv.first]);
}

// First position in [lo, hi] at which the predicate `past` holds, `past` being false
// then true over [lo, hi) and taken as true at hi. The whole warp searches: each step
// probes 32 evenly spaced positions and keeps the stretch between the last false and
// the first true probe, so a range of L positions takes ceil(log32 L) steps.
template <typename Pred>
__device__ __forceinline__ uint64_t WarpFirst(uint64_t lo, uint64_t hi, uint32_t lane,
                                              Pred past) {
  while (lo < hi) {
    const uint64_t step = (hi - lo + 31) / 32;
    const uint64_t p = lo + (lane + 1) * step - 1;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, p >= hi || past(p));
    if (!b) return hi;  // (lane 31 probed hi - 1)
    const uint64_t f = __ffs(b) - 1;
    hi = min(hi, lo + (f + 1) * step - 1);
    lo += f * step;
  }
  return lo;
}

// One warp per 32 consecutive postings. The hits of query posting i (value v, read r)
// are the postings of v's run that follow the segment of (v, r), so what i needs is
// its run's start and end and its segment's end: ballots of "value changes" and
// "value or read changes" between neighbours find the ones inside the warp. A run
// crossing the warp's edge costs one more coalesced step of 32 postings past the
// edge, which settles most runs, and past that a WarpFirst search, no further than
// `occurrence` + 1 postings when the threshold is set (a longer run gives no hits).
// So a warp costs O(1 + log32 L) steps for a run of L postings, whatever L and the
// threshold, and the sweep is linear in the postings up to that factor.
// Every query posting with hits takes the next free slot of its read (slots
// [q_off[r], q_off[r + 1]) - one per micromizer - in any order) and leaves (posting
// index, number of hits) there: ONE scattered 8-byte store per query, as a partial-
// sector write costs a read-modify-write in HBM.
__global__ void __launch_bounds__(kThreads)
JoinSweepKernel(JoinView jv, const uint64_t* __restrict__ q_off,
                uint32_t* __restrict__ cursor, uint64_t* __restrict__ packed) {
  constexpr uint32_t kAll = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t base = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x) & ~31ULL;
  if (base >= jv.n) return;  // (whole warps)
  const uint64_t i = base + lane;
  const bool valid = i < jv.n;
  const uint64_t v = valid ? jv.val[i] : 0;
  const uint64_t o = valid ? jv.org[i] : 0;
  const uint32_t r = static_cast<uint32_t>(o >> 32);
  const bool q = valid && JoinIsQuery(jv, v, o);
  if (!__any_sync(kAll, q)) return;

  uint64_t vn = __shfl_down_sync(kAll, v, 1);
  uint32_t rn = __shfl_down_sync(kAll, r, 1);
  uint64_t vp = __shfl_up_sync(kAll, v, 1);
  const bool has_next = i + 1 < jv.n;
  if (lane == 31 && has_next) {
    vn = jv.val[i + 1];
    rn = static_cast<uint32_t>(jv.org[i + 1] >> 32);
  }
  if (lane == 0 && i > 0) vp = jv.val[i - 1];
  const bool run_tail = !has_next || vn != v;  // (lanes beyond n: tails)
  const uint32_t tails = __ballot_sync(kAll, run_tail);
  const uint32_t seg_tails = __ballot_sync(kAll, run_tail || rn != r);
  const uint32_t heads = __ballot_sync(kAll, i == 0 || vp != v);
  const uint32_t at_or_above = kAll << lane, at_or_below = kAll >> (31 - lane);
  // ends are exclusive; 0 = beyond the warp (every end inside it is >= 1)
  uint64_t run_end = (tails & at_or_above) ? base + __ffs(tails & at_or_above) : 0;
  uint64_t seg_end = (seg_tails & at_or_above) ? base + __ffs(seg_tails & at_or_above) : 0;
  bool over = false;
  const bool limited = jv.occurrence != kAll;

  // the warp's last run goes on past it
  if (__any_sync(kAll, q && run_end == 0)) {
    const uint64_t vl = __shfl_sync(kAll, v, 31);
    const uint32_t rl = __shfl_sync(kAll, r, 31);
    const uint64_t j = base + 32, k = j + lane;
    const bool dv = k >= jv.n || jv.val[k] != vl;
    const uint32_t bv = __ballot_sync(kAll, dv);
    const uint32_t bs =
        __ballot_sync(kAll, dv || static_cast<uint32_t>(jv.org[k] >> 32) != rl);
    uint64_t e_run = bv ? j + __ffs(bv) - 1 : 0;
    bool o_fw = false;
    if (!bv) {  // the run holds [base + 31, j + 32), so j + 32 <= n
      if (limited && 33 > jv.occurrence) {
        o_fw = true;
      } else {
        const uint64_t hi = limited ? min(jv.n, base + 32 + jv.occurrence) : jv.n;
        e_run = WarpFirst(j + 32, hi, lane, [&](uint64_t p) { return jv.val[p] != vl; });
        // still v at hi: the run holds [base + 31, hi], occurrence + 2 postings
        o_fw = e_run == hi && hi < jv.n && jv.val[hi] == vl;
      }
    }
    uint64_t e_seg = bs ? j + __ffs(bs) - 1 : 0;
    if (!bs && !o_fw) {  // postings [j + 32, e_run) are all of v's run, in read order
      e_seg = WarpFirst(j + 32, e_run, lane, [&](uint64_t p) {
        return static_cast<uint32_t>(jv.org[p] >> 32) != rl;
      });
    }
    if (run_end == 0) {
      run_end = e_run;
      over = o_fw;
    }
    if (seg_end == 0) seg_end = e_seg;
  }
  // the warp's first run began before it (only its length matters)
  uint32_t run_start =
      (heads & at_or_below) ? static_cast<uint32_t>(base) + 31 - __clz(heads & at_or_below) : 0;
  if (limited && __any_sync(kAll, q && !over && !(heads & at_or_below))) {
    const uint64_t vf = __shfl_sync(kAll, v, 0);
    const uint64_t e0 = __shfl_sync(kAll, run_end, 0);  // (that run's end)
    const int64_t j = static_cast<int64_t>(base) - 32, k = j + lane;
    const uint32_t bv = __ballot_sync(kAll, k < 0 || jv.val[k] != vf);
    uint64_t s_run;
    if (bv) {
      s_run = static_cast<uint64_t>(j + 32 - __clz(bv));
    } else {
      // the run holds [j, e0); a start before e0 - occurrence - 1 changes nothing
      const uint64_t lo = e0 > jv.occurrence + 1ULL ? e0 - jv.occurrence - 1 : 0;
      s_run = lo >= static_cast<uint64_t>(j)
                  ? static_cast<uint64_t>(j)
                  : WarpFirst(lo, static_cast<uint64_t>(j), lane,
                              [&](uint64_t p) { return jv.val[p] == vf; });
    }
    if (!(heads & at_or_below)) run_start = static_cast<uint32_t>(s_run);
  }
  if (!q || over || (limited && run_end - run_start > jv.occurrence)) return;
  const uint32_t kept = static_cast<uint32_t>(run_end - seg_end);
  if (!kept) return;
  const uint32_t rr = r - jv.first;
  const uint64_t slot = q_off[rr] + atomicAdd(cursor + rr, 1u);
  packed[slot] = (i << 32) | kept;
}

__global__ void UnpackJoin(const uint64_t* __restrict__ packed, uint64_t n,
                           uint32_t* __restrict__ cnt) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) cnt[i] = static_cast<uint32_t>(packed[i]);
}

// ExpandWarpKernel over the slots of JoinSweepKernel: the query's own posting gives
// its origin, its hits follow it in the run (after the postings of the same read)
__global__ void __launch_bounds__(kThreads)
ExpandJoinKernel(const uint64_t* __restrict__ i_org, const uint64_t* __restrict__ packed,
                 uint64_t n_q, const uint64_t* __restrict__ hit_off,
                 uint64_t* __restrict__ h_grp, uint64_t* __restrict__ h_pos) {
  const uint64_t i = (static_cast<uint64_t>(blockIdx.x) * kThreads + threadIdx.x);
  const bool valid = i < n_q;
  const uint64_t pk = valid ? packed[i] : 0;
  const uint32_t my_cnt = static_cast<uint32_t>(pk);
  uint32_t my_first = 0;
  uint64_t my_org = 0;
  if (my_cnt) {
    const uint32_t post = static_cast<uint32_t>(pk >> 32);
    my_org = i_org[post];
    my_first = post + 1;
    while ((i_org[my_first] >> 32) == (my_org >> 32)) ++my_first;  // same read: not a hit
  }
  ExpandWarp(i_org, threadIdx.x & 31, my_cnt, my_first, my_org, valid ? hit_off[i] : 0,
             HitStore{h_grp, h_pos});
}

// per-read offsets out of per-record offsets
__global__ void GatherU64(const uint64_t* __restrict__ src,
                          const uint64_t* __restrict__ idx, uint64_t idx_base,
                          uint64_t n, uint64_t* __restrict__ dst) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  dst[i] = src[idx[i] - idx_base];
}

// positions of over-frequent query minimizers, compacted in sketch order
__global__ void FilteredFlagsToU32(const uint8_t* __restrict__ filt, uint64_t n,
                                   uint32_t* __restrict__ out) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = filt[i];
}
__global__ void ScatterFiltered(const uint8_t* __restrict__ filt,
                                const uint64_t* __restrict__ pos,
                                const uint64_t* __restrict__ q_org,
                                uint64_t q_begin, uint64_t n,
                                uint32_t* __restrict__ out) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n || !filt[i]) return;
  out[pos[i]] = static_cast<uint32_t>(q_org[q_begin + i]) >> 1;
}

// ---------------------------------------------------------------------------
// chaining
// ---------------------------------------------------------------------------

// Bitonic sorting network of the CTA over npad slots (a power of two), ascending:
// exchange(i, j, up) orders slots i < j, the smaller into i when `up`, else into j.
template <int THREADS, typename Exchange>
__device__ __forceinline__ void BitonicSort(uint32_t npad, Exchange exchange) {
  for (uint32_t size = 2; size <= npad; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = threadIdx.x; t < (npad >> 1); t += THREADS) {
        const uint32_t i = 2 * t - (t & (stride - 1));
        exchange(i, i + stride, (i & size) == 0);
      }
      __syncthreads();
    }
  }
}

// sorts (A[i], B[i]) pairs ascending by (A, B); npad is a power of two
template <int THREADS>
__device__ void BitonicSortPairs(uint64_t* A, uint64_t* B, uint32_t npad) {
  BitonicSort<THREADS>(npad, [=](uint32_t i, uint32_t j, bool up) {
    const uint64_t ai = A[i], aj = A[j], bi = B[i], bj = B[j];
    const bool gt = ai > aj || (ai == aj && bi > bj);
    if (gt == up) {
      A[i] = aj;
      A[j] = ai;
      B[i] = bj;
      B[j] = bi;
    }
  });
}

// Everything a CTA needs to chain the hits of one query read. IdxT = u16 for
// the shared-memory path (n <= 65534), u32 for the global scratch path.
template <typename IdxT>
struct ChainWork {
  uint64_t* G;   // npad   group, later band tag
  uint64_t* P;   // npad   positions
  IdxT* LB;      // n + 1  lower bounds, later LIS "minimal"+indices (n + nb + 1)
  IdxT* PD;      // n      predecessor
  IdxT* IB;      // n/4+1  band begin
  IdxT* IE;      // n/4+1  band end
  uint32_t* CNT; // n/4+1  overlaps per band
  // the index arrays for n hits from idx on, CNT at the next 4-byte boundary
  __device__ __forceinline__ void PlaceIndices(IdxT* idx, uint32_t n) {
    const uint32_t nb = n / 4 + 1;
    LB = idx;
    PD = LB + (n + nb + 2);
    IB = PD + (n + 1);
    IE = IB + nb;
    CNT = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(IE + nb) + 3) & ~uintptr_t(3));
  }
};

// BandLis storage of ChainRead: tail(n) at minimal[n], then the chain from minimal[0] on
template <typename IdxT>
struct ArrayLis {
  IdxT *minimal, *predecessor;
  __device__ uint32_t tail(uint32_t n) const { return minimal[n]; }
  __device__ void set_tail(uint32_t n, uint32_t v) const { minimal[n] = static_cast<IdxT>(v); }
  __device__ void set_chain(uint32_t x, uint32_t v) const { minimal[x] = static_cast<IdxT>(v); }
  __device__ uint32_t pred(uint32_t x) const { return predecessor[x]; }
  __device__ void set_pred(uint32_t x, uint32_t v) const { predecessor[x] = static_cast<IdxT>(v); }
};

template <typename IdxT, int THREADS>
__device__ uint32_t ChainRead(const ChainWork<IdxT>& wk, uint32_t n,
                              uint32_t npad, uint32_t lhs_id,
                              const ChainParams& cp, uint32_t* sm32,
                              rvn_overlap* __restrict__ ovl_raw,
                              unsigned long long* __restrict__ ovl_counter,
                              uint64_t ovl_cap, uint64_t* out_base,
                              uint64_t* __restrict__ ovl_key = nullptr, uint64_t key_hi = 0) {
  uint64_t* G = wk.G;
  uint64_t* P = wk.P;
  __shared__ unsigned long long sh_base;

  // 1. order by (group, positions); padding is all-ones and sorts last, and
  //    G[n] doubles as the reference's stop dummy
  BitonicSortPairs<THREADS>(G, P, npad);

  // 2. lower bounds: LB[i] = first j with G[i] - G[j] <= bandwidth
  for (uint32_t i = threadIdx.x; i <= n; i += THREADS) {
    const uint64_t gi = i < n ? G[i] : ~0ULL;
    uint32_t lo = 0, hi = i;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (gi - G[mid] <= cp.bandwidth) {
        hi = mid;
      } else {
        lo = mid + 1;
      }
    }
    wk.LB[i] = static_cast<IdxT>(lo);
  }
  __syncthreads();

  // 3. events: at i (1..n) the window [LB[i-1], i) closes; it qualifies with
  //    >= 4 hits; a qualifying window overlapping the previous qualifying
  //    one extends it. Done chunk-wise with carried state.
  uint32_t carry_prevq = 0;  // last qualifying event index so far (0 = none)
  uint32_t carry_nb = 0;     // bands opened so far
  for (uint32_t base = 1; base <= n; base += THREADS) {
    const uint32_t i = base + threadIdx.x;
    uint32_t e = 0, jp = 0;
    if (i <= n) {
      jp = wk.LB[i - 1];
      const uint64_t gi = i < n ? G[i] : ~0ULL;
      e = (gi - G[jp] > cp.bandwidth) && (i - jp >= 4);
    }
    // previous qualifying event (exclusive max-scan of e ? i : 0)
    const uint32_t incl = BlockInclusiveMax<uint32_t, THREADS>(e ? i : 0u, sm32);
    uint32_t prevq_incl_before;  // max over lanes < this one
    {
      // shift by one lane: recompute exclusive from inclusive of neighbours
      __shared__ uint32_t sh_incl[THREADS];
      sh_incl[threadIdx.x] = incl;
      __syncthreads();
      prevq_incl_before = threadIdx.x ? sh_incl[threadIdx.x - 1] : 0u;
      __syncthreads();
    }
    const uint32_t prevq = max(carry_prevq, prevq_incl_before);
    const uint32_t start = e && (prevq == 0 || prevq <= jp);
    uint32_t tot;
    const uint32_t ex = BlockExclusiveSum<uint32_t, THREADS>(start, sm32, &tot);
    if (e) {
      const uint32_t band = carry_nb + ex + start - 1;  // band this event feeds
      if (start) {
        wk.IB[band] = static_cast<IdxT>(jp);
        // the previous band (if any) ended at the previous qualifying event
        if (prevq != 0) wk.IE[band - 1] = static_cast<IdxT>(prevq);
      }
    }
    carry_nb += tot;
    // last qualifying event of the chunk
    {
      __shared__ uint32_t sh_last;
      if (threadIdx.x == THREADS - 1) sh_last = max(carry_prevq, incl);
      __syncthreads();
      carry_prevq = sh_last;
      __syncthreads();
    }
  }
  const uint32_t nb = carry_nb;
  if (threadIdx.x == 0 && nb) wk.IE[nb - 1] = static_cast<IdxT>(carry_prevq);
  __syncthreads();
  if (nb == 0) return 0;

  // 4. tag hits with their band (2b+1) or the gap before band b (2b), then
  //    order each band by positions with one more (tag, positions) sort
  for (uint32_t i = threadIdx.x; i < npad; i += THREADS) {
    if (i >= n) {
      G[i] = ~0ULL;
      continue;
    }
    // band with the largest begin <= i
    uint32_t lo = 0, hi = nb;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (wk.IB[mid] <= i) {
        lo = mid + 1;
      } else {
        hi = mid;
      }
    }
    // lo = number of bands beginning at or before i
    uint64_t tag;
    if (lo == 0) {
      tag = 0;
    } else if (i < wk.IE[lo - 1]) {
      tag = 2ULL * (lo - 1) + 1;
    } else {
      tag = 2ULL * lo;
    }
    // keep rhs_id/strand of the band reachable after the sort: stash the
    // top 32 group bits in the low half of the tag word
    G[i] = (tag << 32) | (G[i] >> 32);
  }
  __syncthreads();
  BitonicSortPairs<THREADS>(G, P, npad);

  // 5. one thread per band: ram's chain rules (chain.cuh), counting the overlaps
  IdxT* MINI = wk.LB;  // re-used: per band (len + 1) entries at IB[b] + b
  for (uint32_t b = threadIdx.x; b < nb; b += THREADS) {
    const uint32_t jb = wk.IB[b];
    const uint64_t* Pb = P + jb;
    const ArrayLis<IdxT> lis{MINI + jb + b, wk.PD + jb};
    const bool strand = G[jb] & 1;
    const uint32_t longest =
        BandLis(wk.IE[b] - jb, strand, cp.chain, [&](uint32_t t) { return Pb[t]; }, lis);
    uint32_t emitted = 0;
    ForEachChainOverlap(longest, strand, cp, [&](uint32_t x) { return Pb[lis.minimal[x]]; },
                        [&](uint64_t, uint64_t, uint32_t) { ++emitted; });
    wk.CNT[b] = emitted;
    wk.IE[b] = static_cast<IdxT>(longest);  // the chain length, for the writer
  }
  __syncthreads();

  // 6. place the overlaps of all bands in band order
  uint32_t carry = 0;
  __shared__ uint32_t sh_total;
  // first pass: total
  {
    uint32_t local = 0;
    for (uint32_t b = threadIdx.x; b < nb; b += THREADS) local += wk.CNT[b];
    uint32_t tot;
    BlockExclusiveSum<uint32_t, THREADS>(local, sm32, &tot);
    if (threadIdx.x == 0) {
      sh_total = tot;
      sh_base = tot ? atomicAdd(ovl_counter, static_cast<unsigned long long>(tot))
                    : 0ULL;
    }
    __syncthreads();
  }
  const uint32_t total = sh_total;
  const uint64_t base = sh_base;
  *out_base = base;
  if (total == 0 || base + total > ovl_cap) return total;

  for (uint32_t b0 = 0; b0 < nb; b0 += THREADS) {
    const uint32_t b = b0 + threadIdx.x;
    const uint32_t mine = b < nb ? wk.CNT[b] : 0;
    uint32_t tot;
    const uint32_t ex = BlockExclusiveSum<uint32_t, THREADS>(mine, sm32, &tot);
    if (mine) {
      rvn_overlap* dst = ovl_raw + base + carry + ex;
      // (pair-at-a-time callers: emission sequence number of every overlap)
      uint64_t* kdst = ovl_key ? ovl_key + base + carry + ex : nullptr;
      uint32_t seq = carry + ex;
      const uint32_t jb = wk.IB[b];
      const uint64_t* Pb = P + jb;
      const IdxT* chain = MINI + jb + b;
      const bool strand = G[jb] & 1;
      const uint32_t rhs_id = static_cast<uint32_t>(G[jb] & 0xFFFFFFFFu) >> 1;
      ForEachChainOverlap(wk.IE[b], strand, cp, [&](uint32_t x) { return Pb[chain[x]]; },
                          [&](uint64_t first, uint64_t last, uint32_t score) {
                            *dst++ = MakeOverlap(lhs_id, rhs_id, strand, cp.k, first, last,
                                                 score);
                            if (kdst) *kdst++ = key_hi | seq++;
                          });
    }
    carry += tot;
  }
  return total;
}

constexpr uint32_t kChainSmemCap = 65535;  // hits per read on the split path (16-bit offsets)
constexpr uint32_t kSplitMaxTable = 8192;  // pair hash table entries per read, at most
constexpr uint32_t kPairMaxHits = 8191;    // hits of one pair PairChainKernel holds on chip
constexpr uint32_t kThreadPairMax = 63;   // larger (rhs, strand) pairs get a CTA each

// ---------------------------------------------------------------------------
// Fast path, two kernels.
//
// Bands never span two (rhs_id, strand) pairs (group keys of different pairs
// differ by >= 2^30 > bandwidth), so the reference's per-query sort by group is
// not needed.
//  SplitKernel  one CTA per query read: the read's hits are split by pair with
//               a shared-memory hash table; pairs with < 4 hits (about half of
//               all hits: spurious key matches) are dropped on the spot; the
//               rest is written pair-contiguous to HBM with one descriptor per
//               pair, pairs of a read in ascending key order (= the reference's
//               emission order).
//  GroupChainKernel  ONE THREAD PER PAIR over all pairs of all reads, largest
//               pairs first (size-sorted, so the lanes of a warp carry similar
//               work and nothing waits at a barrier): ChainPairSerial (chain.cuh).
//               Overlaps go to a global list keyed (pair index, sequence number)
//               and are put back in emission order by a radix sort of the keys.
// ---------------------------------------------------------------------------
struct GroupDesc {
  uint32_t hit_off, cnt, gid, lhs_id;
};

struct SplitLayout {
  uint32_t hs, gpad;
  size_t hk, hc, gl, bytes;
};

__host__ __device__ inline SplitLayout MakeSplitLayout(uint32_t n) {
  SplitLayout L;
  // open addressing, never full: distinct pairs <= n < hs. (A smaller table
  // does fill up: a random key match drags in every read covering that locus,
  // so single-hit pairs are about as many as half the hits.)
  uint32_t hs = 64;
  while (hs < n + 1 && hs < kSplitMaxTable) hs <<= 1;
  L.hs = hs;  // (reads beyond 8191 hits: a full table sends the read to the generic path)
  uint32_t gpad = 2;
  while (gpad < n / 4 + 1 && gpad < hs) gpad <<= 1;
  L.gpad = gpad;
  size_t o = 0;
  L.hk = o; o += 4ULL * hs;
  L.hc = o; o += 4ULL * hs;
  L.gl = o; o += 8ULL * gpad;
  L.bytes = (o + 15) & ~size_t(15);
  return L;
}

__device__ __forceinline__ uint32_t HashGid(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

template <int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB)
SplitKernel(const uint64_t* __restrict__ h_grp, const uint64_t* __restrict__ h_pos,
            const uint64_t* __restrict__ read_hit_off,
            const uint32_t* __restrict__ lhs_ids,
            const uint32_t* __restrict__ read_list,
            unsigned long long* __restrict__ totals,  // [0] pairs, [1] kept hits
            GroupDesc* __restrict__ desc, uint32_t* __restrict__ desc_cnt,
            uint32_t* __restrict__ desc_idx, uint32_t* __restrict__ g_diag,
            uint64_t* __restrict__ g_pos, uint64_t* __restrict__ group_loc,
            uint32_t* __restrict__ fallback_list,
            unsigned int* __restrict__ fallback_cnt) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint32_t sm32[34];
  __shared__ uint32_t sh_bail;
  __shared__ unsigned long long sh_gbase, sh_hbase;
  const uint32_t r = read_list[blockIdx.x];
  const uint64_t hb = read_hit_off[r];
  const uint32_t n = static_cast<uint32_t>(read_hit_off[r + 1] - hb);
  const SplitLayout L = MakeSplitLayout(n);
  uint32_t* HK = reinterpret_cast<uint32_t*>(smem + L.hk);
  uint32_t* HC = reinterpret_cast<uint32_t*>(smem + L.hc);
  uint64_t* GL = reinterpret_cast<uint64_t*>(smem + L.gl);
  const uint32_t hmask = L.hs - 1;
  const uint64_t* hg = h_grp + hb;
  const uint64_t* hp = h_pos + hb;

  // ---- hash table of (rhs_id, strand) pairs with their hit counts ----
  for (uint32_t i = threadIdx.x; i < L.hs; i += THREADS) {
    HK[i] = 0xFFFFFFFFu;
    HC[i] = 0;
  }
  if (threadIdx.x == 0) sh_bail = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n; i += THREADS) {
    const uint32_t gid = static_cast<uint32_t>(hg[i] >> 32);
    uint32_t s = HashGid(gid) & hmask;
    uint32_t probes = 0;
    while (true) {
      const uint32_t prev = atomicCAS(&HK[s], 0xFFFFFFFFu, gid);
      if (prev == 0xFFFFFFFFu || prev == gid) break;
      s = (s + 1) & hmask;
      if (++probes > hmask) {  // table full (only possible beyond 8191 hits)
        sh_bail = 1;
        break;
      }
    }
    if (probes <= hmask) atomicAdd(&HC[s], 1u);
  }
  __syncthreads();
  if (sh_bail) {  // more distinct pairs than the table holds: the generic kernel
    if (threadIdx.x == 0) fallback_list[atomicAdd(fallback_cnt, 1u)] = r;
    return;
  }

  // ---- pairs with >= 4 hits: list + offsets inside the read's kept hits ----
  uint32_t carry = 0;  // low 16: pairs so far, high 16: kept hits so far
  for (uint32_t b = 0; b < L.hs; b += THREADS) {
    const uint32_t s = b + threadIdx.x;
    const uint32_t cnt = s < L.hs ? HC[s] : 0;
    const uint32_t keep = cnt >= 4;
    if (cnt > kPairMaxHits) sh_bail = 1;  // (a pair PairChainKernel cannot hold on chip)
    uint32_t tot;
    const uint32_t ex = BlockExclusiveSum<uint32_t, THREADS>(
        keep ? ((cnt << 16) | 1u) : 0u, sm32, &tot);
    if (s < L.hs) {
      if (keep) {
        const uint32_t at = carry + ex;
        GL[at & 0xFFFF] = (static_cast<uint64_t>(HK[s]) << 32) | s;
        HC[s] = (cnt << 16) | (at >> 16);  // (count, offset)
      } else {
        HC[s] = 0xFFFFFFFFu;  // dropped
      }
    }
    carry += tot;
  }
  const uint32_t ng = carry & 0xFFFF, nh = carry >> 16;
  __syncthreads();
  if (sh_bail) {  // a very large pair: the generic kernel takes this read
    if (threadIdx.x == 0) fallback_list[atomicAdd(fallback_cnt, 1u)] = r;
    return;
  }
  if (ng == 0) {
    if (threadIdx.x == 0) group_loc[r] = 0;
    return;
  }

  // ---- pairs in ascending key order; reserve descriptor and hit space ----
  uint32_t gpad = 2;
  while (gpad < ng) gpad <<= 1;
  for (uint32_t i = ng + threadIdx.x; i < gpad; i += THREADS) GL[i] = ~0ULL;
  if (threadIdx.x == 0) {
    sh_gbase = atomicAdd(&totals[0], static_cast<unsigned long long>(ng));
    sh_hbase = atomicAdd(&totals[1], static_cast<unsigned long long>(nh));
  }
  __syncthreads();
  BitonicSort<THREADS>(gpad, [=](uint32_t i, uint32_t j, bool up) {
    const uint64_t a = GL[i], c2 = GL[j];
    if ((a > c2) == up) {
      GL[i] = c2;
      GL[j] = a;
    }
  });
  const uint64_t gbase = sh_gbase, hbase = sh_hbase;
  const uint32_t lhs_id = lhs_ids[r];
  for (uint32_t q = threadIdx.x; q < ng; q += THREADS) {
    const uint64_t e = GL[q];
    const uint32_t s = static_cast<uint32_t>(e);
    const uint32_t v = HC[s];
    GroupDesc d;
    d.hit_off = static_cast<uint32_t>(hbase) + (v & 0xFFFF);
    d.cnt = v >> 16;
    d.gid = static_cast<uint32_t>(e >> 32);
    d.lhs_id = lhs_id;
    desc[gbase + q] = d;
    desc_cnt[gbase + q] = d.cnt;
    desc_idx[gbase + q] = static_cast<uint32_t>(gbase + q);
    HC[s] = v & 0xFFFF;  // fill cursor
  }
  if (threadIdx.x == 0) group_loc[r] = (gbase << 24) | ng;
  __syncthreads();

  // ---- scatter the hits of kept pairs (order inside a pair is free) ----
  for (uint32_t i = threadIdx.x; i < n; i += THREADS) {
    const uint64_t g = hg[i];
    const uint32_t gid = static_cast<uint32_t>(g >> 32);
    uint32_t s = HashGid(gid) & hmask;
    while (HK[s] != gid) s = (s + 1) & hmask;
    if (HC[s] == 0xFFFFFFFFu) continue;
    const uint64_t at = hbase + atomicAdd(&HC[s], 1u);
    g_diag[at] = static_cast<uint32_t>(g);
    g_pos[at] = hp[i];
  }
}

// thread t of the launch handles pair order[first + t]; every pair of this launch has at
// most m_cap hits (the launch is one size class). A pair's hits live in shared memory,
// interleaved across the CTA's threads (element i of thread t at [i * T + t]): every
// thread walks its own column, same-index accesses of a warp are conflict-free, and no
// barrier is needed.
__global__ void GroupChainKernel(const GroupDesc* __restrict__ desc,
                                 const uint32_t* __restrict__ order, uint64_t first,
                                 uint64_t last, uint32_t m_cap,
                                 const uint32_t* __restrict__ g_diag,
                                 const uint64_t* __restrict__ g_pos, ChainParams cp,
                                 rvn_overlap* __restrict__ out,
                                 uint64_t* __restrict__ out_key,
                                 unsigned long long* __restrict__ out_cnt,
                                 uint64_t out_cap) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t T = blockDim.x;
  const uint64_t t = first + static_cast<uint64_t>(blockIdx.x) * T + threadIdx.x;
  if (t >= last) return;
  Column c;
  c.P = reinterpret_cast<uint64_t*>(smem) + threadIdx.x;
  c.D = reinterpret_cast<uint32_t*>(smem + 8ULL * m_cap * T) + threadIdx.x;
  c.T = T;
  const uint32_t g = order[t];
  const GroupDesc d = desc[g];
  for (uint32_t i = 0; i < d.cnt; ++i) {
    c.p(i) = g_pos[d.hit_off + i];
    c.d(i) = g_diag[d.hit_off + i];
  }
  const uint64_t key_hi = static_cast<uint64_t>(g) << 16;
  uint32_t seq = 0;
  ChainPairSerial(c, d.cnt, d.gid, d.lhs_id, cp, [&](const rvn_overlap& o) {
    const unsigned long long slot = atomicAdd(out_cnt, 1ULL);
    if (slot < out_cap) {
      out[slot] = o;
      out_key[slot] = key_hi | seq++;
    }
  });
}

// One CTA per (query, rhs, strand) pair with more than kThreadPairMax hits - the
// true overlaps, above all on HiFi reads where a pair holds hundreds of hits: the
// pair's hits live in shared memory, both orders come from parallel bitonic
// sorts and the bands from block scans (ChainRead); only the LIS of a band is one
// thread's work. CTA blockIdx.x handles pair order[first + blockIdx.x]; every
// pair of a launch has at most npad - 1 hits.
constexpr int kPairThreads = 64;

__host__ __device__ inline size_t PairChainSmem(uint32_t npad) {
  const uint32_t n = npad - 1, nb = n / 4 + 1;
  size_t o = 16ULL * npad;                        // G, P
  o += 2ULL * (n + nb + 2) + 2ULL * (n + 1) + 2ULL * 2 * nb;  // LB, PD, IB, IE (u16)
  o = (o + 3) & ~size_t(3);
  o += 4ULL * nb;                                 // CNT
  return (o + 15) & ~size_t(15);
}

__global__ void __launch_bounds__(kPairThreads)
PairChainKernel(const GroupDesc* __restrict__ desc, const uint32_t* __restrict__ order,
                uint64_t first, uint32_t npad, const uint32_t* __restrict__ g_diag,
                const uint64_t* __restrict__ g_pos, ChainParams cp,
                rvn_overlap* __restrict__ out, uint64_t* __restrict__ out_key,
                unsigned long long* __restrict__ out_cnt, uint64_t out_cap) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint32_t sm32[34];
  const uint32_t g = order[first + blockIdx.x];
  const GroupDesc d = desc[g];
  const uint32_t n = d.cnt;
  ChainWork<uint16_t> wk;
  wk.G = reinterpret_cast<uint64_t*>(smem);
  wk.P = wk.G + npad;
  wk.PlaceIndices(reinterpret_cast<uint16_t*>(wk.P + npad), npad - 1);
  // padding beyond the pair's hits sorts last (all ones), like the reference's dummy
  uint32_t np2 = 8;
  while (np2 < n + 1) np2 <<= 1;
  for (uint32_t i = threadIdx.x; i < np2; i += kPairThreads) {
    wk.G[i] = i < n ? (static_cast<uint64_t>(d.gid) << 32) | g_diag[d.hit_off + i] : ~0ULL;
    wk.P[i] = i < n ? g_pos[d.hit_off + i] : ~0ULL;
  }
  __syncthreads();
  uint64_t base = 0;
  ChainRead<uint16_t, kPairThreads>(wk, n, np2, d.lhs_id, cp, sm32, out, out_cnt, out_cap, &base,
                                    out_key, static_cast<uint64_t>(g) << 16);
}

// first index of a descending-sorted count array with count <= bound[i]
__global__ void SizeClassStarts(const uint32_t* __restrict__ sorted_cnt, uint64_t n,
                                const uint32_t* __restrict__ bound, uint32_t n_bounds,
                                uint64_t* __restrict__ start) {
  const uint32_t i = threadIdx.x;
  if (i >= n_bounds) return;
  const uint32_t bnd = bound[i];
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (sorted_cnt[mid] > bnd) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  start[i] = lo;
}

__global__ void IotaU32(uint32_t* __restrict__ out, uint64_t n) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<uint32_t>(i);
}

__global__ void GatherOverlapsByIndex(const rvn_overlap* __restrict__ src,
                                      const uint32_t* __restrict__ idx, uint64_t n,
                                      rvn_overlap* __restrict__ dst) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n * 2) return;
  const uint4* s = reinterpret_cast<const uint4*>(src);
  reinterpret_cast<uint4*>(dst)[i] = s[static_cast<uint64_t>(idx[i >> 1]) * 2 + (i & 1)];
}

// per listed read: where its overlaps sit in the key-sorted list
__global__ void LocateReadOverlaps(const uint64_t* __restrict__ sorted_key,
                                   uint64_t n_keys,
                                   const uint32_t* __restrict__ read_list,
                                   uint32_t n_list,
                                   const uint64_t* __restrict__ group_loc,
                                   uint64_t base0, uint64_t* __restrict__ ovl_loc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_list) return;
  const uint32_t r = read_list[i];
  const uint64_t gl = group_loc[r];
  const uint64_t gbase = gl >> 24, ng = gl & 0xFFFFFF;
  if (ng == 0) {
    ovl_loc[r] = 0;
    return;
  }
  auto lower = [&](uint64_t key) {
    uint64_t lo = 0, hi = n_keys;
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo) / 2;
      if (sorted_key[mid] < key) {
        lo = mid + 1;
      } else {
        hi = mid;
      }
    }
    return lo;
  };
  const uint64_t a = lower(gbase << 16), b = lower((gbase + ng) << 16);
  ovl_loc[r] = b > a ? ((base0 + a) << 24) | (b - a) : 0;
}

// global-memory path for reads with more hits than shared memory holds: one
// CTA per listed read, arrays in a scratch slab (u32 indices)
__global__ void __launch_bounds__(kThreads)
ChainKernelGlobal(const uint64_t* __restrict__ h_grp,
                  const uint64_t* __restrict__ h_pos,
                  const uint64_t* __restrict__ read_hit_off,
                  const uint32_t* __restrict__ lhs_ids,
                  const uint32_t* __restrict__ big_reads,
                  const uint64_t* __restrict__ slab64_off,
                  const uint64_t* __restrict__ slab32_off,
                  uint64_t* __restrict__ slab64, uint32_t* __restrict__ slab32,
                  ChainParams cp, rvn_overlap* __restrict__ ovl_raw,
                  unsigned long long* __restrict__ ovl_counter,
                  uint64_t ovl_cap, uint64_t* __restrict__ ovl_loc) {
  __shared__ uint32_t sm32[34];
  const uint32_t r = big_reads[blockIdx.x];
  const uint64_t hb = read_hit_off[r];
  const uint32_t n = static_cast<uint32_t>(read_hit_off[r + 1] - hb);
  uint32_t npad = 8;
  while (npad < n + 1) npad <<= 1;

  ChainWork<uint32_t> wk;
  wk.G = slab64 + slab64_off[blockIdx.x];
  wk.P = wk.G + npad;
  wk.PlaceIndices(slab32 + slab32_off[blockIdx.x], n);

  for (uint32_t i = threadIdx.x; i < npad; i += kThreads) {
    wk.G[i] = i < n ? h_grp[hb + i] : ~0ULL;
    wk.P[i] = i < n ? h_pos[hb + i] : ~0ULL;
  }
  __syncthreads();
  uint64_t base = 0;
  const uint32_t total = ChainRead<uint32_t, kThreads>(
      wk, n, npad, lhs_ids[r], cp, sm32, ovl_raw, ovl_counter, ovl_cap,
      &base);
  if (threadIdx.x == 0) ovl_loc[r] = total ? (base << 24) | total : 0;
}

__global__ void OverlapCounts(const uint64_t* __restrict__ ovl_loc, uint64_t n,
                              uint32_t* __restrict__ cnt) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) cnt[i] = static_cast<uint32_t>(ovl_loc[i] & 0xFFFFFF);
}

// move every read's overlaps from its reserved slab to query order
__global__ void ReorderOverlaps(const rvn_overlap* __restrict__ raw,
                                const uint64_t* __restrict__ ovl_loc,
                                const uint64_t* __restrict__ ovl_off,
                                uint32_t n_reads, rvn_overlap* __restrict__ out) {
  const uint32_t r = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (r >= n_reads) return;
  const uint64_t loc = ovl_loc[r];
  const uint32_t cnt = static_cast<uint32_t>(loc & 0xFFFFFF);
  const uint64_t src = loc >> 24, dst = ovl_off[r];
  const uint4* s = reinterpret_cast<const uint4*>(raw + src);
  uint4* d = reinterpret_cast<uint4*>(out + dst);
  for (uint32_t i = threadIdx.x & 31; i < cnt * 2; i += 32) d[i] = s[i];
}

// The self-join's slots for reads [first, i_last): one sweep per index (and occurrence
// threshold) serves all later flushes of the batch, which stage 1 runs in read order.
// Reads before `first` are left out: their flushes took the probe path, and their
// thresholds would cost a sketch of reads that are no longer sketched. The slot
// offsets are kept with the slots, as a flush over reads outside the batch replaces
// the micromizer counts (c.qt.h_off). Needs the thresholds t of reads [first, i_last): the
// batch's own (c.jt) after a chunked build, else c.qt.
void JoinSweep(Ctx& c, uint32_t first, const Thresholds& t) {
  const uint32_t nr = c.i_last - first;
  const uint64_t t0 = first - t.first, base = t.h_off[t0];
  c.h_j_off.resize(nr + 1ULL);
  for (uint32_t i = 0; i <= nr; ++i) c.h_j_off[i] = t.h_off[t0 + i] - base;
  const uint64_t n_q = c.h_j_off[nr];
  uint64_t* off = c.j_off.reserve(nr + 1ULL);
  RVN_CUDA(cudaMemcpyAsync(off, c.h_j_off.data(), (nr + 1ULL) * sizeof(uint64_t),
                           cudaMemcpyHostToDevice, c.stream));
  uint32_t* cursor = c.j_cursor.reserve(nr + 1ULL);
  uint64_t* packed = c.j_packed.reserve(n_q + 1);
  RVN_CUDA(cudaMemsetAsync(cursor, 0, (nr + 1ULL) * sizeof(uint32_t), c.stream));
  RVN_CUDA(cudaMemsetAsync(packed, 0, (n_q + 1) * sizeof(uint64_t), c.stream));
  if (c.i_n > 0 && n_q > 0) {
    const IndexView ix = IndexOf(c);
    JoinView jv{ix.val, ix.org, ix.n, ix.occurrence, t.val.get() + t0, t.pos.get() + t0, first,
                c.i_last};
    JoinSweepKernel<<<CeilDiv(c.i_n, kThreads), kThreads, 0, c.stream>>>(jv, off, cursor,
                                                                          packed);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));  // (h_j_off staging)
  c.j_gen = c.i_gen;
  c.j_occurrence = c.occurrence;
  c.j_first = first;
}

struct HitCounts {
  uint64_t n_q = 0, n_hits = 0;  // query records, seed hits
};

// Per-read hit ranges of the range's nr reads: read_hit_off[i] = hit_off[read_off[i] -
// q_begin] for i in [0, nr], on the device and in h_rho.
void ReadHitRanges(Ctx& c, const uint64_t* hit_off, const uint64_t* read_off, uint64_t q_begin,
                   uint32_t nr, uint64_t* read_hit_off, std::vector<uint64_t>& h_rho) {
  GatherU64<<<CeilDiv(nr + 1ULL, kThreads), kThreads, 0, c.stream>>>(
      hit_off, read_off, q_begin, nr + 1ULL, read_hit_off);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  RVN_CUDA(cudaMemcpyAsync(h_rho.data(), read_hit_off, (nr + 1ULL) * sizeof(uint64_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

// Stage-1 hits of reads [first, last) inside the index batch, by the self-join: the
// sweep if the slots are stale, then this range's slice of the slots is scanned and
// expanded into c.h_grp / c.h_pos.
HitCounts JoinHits(Ctx& c, uint32_t first, uint32_t last, uint64_t* read_hit_off,
                   std::vector<uint64_t>& h_rho) {
  const uint32_t nr = last - first;
  HitCounts h;
  const bool sweep = c.j_gen != c.i_gen || c.j_occurrence != c.occurrence || first < c.j_first;
  const bool batch = c.jt_gen == c.i_gen;
  if (sweep && !batch && !c.qt.Covers(first, c.i_last)) {
    EnsureThresholds(c, first, c.i_last);  // (its sketch and micromize time are not probe's)
  }
  TimerBegin(c, "probe");
  if (sweep) JoinSweep(c, first, batch ? c.jt : c.qt);
  const uint64_t b0 = first - c.j_first;
  const uint64_t q_begin = c.h_j_off[b0];
  h.n_q = c.h_j_off[b0 + nr] - q_begin;
  const uint64_t* packed = c.j_packed.get() + q_begin;
  uint64_t* hit_off = c.m_hit_off.reserve(h.n_q + 2);
  if (h.n_q > 0) {
    uint32_t* cnt = c.m_cnt.reserve(h.n_q + 1);
    UnpackJoin<<<CeilDiv(h.n_q, kThreads), kThreads, 0, c.stream>>>(packed, h.n_q, cnt);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    ExclusiveScanU32(c, cnt, hit_off, h.n_q);
    h.n_hits = ReadU64(c, hit_off + h.n_q);
  } else {
    RVN_CUDA(cudaMemsetAsync(hit_off, 0, sizeof(uint64_t), c.stream));
  }
  TimerEnd(c);
  TimerBegin(c, "expand");
  uint64_t* hg = c.h_grp.reserve(h.n_hits + 1);
  uint64_t* hp = c.h_pos.reserve(h.n_hits + 1);
  if (h.n_hits > 0) {
    ExpandJoinKernel<<<CeilDiv(h.n_q, kThreads), kThreads, 0, c.stream>>>(
        c.i_org.get(), packed, h.n_q, hit_off, hg, hp);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  ReadHitRanges(c, hit_off, c.j_off.get() + b0, q_begin, nr, read_hit_off, h_rho);
  TimerEnd(c);
  c.r_filt_off.reserve(nr + 2ULL);
  for (uint32_t i = 0; i <= nr; ++i) c.r_filt_off.get()[i] = 0;
  return h;
}

// Positions of the over-frequent query minimizers (filt) of the range's nr reads, in
// sketch order: c.r_filtered, and per-read offsets into it in c.r_filt_off.
void FilteredPositions(Ctx& c, const uint8_t* filt, const uint64_t* qo, uint64_t q_begin,
                       uint64_t n_q, const uint64_t* read_off, uint32_t nr) {
  uint32_t* f32 = c.m_first.get();  // `first` is dead after ExpandKernel
  FilteredFlagsToU32<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
      filt, n_q, f32);
  uint64_t* fpos = c.m_filt_off.reserve(n_q + 2);
  ExclusiveScanU32(c, f32, fpos, n_q);
  const uint64_t n_filtered = ReadU64(c, fpos + n_q);
  uint32_t* fout = c.m_filtered.reserve(n_filtered + 1);
  ScatterFiltered<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
      filt, fpos, qo, q_begin, n_q, fout);
  RVN_LAUNCH_CHECK();
  c.launches += 2;
  // per-read offsets of the filtered list
  uint64_t* froff = c.m_filtered_off.reserve(nr + 2ULL);
  GatherU64<<<CeilDiv(nr + 1ULL, kThreads), kThreads, 0, c.stream>>>(
      fpos, read_off, q_begin, nr + 1ULL, froff);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  c.m_n_filtered = n_filtered;
  if (!c.m_filtered_host) return;  // (stage 2 consumes them on the device)
  uint32_t* hf = c.r_filtered.reserve(n_filtered + 1);
  RVN_CUDA(cudaMemcpyAsync(hf, fout, n_filtered * sizeof(uint32_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(c.r_filt_off.get(), froff,
                           (nr + 1ULL) * sizeof(uint64_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

// Hits of reads [first, last) by probing the index with their query records (the
// micromizers with minhash, else the full sketch) into c.h_grp / c.h_pos, and the
// filtered positions if wanted (stage 2).
HitCounts ProbeHits(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal,
                    bool avoid_symmetric, bool minhash, bool want_filtered,
                    uint64_t* read_hit_off, std::vector<uint64_t>& h_rho) {
  const uint32_t nr = last - first;
  HitCounts h;
  // ---- query records ----
  const RecordSet& q = minhash ? c.mm : c.sk;
  if (minhash && !q.Covers(first, last)) EnsureMicromizers(c, first, last);
  if (!minhash && !q.Covers(first, last)) EnsureSketch(c, first, last);
  const ValView qv = q.Values();  // query values: u32 for full sketches of k <= 15, else u64
  const uint64_t* qo = q.org.get();
  const uint64_t off_base_read = first - q.first;  // index of `first` inside the offsets arrays
  const uint64_t* d_read_off = q.off.get();
  const uint64_t q_begin = q.h_off[off_base_read];
  const uint64_t n_q = q.h_off[off_base_read + nr] - q_begin;
  h.n_q = n_q;

  const IndexView ix = IndexOf(c);

  // ---- probe + expand ----
  TimerBegin(c, "probe");
  uint32_t* cnt = c.m_cnt.reserve(n_q + 1);
  uint32_t* frst = c.m_first.reserve(n_q + 1);
  uint8_t* filt = c.m_filt.reserve(n_q + 1);
  uint64_t* hit_off = c.m_hit_off.reserve(n_q + 2);
  // kept postings = a suffix of the run (or the whole run): see ProbeSuffix
  const bool suffix = (avoid_equal && avoid_symmetric && c.i_sorted_ids) ||
                      (!avoid_equal && !avoid_symmetric);
  if (n_q > 0) {
    if (suffix && n_q >= (1u << 16) && n_q < 0xFFFFFFFFULL) {
      // sort the queries by value, probe in that order, results back by index
      uint64_t* k1 = c.m_sq_key.reserve(n_q + 2);
      uint64_t* k2 = c.m_sq_key2.reserve(n_q);
      uint32_t* v1 = c.m_sq_idx.reserve(n_q);
      uint32_t* v2 = c.m_sq_idx2.reserve(n_q);
      IotaU32<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(v1, n_q);
      // FULL value order: consecutive probes then walk consecutive buckets, values
      // and postings (the reads of a warp fall into a few hundred bytes instead of
      // one 32-byte sector per probe per array)
      const int hi_bit = static_cast<int>(2 * c.prm.k);
      int w_q;
      ValView sorted_qv;
      if (qv.is32) {
        const uint32_t* src = static_cast<const uint32_t*>(qv.p) + q_begin;
        uint32_t* a32 = reinterpret_cast<uint32_t*>(k1);
        uint32_t* b32 = a32 + n_q + (n_q & 1);  // second half of k1 (8-byte aligned)
        w_q = RadixSortPairs(c, src, a32, b32, v1, v2, v1, n_q, 0, hi_bit);
        sorted_qv = ValView{w_q < 0 ? src : (w_q == 0 ? a32 : b32), 1};
      } else {
        const uint64_t* src = static_cast<const uint64_t*>(qv.p) + q_begin;
        w_q = RadixSortPairs(c, src, k1, k2, v1, v2, v1, n_q, 0, hi_bit);
        sorted_qv = ValView{w_q < 0 ? src : (w_q == 0 ? k1 : k2), 0};
      }
      const uint32_t* sorted_qi = w_q == 0 ? v2 : v1;
      // (a key buffer the sort did not end in receives the packed results)
      uint64_t* packed = (qv.is32 || w_q == 0) ? k2 : k1;
      ProbeSortedKernel<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
          ix, sorted_qv, sorted_qi, qo, q_begin, n_q, avoid_equal, packed);
      UnpackProbe<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(packed, n_q, cnt, frst, filt);
      c.launches += (2 * c.prm.k + 7) / 8 + 5;
    } else if (suffix) {
      ProbeSuffixKernel<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
          ix, qv, qo, q_begin, n_q, avoid_equal, cnt, frst, filt);
    } else {
      ProbeKernel<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
          ix, qv, qo, q_begin, n_q, avoid_equal, avoid_symmetric, cnt, frst, filt);
    }
    RVN_LAUNCH_CHECK();
    ++c.launches;
    ExclusiveScanU32(c, cnt, hit_off, n_q);
    h.n_hits = ReadU64(c, hit_off + n_q);
  } else {
    RVN_CUDA(cudaMemsetAsync(hit_off, 0, sizeof(uint64_t), c.stream));
  }
  TimerEnd(c);
  TimerBegin(c, "expand");
  uint64_t* hg = c.h_grp.reserve(h.n_hits + 1);
  uint64_t* hp = c.h_pos.reserve(h.n_hits + 1);
  if (h.n_hits > 0) {
    if (suffix) {
      ExpandWarpKernel<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
          ix, qo, q_begin, n_q, cnt, frst, hit_off, hg, hp);
    } else {
      ExpandKernel<<<CeilDiv(n_q, kThreads), kThreads, 0, c.stream>>>(
          ix, qv, qo, q_begin, n_q, avoid_equal, avoid_symmetric, cnt, frst,
          hit_off, hg, hp);
    }
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  ReadHitRanges(c, hit_off, d_read_off + off_base_read, q_begin, nr, read_hit_off, h_rho);
  TimerEnd(c);

  c.r_filt_off.reserve(nr + 2ULL);
  for (uint32_t i = 0; i <= nr; ++i) c.r_filt_off.get()[i] = 0;
  c.m_n_filtered = 0;
  if (want_filtered && n_q > 0) {
    FilteredPositions(c, filt, qo, q_begin, n_q, d_read_off + off_base_read, nr);
  }
  return h;
}

// read size classes of the split path: n hits take the first class with n + 1 <= bound
constexpr uint32_t kSplitBounds[] = {256, 512, 1024, 2048, 4096, 8192, 65536};
constexpr int kSplitClasses = sizeof(kSplitBounds) / sizeof(kSplitBounds[0]);
// pair size classes, descending: one launch chains the pairs with
// kPairBounds[b + 1] < hits <= kPairBounds[b]; a CTA per pair (PairChainKernel, shared
// memory by class) above kThreadPairMax, a thread per pair from there on
// (GroupChainKernel: shared memory per CTA = threads x class bound x 12 B)
constexpr uint32_t kPairBounds[] = {8191, 4095, 2047, 1023, 511, 255, 127,
                                    kThreadPairMax, 48, 32, 24, 16, 8};
constexpr uint32_t kPairClasses = sizeof(kPairBounds) / sizeof(kPairBounds[0]);
constexpr uint32_t kFirstThreadClass = 7;
static_assert(kPairBounds[kFirstThreadClass] == kThreadPairMax,
              "pairs of up to kThreadPairMax hits get a thread each");
constexpr int kGroupSmemLimit = 200 * 1024;        // GroupChainKernel's dynamic shared memory
constexpr uint64_t kGroupSmemBudget = 196 * 1024;  // what one of its CTAs may take

struct ReadRoutes {
  std::vector<uint32_t> split[kSplitClasses];  // the split path, by size class
  std::vector<uint32_t> global;                // the global-memory path (ChainKernelGlobal)
};

// Where each read is chained: reads beyond kChainSmemCap hits, and all reads when
// chain < 1, on the global-memory path, the others on the split path. Reads of fewer
// than 4 hits form no band and go nowhere (their ovl_loc stays 0).
ReadRoutes ClassifyReads(const std::vector<uint64_t>& h_rho, uint32_t nr, bool split_ok) {
  ReadRoutes r;
  for (uint32_t i = 0; i < nr; ++i) {
    const uint64_t n = h_rho[i + 1] - h_rho[i];
    if (n < 4) continue;
    if (n > kChainSmemCap || !split_ok) {
      r.global.push_back(i);
      continue;
    }
    int k = 0;
    while (kSplitBounds[k] < n + 1) ++k;
    r.split[k].push_back(i);
  }
  return r;
}

// the split path's pairs: descriptors, and their hits pair-contiguous
struct PairSplit {
  const uint32_t* d_list;  // the split reads on the device, largest size class first
  uint32_t n_reads;
  GroupDesc* desc;
  uint32_t *dcnt, *didx, *g_diag;
  uint64_t *g_pos, *group_loc;
  uint64_t n_groups;
};

// Splits the hits of the split path's reads by pair (SplitKernel, one launch per size
// class, largest first). The reads SplitKernel hands back - more distinct pairs than
// its table holds, or a pair of more than kPairMaxHits hits - join routes.global in
// read order. counter[1] and [2] count the pairs and their hits.
PairSplit SplitPairs(Ctx& c, const uint64_t* hg, const uint64_t* hp,
                     const uint64_t* read_hit_off, const uint32_t* lhs_ids, ReadRoutes& routes,
                     uint32_t nr, uint64_t n_hits, uint64_t n_q, uint64_t* counter) {
  PairSplit s{};
  std::vector<uint32_t> list;
  for (int k = kSplitClasses - 1; k >= 0; --k) {
    list.insert(list.end(), routes.split[k].begin(), routes.split[k].end());
  }
  s.n_reads = static_cast<uint32_t>(list.size());
  uint32_t* d_list = c.m_first.reserve(std::max<size_t>(list.size(), n_q) + 1);
  s.d_list = d_list;
  uint32_t* d_fb = c.m_fallback.reserve(nr + 4ULL);
  RVN_CUDA(cudaMemsetAsync(d_fb, 0, 2 * sizeof(uint32_t), c.stream));
  if (list.empty()) return s;
  RVN_CUDA(cudaMemcpyAsync(d_list, list.data(), list.size() * sizeof(uint32_t),
                           cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));  // (list goes out of scope)

  const uint64_t max_groups = n_hits / 4 + 1;
  s.desc = reinterpret_cast<GroupDesc*>(c.m_desc.reserve(max_groups * (sizeof(GroupDesc) / 4)));
  s.dcnt = c.m_desc_cnt.reserve(max_groups);
  s.didx = c.m_desc_idx.reserve(max_groups);
  s.g_diag = c.m_gdiag.reserve(n_hits + 1);
  s.g_pos = c.m_gpos.reserve(n_hits + 1);
  c.m_desc_cnt2.reserve(max_groups);  // (ChainPairs' sort buffers)
  c.m_desc_idx2.reserve(max_groups);
  s.group_loc = c.m_group_loc.reserve(nr + 1ULL);
  // counters: [0] overlaps (global-memory path), [1] pairs, [2] kept hits,
  // [3] overlaps of the pairs
  RVN_CUDA(cudaMemsetAsync(counter, 0, 4 * sizeof(uint64_t), c.stream));
  auto* ctr = reinterpret_cast<unsigned long long*>(counter);
  size_t off = 0;
  for (int k = kSplitClasses - 1; k >= 0; --k) {  // largest class first
    const unsigned cnt = static_cast<unsigned>(routes.split[k].size());
    if (cnt == 0) continue;
    const size_t smem = MakeSplitLayout(kSplitBounds[k] - 1).bytes;
    const uint32_t* lst = d_list + off;
    off += cnt;
    const bool wide = kSplitBounds[k] > 2048;
    auto kern = wide ? SplitKernel<256, 2> : SplitKernel<128, 8>;
    if (wide) {
      RVN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    static_cast<int>(MakeSplitLayout(kChainSmemCap).bytes)));
    }
    kern<<<cnt, wide ? 256 : 128, smem, c.stream>>>(hg, hp, read_hit_off, lhs_ids, lst, ctr + 1,
                                                    s.desc, s.dcnt, s.didx, s.g_diag, s.g_pos,
                                                    s.group_loc, d_fb + 2, d_fb);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  // pair count, reads handed back
  uint64_t* hpin = c.pin64.reserve(8);
  RVN_CUDA(cudaMemcpyAsync(hpin, counter, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                           c.stream));
  std::vector<uint32_t> fb(2);
  RVN_CUDA(cudaMemcpyAsync(fb.data(), d_fb, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                           c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  s.n_groups = hpin[1];
  const uint32_t nfb = fb[0];
  if (nfb) {
    fb.resize(nfb);
    RVN_CUDA(cudaMemcpyAsync(fb.data(), d_fb + 2, nfb * sizeof(uint32_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    std::sort(fb.begin(), fb.end());
    routes.global.insert(routes.global.end(), fb.begin(), fb.end());
  }
  if (s.n_groups >= 0xFFFFFFFFULL) throw LimitError("2^32 or more seed pairs");
  // GroupDesc::hit_off is 32 bits wide
  if (hpin[2] >= 0xFFFFFFFFULL) throw LimitError("2^32 or more chained seed hits in one flush");
  return s;
}

// Chains every pair, largest first (a stable descending radix sort of the pair sizes,
// so that the lanes of a warp get pairs of similar size), one launch per size class of
// kPairBounds. The overlaps land in c.m_ovl_tmp in any order, keyed (pair index,
// sequence number) in c.m_okey; returns their number.
uint64_t ChainPairs(Ctx& c, const PairSplit& s, const ChainParams& cp, uint64_t ovl_cap,
                    uint64_t* counter) {
  uint32_t* dcnt2 = c.m_desc_cnt2.get();
  uint32_t* didx2 = c.m_desc_idx2.get();
  const int w_desc = RadixSortPairs(c, s.dcnt, dcnt2, s.dcnt, s.didx, didx2, s.didx, s.n_groups,
                                    0, 13, /*descending=*/true);
  const uint32_t* sorted_cnt = w_desc == 0 ? dcnt2 : s.dcnt;
  const uint32_t* sorted_idx = w_desc == 0 ? didx2 : s.didx;
  rvn_overlap* tmp_ovl = c.m_ovl_tmp.reserve(ovl_cap);
  uint64_t* key = c.m_okey.reserve(ovl_cap);
  uint32_t* d_bounds = c.m_bounds.reserve(kPairClasses);
  uint64_t* d_starts = c.m_starts.reserve(kPairClasses + 1);
  RVN_CUDA(cudaMemcpyAsync(d_bounds, kPairBounds, sizeof(kPairBounds), cudaMemcpyHostToDevice,
                           c.stream));
  SizeClassStarts<<<1, 32, 0, c.stream>>>(sorted_cnt, s.n_groups, d_bounds, kPairClasses,
                                          d_starts);
  uint64_t h_starts[kPairClasses + 1];
  RVN_CUDA(cudaMemcpyAsync(h_starts, d_starts, kPairClasses * sizeof(uint64_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  h_starts[kPairClasses] = s.n_groups;
  h_starts[0] = 0;  // (no pair of the split path has more than kPairMaxHits hits)
  RVN_CUDA(cudaFuncSetAttribute(GroupChainKernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kGroupSmemLimit));
  RVN_CUDA(cudaFuncSetAttribute(PairChainKernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(PairChainSmem(kPairMaxHits + 1))));
  auto* ctr = reinterpret_cast<unsigned long long*>(counter);
  for (uint32_t b = 0; b < kPairClasses; ++b) {
    const uint64_t lo = h_starts[b], hi = h_starts[b + 1];
    if (hi <= lo) continue;
    if (b < kFirstThreadClass) {
      const uint32_t npad = kPairBounds[b] + 1;
      PairChainKernel<<<static_cast<unsigned>(hi - lo), kPairThreads, PairChainSmem(npad),
                        c.stream>>>(s.desc, sorted_idx, lo, npad, s.g_diag, s.g_pos, cp, tmp_ovl,
                                    key, ctr + 3, ovl_cap);
    } else {
      uint32_t threads = 128;
      while (threads > 8 && 12ULL * kPairBounds[b] * threads > kGroupSmemBudget) threads >>= 1;
      const size_t smem = 12ULL * kPairBounds[b] * threads;
      GroupChainKernel<<<CeilDiv(hi - lo, threads), threads, smem, c.stream>>>(
          s.desc, sorted_idx, lo, hi, kPairBounds[b], s.g_diag, s.g_pos, cp, tmp_ovl, key,
          ctr + 3, ovl_cap);
    }
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  const uint64_t n_ovl = ReadU64(c, counter + 3);
  if (n_ovl > ovl_cap) throw LimitError("overlap slab overflow");
  if (n_ovl >= 0xFFFFFFFFULL) throw LimitError("2^32 or more overlaps");
  return n_ovl;
}

// Puts the n_ovl overlaps of ChainPairs in emission order = (pair index, sequence
// number) at the front of raw, and points each split read's ovl_loc at its own.
void OrderPairOverlaps(Ctx& c, const PairSplit& s, uint64_t n_ovl, uint64_t ovl_cap,
                       rvn_overlap* raw, uint64_t* loc) {
  uint64_t* key = c.m_okey.get();
  uint64_t* key2 = c.m_okey2.reserve(ovl_cap);
  uint32_t* oidx = c.m_oidx.reserve(ovl_cap);
  uint32_t* oidx2 = c.m_oidx2.reserve(ovl_cap);
  IotaU32<<<CeilDiv(n_ovl, kThreads), kThreads, 0, c.stream>>>(oidx, n_ovl);
  int key_bits = 17;
  while (key_bits < 64 && (1ULL << (key_bits - 16)) < s.n_groups) ++key_bits;
  const int w_ovl = RadixSortPairs(c, key, key2, key, oidx, oidx2, oidx, n_ovl, 0, key_bits);
  const uint64_t* sorted_key = w_ovl == 0 ? key2 : key;
  const uint32_t* sorted_oidx = w_ovl == 0 ? oidx2 : oidx;
  GatherOverlapsByIndex<<<CeilDiv(n_ovl * 2, kThreads), kThreads, 0, c.stream>>>(
      c.m_ovl_tmp.get(), sorted_oidx, n_ovl, raw);
  LocateReadOverlaps<<<CeilDiv(s.n_reads, kThreads), kThreads, 0, c.stream>>>(
      sorted_key, n_ovl, s.d_list, s.n_reads, s.group_loc, 0, loc);
  RVN_LAUNCH_CHECK();
  c.launches += 3;
}

// Chains the listed reads whole on the global-memory path (ChainKernelGlobal, a CTA
// per read over a scratch slab), appending to raw behind what counter[0] holds.
void ChainWholeReads(Ctx& c, const std::vector<uint32_t>& reads, const uint64_t* hg,
                     const uint64_t* hp, const uint64_t* read_hit_off,
                     const std::vector<uint64_t>& h_rho, const uint32_t* lhs_ids,
                     const ChainParams& cp, rvn_overlap* raw, uint64_t* counter,
                     uint64_t ovl_cap, uint64_t* loc) {
  if (reads.empty()) return;
  std::vector<uint64_t> off64(reads.size() + 1, 0), off32(reads.size() + 1, 0);
  for (size_t i = 0; i < reads.size(); ++i) {
    const uint64_t n = h_rho[reads[i] + 1] - h_rho[reads[i]];
    if (n >= 0x7FFFFFFFULL) throw LimitError("a query has 2^31 or more hits");
    uint64_t npad = 8;
    while (npad < n + 1) npad <<= 1;
    const uint64_t nbmax = n / 4 + 1;
    off64[i + 1] = off64[i] + 2 * npad;
    off32[i + 1] = off32[i] + (n + nbmax + 2) + (n + 1) + 3 * nbmax + 4;
  }
  uint64_t* slab64 = c.m_scratch64.reserve(off64.back() + 2 * (reads.size() + 1) + 8);
  uint32_t* slab32 = c.m_scratch32.reserve(off32.back() + reads.size() + 8);
  // offsets and the read list ride at the tail of the slabs
  uint64_t* d_off64 = slab64 + off64.back();
  uint64_t* d_off32 = d_off64 + reads.size() + 1;
  uint32_t* d_reads = slab32 + off32.back();
  RVN_CUDA(cudaMemcpyAsync(d_off64, off64.data(), (reads.size() + 1) * 8,
                           cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_off32, off32.data(), (reads.size() + 1) * 8,
                           cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_reads, reads.data(), reads.size() * 4, cudaMemcpyHostToDevice,
                           c.stream));
  ChainKernelGlobal<<<static_cast<unsigned>(reads.size()), kThreads, 0, c.stream>>>(
      hg, hp, read_hit_off, lhs_ids, d_reads, d_off64, d_off32, slab64, slab32, cp, raw,
      reinterpret_cast<unsigned long long*>(counter), ovl_cap, loc);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  RVN_CUDA(cudaStreamSynchronize(c.stream));  // host vectors go out of scope
}

// Moves every read's overlaps from where raw holds them (ovl_loc) to query order in
// c.m_ovl / c.m_ovl_off; returns their number.
uint64_t ApplyQueryOrder(Ctx& c, const rvn_overlap* raw, const uint64_t* loc, uint32_t nr,
                         uint64_t ovl_cap) {
  uint32_t* ocnt = c.m_cnt.reserve(nr + 1ULL);
  uint64_t* ooff = c.m_ovl_off.reserve(nr + 2ULL);
  uint64_t n_ovl = 0;
  if (nr > 0) {
    OverlapCounts<<<CeilDiv(nr, kThreads), kThreads, 0, c.stream>>>(loc, nr, ocnt);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    ExclusiveScanU32(c, ocnt, ooff, nr);
    n_ovl = ReadU64(c, ooff + nr);
  } else {
    RVN_CUDA(cudaMemsetAsync(ooff, 0, sizeof(uint64_t), c.stream));
  }
  if (n_ovl > ovl_cap) throw LimitError("overlap slab overflow");
  rvn_overlap* ordered = c.m_ovl.reserve(n_ovl + 1);
  if (n_ovl > 0) {
    ReorderOverlaps<<<CeilDiv(nr, kThreads / 32), kThreads, 0, c.stream>>>(raw, loc, ooff, nr,
                                                                          ordered);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  return n_ovl;
}

}  // namespace

// Chains hits that are already grouped by query read: hits of read i of the
// range are h_grp/h_pos[read_hit_off[i] .. read_hit_off[i+1]) (any order inside
// a read). Leaves the overlaps in query order in c.m_ovl / c.m_ovl_off.
uint64_t ChainGroupedHits(Ctx& c, const uint64_t* hg, const uint64_t* hp,
                          const uint64_t* read_hit_off,
                          const std::vector<uint64_t>& h_rho, const uint32_t* lhs_ids,
                          uint32_t nr, uint64_t n_hits, uint64_t n_q) {
  TimerBegin(c, "chain");
  ChainParams cp{c.prm.k, c.prm.bandwidth, c.prm.chain, c.prm.matches, c.prm.gap};
  const uint64_t ovl_cap = n_hits / std::max(1u, std::min(c.prm.chain, 4u)) + 16;
  rvn_overlap* raw = c.m_ovl_raw.reserve(ovl_cap);
  uint64_t* loc = c.m_ovl_loc.reserve(nr + 1ULL);
  uint64_t* counter = c.m_counter.reserve((1u << 16) + 8);
  RVN_CUDA(cudaMemsetAsync(counter, 0, sizeof(uint64_t), c.stream));
  RVN_CUDA(cudaMemsetAsync(loc, 0, (nr + 1ULL) * sizeof(uint64_t), c.stream));

  ReadRoutes routes = ClassifyReads(h_rho, nr, c.prm.chain >= 1);
  const PairSplit s =
      SplitPairs(c, hg, hp, read_hit_off, lhs_ids, routes, nr, n_hits, n_q, counter);
  if (s.n_reads) {
    uint64_t n_pair_ovl = 0;
    if (s.n_groups) {
      n_pair_ovl = ChainPairs(c, s, cp, ovl_cap, counter);
      if (n_pair_ovl) OrderPairOverlaps(c, s, n_pair_ovl, ovl_cap, raw, loc);
    }
    // the global-memory path appends behind the pairs' overlaps
    RVN_CUDA(cudaMemcpyAsync(counter, &n_pair_ovl, sizeof(uint64_t), cudaMemcpyHostToDevice,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  }
  ChainWholeReads(c, routes.global, hg, hp, read_hit_off, h_rho, lhs_ids, cp, raw, counter,
                  ovl_cap, loc);
  const uint64_t n_ovl = ApplyQueryOrder(c, raw, loc, nr, ovl_cap);
  TimerEnd(c);
  return n_ovl;
}

void MapRange(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal,
              bool avoid_symmetric, bool minhash, bool want_filtered,
              bool fetch) {
  if (!c.i_valid) throw StateError("Map before Minimize");
  c.r_valid = false;
  const uint32_t nr = last - first;

  // ---- seed hits: self-join for stage 1 with the query reads inside the index
  // batch, else probes of the index ----
  const bool join = c.self_join && minhash && avoid_equal && avoid_symmetric && !want_filtered &&
                    c.i_from_sketch && c.i_sorted_ids && c.ids_identity && first >= c.i_first &&
                    last <= c.i_last;
  uint64_t* read_hit_off = c.m_read_hit_off.reserve(nr + 2ULL);
  std::vector<uint64_t> h_rho(nr + 1ULL);  // read_hit_off on the host
  const HitCounts h =
      join ? JoinHits(c, first, last, read_hit_off, h_rho)
           : ProbeHits(c, first, last, avoid_equal, avoid_symmetric, minhash, want_filtered,
                       read_hit_off, h_rho);
  const uint64_t n_q = h.n_q, n_hits = h.n_hits;
  const uint64_t* hg = c.h_grp.get();
  const uint64_t* hp = c.h_pos.get();

  if (c.keep_hits) {
    uint64_t* g = c.r_hit_grp.reserve(n_hits + 1);
    uint64_t* p = c.r_hit_pos.reserve(n_hits + 1);
    uint64_t* o = c.r_hit_off.reserve(nr + 2ULL);
    RVN_CUDA(cudaMemcpyAsync(g, hg, n_hits * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(p, hp, n_hits * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    for (uint32_t i = 0; i <= nr; ++i) o[i] = h_rho[i];
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    c.r_n_hits = n_hits;
  }

  // ---- chain ----
  const uint64_t n_ovl =
      ChainGroupedHits(c, hg, hp, read_hit_off, h_rho, c.d_ids.get() + first, nr, n_hits, n_q);
  const rvn_overlap* ordered = c.m_ovl.get();
  const uint64_t* ooff = c.m_ovl_off.get();

  // ---- results to the host ----
  if (fetch) {
    rvn_overlap* ho = c.r_ovl.reserve(n_ovl + 1);
    uint64_t* hoff = c.r_ovl_off.reserve(nr + 2ULL);
    RVN_CUDA(cudaMemcpyAsync(ho, ordered, n_ovl * sizeof(rvn_overlap),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(hoff, ooff, (nr + 1ULL) * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  }
  c.r_n_ovl = n_ovl;
  c.m_hits = n_hits;
  c.m_first_read = first;
  c.m_last_read = last;
  c.r_valid = fetch;

  c.stats.query_bases += ReadBases(c, first, last);
  c.stats.query_records += n_q;
  c.stats.hits += n_hits;
  c.stats.overlaps += n_ovl;
}

}  // namespace rvn
