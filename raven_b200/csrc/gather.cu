// raven_b200 — per-read overlap lists on the device: gather + truncation.
//
// Replaces the serial gather and the per-pile truncation tasks of
// raven::FindOverlapsAndCreatePiles (RavenLib/src/construct.cc:72-78,87-109):
//     for every mapped overlap o, in query order:
//         overlaps[o.lhs_id].push_back(o); overlaps[o.rhs_id].push_back(reverse(o))
//     for every list that grew: if size >= kMax: std::sort by length desc,
//         keep the first kMax
// On the device the arrival order of a read's new records is reconstructed
// without any serial pass: all records where the read is the rhs come from
// earlier queries (lhs_id < rhs_id), ordered by overlap index, followed by the
// read's own query block. A stable radix sort of overlap indices by rhs_id
// gives the first part, the block offset the second. The truncation replays
// libstdc++'s std::sort (introsort.cuh), one thread per read.

#include "engine.cuh"
#include "introsort.cuh"

namespace rvn {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ rvn_overlap ReverseOverlap(const rvn_overlap& o) {
  rvn_overlap r;  // overlap_utils.cc:5-8
  r.lhs_id = o.rhs_id;
  r.lhs_begin = o.rhs_begin;
  r.lhs_end = o.rhs_end;
  r.rhs_id = o.lhs_id;
  r.rhs_begin = o.lhs_begin;
  r.rhs_end = o.lhs_end;
  r.score = o.score;
  r.strand = o.strand;
  return r;
}

__device__ __forceinline__ uint32_t OverlapLength(const rvn_overlap& o) {
  const uint32_t a = o.rhs_end - o.rhs_begin, b = o.lhs_end - o.lhs_begin;
  return a > b ? a : b;  // overlap_utils.cc:10-12
}

__global__ void RhsKeys(const rvn_overlap* __restrict__ ovl, uint32_t m, Window w,
                        uint32_t* __restrict__ key, uint32_t* __restrict__ idx,
                        uint32_t* __restrict__ rhs_cnt) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  const uint32_t r = w.Slot(ovl[e].rhs_id);
  key[e] = r;
  idx[e] = e;
  atomicAdd(&rhs_cnt[r], 1u);
}

// total[s] = kept so far + new records as rhs + new records as lhs (query block)
// of the read in slot s
__global__ void ListTotals(const uint32_t* __restrict__ old_cnt,
                           const uint32_t* __restrict__ rhs_cnt,
                           const uint64_t* __restrict__ q_ovl_off, uint32_t k0,
                           uint32_t k1, Window w, uint32_t mod, uint32_t rem,
                           uint32_t* __restrict__ total) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= w.size()) return;
  const uint32_t r = w.Id(s);
  if (r % mod != rem) {  // not this context's read: its list stays empty
    total[s] = old_cnt[s];
    return;
  }
  uint32_t lhs = 0;
  if (r >= k0 && r < k1) {
    lhs = static_cast<uint32_t>(q_ovl_off[r - k0 + 1] - q_ovl_off[r - k0]);
  }
  total[s] = old_cnt[s] + rhs_cnt[s] + lhs;
}

// one warp per read: carry the kept records over into the staging list
__global__ void __launch_bounds__(kThreads)
CopyOld(const rvn_overlap* __restrict__ lists, const uint64_t* __restrict__ g_off,
        const uint32_t* __restrict__ old_cnt, const uint64_t* __restrict__ t_off,
        uint32_t n, rvn_overlap* __restrict__ stage) {
  const uint32_t r = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (r >= n) return;
  const uint32_t cnt = old_cnt[r];
  const uint4* s = reinterpret_cast<const uint4*>(lists + g_off[r]);
  uint4* d = reinterpret_cast<uint4*>(stage + t_off[r]);
  for (uint32_t i = threadIdx.x & 31; i < cnt * 2; i += 32) d[i] = s[i];
}

__global__ void PlaceRhs(const rvn_overlap* __restrict__ ovl,
                         const uint32_t* __restrict__ sorted_idx, uint32_t m,
                         const uint64_t* __restrict__ rhs_off,
                         const uint32_t* __restrict__ old_cnt,
                         const uint64_t* __restrict__ t_off, Window w, uint32_t mod,
                         uint32_t rem, rvn_overlap* __restrict__ stage) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const rvn_overlap o = ovl[sorted_idx[p]];
  if (o.rhs_id % mod != rem) return;
  const uint32_t r = w.Slot(o.rhs_id);
  const uint64_t rank = p - rhs_off[r];
  stage[t_off[r] + old_cnt[r] + rank] = ReverseOverlap(o);
}

__global__ void PlaceLhs(const rvn_overlap* __restrict__ ovl, uint32_t m,
                         const uint64_t* __restrict__ q_ovl_off, uint32_t k0,
                         const uint32_t* __restrict__ rhs_cnt,
                         const uint32_t* __restrict__ old_cnt,
                         const uint64_t* __restrict__ t_off, Window w, uint32_t mod,
                         uint32_t rem, rvn_overlap* __restrict__ stage) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  const rvn_overlap o = ovl[e];
  if (o.lhs_id % mod != rem) return;
  const uint32_t r = w.Slot(o.lhs_id);
  const uint64_t rank = e - q_ovl_off[o.lhs_id - k0];
  stage[t_off[r] + old_cnt[r] + rhs_cnt[r] + rank] = o;
}

// one thread per read: the reference's truncation rule on the staged list
__global__ void __launch_bounds__(128)
Truncate(const rvn_overlap* __restrict__ stage, const uint64_t* __restrict__ t_off,
         const uint32_t* __restrict__ total, const uint32_t* __restrict__ old_cnt,
         uint32_t n, uint64_t kmax, uint64_t* __restrict__ pairs,
         uint32_t* __restrict__ kept) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t s = total[r];
  const bool grew = s != old_cnt[r];
  if (!grew || s < kmax) {
    kept[r] = s;  // untouched lists are not re-sorted (construct.cc:81-85,94-96)
    return;
  }
  const uint64_t b = t_off[r];
  uint64_t* p = pairs + b;
  for (uint32_t i = 0; i < s; ++i) {
    p[i] = (static_cast<uint64_t>(OverlapLength(stage[b + i])) << 32) | i;
  }
  stdsort::Sort(p, p + s);
  kept[r] = static_cast<uint32_t>(kmax);
}

// one warp per read: staged list (in sorted order where it was sorted) ->
// compact persistent list
__global__ void __launch_bounds__(kThreads)
Compact(const rvn_overlap* __restrict__ stage, const uint64_t* __restrict__ t_off,
        const uint32_t* __restrict__ total, const uint32_t* __restrict__ old_cnt,
        const uint32_t* __restrict__ kept, const uint64_t* __restrict__ pairs,
        uint64_t kmax, const uint64_t* __restrict__ new_off, uint32_t n,
        rvn_overlap* __restrict__ lists) {
  const uint32_t r = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (r >= n) return;
  const uint32_t s = total[r], kp = kept[r];
  const bool sorted = s != old_cnt[r] && s >= kmax;
  const uint64_t b = t_off[r];
  const uint4* src = reinterpret_cast<const uint4*>(stage + b);
  uint4* dst = reinterpret_cast<uint4*>(lists + new_off[r]);
  for (uint32_t i = threadIdx.x & 31; i < kp * 2; i += 32) {
    const uint32_t rec = i >> 1;
    const uint32_t from = sorted ? static_cast<uint32_t>(pairs[b + rec]) : rec;
    dst[i] = src[from * 2 + (i & 1)];
  }
}

}  // namespace

void GatherReset(Ctx& c) {
  const uint32_t n = c.n_reads;
  c.g_cur = 0;
  c.g_total = 0;
  uint32_t* cnt = c.g_cnt.reserve(n + 1ULL);
  uint64_t* off = c.g_off.reserve(n + 2ULL);
  RVN_CUDA(cudaMemsetAsync(cnt, 0, (n + 1ULL) * sizeof(uint32_t), c.stream));
  RVN_CUDA(cudaMemsetAsync(off, 0, (n + 2ULL) * sizeof(uint64_t), c.stream));
}

// one flush of the reference's gather: `ovl` holds the m64 overlaps mapped for
// the queries [k0, k1) in query order, q_ovl_off their per-query offsets
// (relative to ovl, k1 - k0 + 1 entries); both on the device. Every read an
// overlap names lies in the window `w`; the lists of its reads are indexed by slot.
void GatherFlush(Ctx& c, const rvn_overlap* ovl, const uint64_t* q_ovl_off,
                 uint64_t m64, uint32_t k0, uint32_t k1, uint64_t kmax, const Window& w,
                 const uint64_t* row_off, uint64_t row_stride, uint32_t mark,
                 uint64_t* mark_off) {
  const uint32_t n = w.size();
  if (m64 == 0) {
    if (mark_off) *mark_off = ReadU64(c, c.g_off.get() + mark);
    return;
  }
  if (m64 >= 0xFFFFFFFFULL) throw LimitError("2^32 or more overlaps in one flush");
  const uint32_t m = static_cast<uint32_t>(m64);
  TimerBegin(c, "gather");
  // arrival order of the mirrored records: overlap indices stably sorted by rhs
  uint32_t* key = c.g_key.reserve(m);
  uint32_t* idx = c.g_idx.reserve(m);
  uint32_t* key2 = c.g_key2.reserve(m);
  uint32_t* idx2 = c.g_idx2.reserve(m);
  uint32_t* rhs_cnt = c.g_rhs_cnt.reserve(n + 1ULL);
  uint64_t* rhs_off = c.g_rhs_off.reserve(n + 2ULL);
  RVN_CUDA(cudaMemsetAsync(rhs_cnt, 0, (n + 1ULL) * sizeof(uint32_t), c.stream));
  RhsKeys<<<CeilDiv(m, kThreads), kThreads, 0, c.stream>>>(ovl, m, w, key, idx, rhs_cnt);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  int bits = 1;
  while ((1ULL << bits) < n) ++bits;
  // stable: records of one rhs read keep their overlap-index order (radix.cu); slots
  // of the index batch are in read order, and every rhs read is in the batch
  const int w_rhs = RadixSortPairs(c, key, key2, key, idx, idx2, idx, m, 0, bits);
  const uint32_t* sorted_idx = w_rhs == 0 ? idx2 : idx;
  ExclusiveScanU32(c, rhs_cnt, rhs_off, n);

  // staging list: kept records + new records per read
  uint32_t* total = c.g_total_cnt.reserve(n + 1ULL);
  uint64_t* t_off = c.g_t_off.reserve(n + 2ULL);
  ListTotals<<<CeilDiv(n, kThreads), kThreads, 0, c.stream>>>(
      c.g_cnt.get(), rhs_cnt, q_ovl_off, k0, k1, w, c.own_mod, c.own_rem, total);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  ExclusiveScanU32(c, total, t_off, n);
  // known without a read-back: compact lists hold g_total records, rows at most
  // row_stride per slot
  const uint64_t staged = (row_off ? n * row_stride : c.g_total) + 2ULL * m;
  rvn_overlap* stage = c.g_stage.reserve(staged + 1);
  uint64_t* pairs = c.g_pairs.reserve(staged + 1);
  uint32_t* kept = c.g_kept.reserve(n + 1ULL);
  const rvn_overlap* lists = c.g_list[c.g_cur].get();
  const uint64_t* old_off = row_off ? row_off : c.g_off.get();

  CopyOld<<<CeilDiv(n, kThreads / 32), kThreads, 0, c.stream>>>(
      lists, old_off, c.g_cnt.get(), t_off, n, stage);
  PlaceRhs<<<CeilDiv(m, kThreads), kThreads, 0, c.stream>>>(
      ovl, sorted_idx, m, rhs_off, c.g_cnt.get(), t_off, w, c.own_mod, c.own_rem, stage);
  PlaceLhs<<<CeilDiv(m, kThreads), kThreads, 0, c.stream>>>(
      ovl, m, q_ovl_off, k0, rhs_cnt, c.g_cnt.get(), t_off, w, c.own_mod, c.own_rem, stage);
  Truncate<<<CeilDiv(n, 128), 128, 0, c.stream>>>(stage, t_off, total,
                                                   c.g_cnt.get(), n, kmax, pairs,
                                                   kept);
  RVN_LAUNCH_CHECK();
  c.launches += 4;

  if (row_off) {
    // every list goes back to its row (the caller sized both list buffers)
    Compact<<<CeilDiv(n, kThreads / 32), kThreads, 0, c.stream>>>(
        stage, t_off, total, c.g_cnt.get(), kept, pairs, kmax, row_off, n,
        c.g_list[c.g_cur ^ 1].get());
    RVN_LAUNCH_CHECK();
    ++c.launches;
  } else {
    uint64_t* new_off = c.g_off_alt.reserve(n + 2ULL);
    ExclusiveScanU32(c, kept, new_off, n);
    const uint64_t new_total = ReadU64(c, new_off + n, new_off + mark, mark_off);
    rvn_overlap* next = c.g_list[c.g_cur ^ 1].reserve(new_total + 1);
    Compact<<<CeilDiv(n, kThreads / 32), kThreads, 0, c.stream>>>(
        stage, t_off, total, c.g_cnt.get(), kept, pairs, kmax, new_off, n, next);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    c.g_off.swap(c.g_off_alt);
    c.g_total = new_total;
  }
  // the new lists become current
  c.g_cur ^= 1;
  c.g_cnt.swap(c.g_kept);
  TimerEnd(c);
}

namespace {

__global__ void WindowTablesKernel(Window w, const uint64_t* __restrict__ poff,
                                   uint64_t stride, uint64_t* __restrict__ row_off,
                                   uint64_t* __restrict__ pile_off) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > w.size()) return;
  const uint32_t nb = w.b1 - w.b0;
  row_off[s] = s * stride;
  pile_off[s] = s <= nb ? poff[w.b0 + s] - poff[w.b0]
                        : (poff[w.b1] - poff[w.b0]) + (poff[w.a0 + (s - nb)] - poff[w.a0]);
}

}  // namespace

void WindowTables(Ctx& c, const Window& w, const uint64_t* d_poff, uint64_t stride,
                  uint64_t* row_off, uint64_t* pile_off) {
  WindowTablesKernel<<<CeilDiv(w.size() + 1ULL, kThreads), kThreads, 0, c.stream>>>(
      w, d_poff, stride, row_off, pile_off);
  RVN_LAUNCH_CHECK();
  ++c.launches;
}

void GatherFetch(Ctx& c) {
  const uint32_t n = c.n_reads;
  c.st_ovl.reserve(c.g_total + 1);
  RVN_CUDA(cudaMemcpyAsync(c.st_ovl_off.reserve(n + 1ULL), c.g_off.get(),
                           (n + 1ULL) * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                           c.stream));
  if (c.g_total) {
    RVN_CUDA(cudaMemcpyAsync(c.st_ovl.get(), c.g_list[c.g_cur].get(),
                             c.g_total * sizeof(rvn_overlap),
                             cudaMemcpyDeviceToHost, c.stream));
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

}  // namespace rvn
