// raven_b200 — pile-o-gram coverage update on sm_90a.
//
// Replaces raven::Pile::AddLayers (RavenLib/src/pile.cc:33-62; bins of 16
// bases, kPSS = 4, pile.h:21). The reference sorts begin/end marks per pile
// and sweeps; here every overlap side drops +1/-1 into a per-bin difference
// array (atomics), and one warp per pile turns the differences into coverage
// with a shuffle scan and adds it to the uint16 bins, saturating at 65535.
// The running coverage is kept modulo 2^32 exactly like the reference's
// unsigned counter, so the result is bit-identical (DESIGN.md).
#include <algorithm>

#include "engine.cuh"

namespace rvn {

namespace {

__device__ __forceinline__ void AddMarks(uint32_t id, uint32_t begin, uint32_t end,
                                         const uint64_t* __restrict__ bin_off, Window w,
                                         uint32_t mod, uint32_t rem,
                                         int32_t* __restrict__ diff) {
  if (id % mod != rem) return;
  const uint32_t p = w.Slot(id);
  if (p >= w.size()) return;
  const uint64_t base = bin_off[p] + p;
  const uint64_t bins = bin_off[p + 1] - bin_off[p];
  const uint32_t b = (begin >> 4) + 1, e = (end >> 4) - 1;
  if (b <= bins && e <= bins) {
    atomicAdd(diff + base + b, 1);
    atomicAdd(diff + base + e, -1);
  }
}

// pile of slot p owns diff[bin_off[p] + p .. bin_off[p+1] + p]  (bins + 1 slots);
// only the piles this context owns (id % mod == rem) are maintained
__global__ void ScatterMarks(const rvn_overlap* __restrict__ ovl, uint64_t n,
                             const uint64_t* __restrict__ bin_off, Window w,
                             uint32_t mod, uint32_t rem, int32_t* __restrict__ diff) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const rvn_overlap o = ovl[i];
  AddMarks(o.lhs_id, o.lhs_begin, o.lhs_end, bin_off, w, mod, rem, diff);
  AddMarks(o.rhs_id, o.rhs_begin, o.rhs_end, bin_off, w, mod, rem, diff);
}

// one warp per pile: inclusive scan of the differences, saturating add,
// and the differences are cleared for the next call (piles by slot: a window
// other than all reads is only used with mod == 1). Piles from the owned ones
// at or above `first` on (first is a multiple of mod).
__global__ void __launch_bounds__(256)
ApplyCoverage(uint16_t* __restrict__ data, const uint64_t* __restrict__ bin_off,
              uint32_t first, uint32_t n_piles, uint32_t mod, uint32_t rem,
              int32_t* __restrict__ diff) {
  const uint64_t p64 =
      first + static_cast<uint64_t>(blockIdx.x * 8 + (threadIdx.x >> 5)) * mod + rem;
  if (p64 >= n_piles) return;
  const uint32_t p = static_cast<uint32_t>(p64);
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t b0 = bin_off[p];
  const uint32_t bins = static_cast<uint32_t>(bin_off[p + 1] - b0);
  int32_t* d = diff + b0 + p;
  uint16_t* out = data + b0;
  uint32_t carry = 0;
  for (uint32_t base = 0; base <= bins; base += 32) {
    const uint32_t i = base + lane;
    uint32_t v = i <= bins ? static_cast<uint32_t>(d[i]) : 0u;
    if (i <= bins && v) d[i] = 0;
    uint32_t incl = v;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, incl, s);
      if (lane >= s) incl += o;
    }
    const uint32_t cov = carry + incl;
    if (i < bins && cov != 0) {
      const uint32_t sum = static_cast<uint32_t>(out[i]) + cov;  // wraps like the reference
      out[i] = sum < 65535u ? static_cast<uint16_t>(sum) : 65535;
    }
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
}

}  // namespace

void PileAddLayersDevice(Ctx& c, uint16_t* d_data, const uint64_t* d_off, uint64_t bins,
                         const Window& w, const rvn_overlap* d_ovl, uint64_t n_ovl,
                         uint32_t first) {
  const uint32_t n_piles = w.size();
  first -= first % c.own_mod;  // (the piles below `first` have no marks)
  if (n_piles <= first || n_ovl == 0) return;
  const uint64_t slots = bins + n_piles;
  if (c.p_diff.cap < slots) {
    int32_t* d = c.p_diff.reserve(slots);
    RVN_CUDA(cudaMemsetAsync(d, 0, c.p_diff.cap * sizeof(int32_t), c.stream));
  }
  TimerBegin(c, "pile");
  ScatterMarks<<<CeilDiv(n_ovl, 256), 256, 0, c.stream>>>(
      d_ovl, n_ovl, d_off, w, c.own_mod, c.own_rem, c.p_diff.get());
  const uint32_t owned = CeilDiv(n_piles - first, c.own_mod);
  ApplyCoverage<<<CeilDiv(owned, 8), 256, 0, c.stream>>>(d_data, d_off, first, n_piles,
                                                         c.own_mod, c.own_rem, c.p_diff.get());
  RVN_LAUNCH_CHECK();
  c.launches += 2;
  TimerEnd(c);
  c.stats.pile_bins += bins;
}

}  // namespace rvn

// ---------------------------------------------------------------------------
// raven::Pile::AddKmers (RavenLib/src/pile.cc:64-120): a position of an
// over-frequent minimizer marks its pile bin unless the k-mer is of low
// complexity. Three successive compressions, each must leave >= k/2 + 1
// characters: (1) homopolymer runs, (2) equal neighbouring 2-mers taken at even
// offsets, (3) equal neighbouring 2-mers taken at odd offsets. A pure function
// of <= 31 bases: one thread per position.
// ---------------------------------------------------------------------------
namespace rvn {

namespace {

__device__ __forceinline__ uint32_t BaseAt(const uint64_t* __restrict__ w, uint32_t i) {
  return static_cast<uint32_t>(w[i >> 5] >> ((i & 31) << 1)) & 3u;
}

// unique-consecutive over `n` tokens; tokens are (value, width) packed as
// value | width << 8; returns the number of characters kept and rewrites c[]
__device__ uint32_t CompressPairs(uint8_t* c, uint32_t n, uint32_t first_single) {
  // tokenise: an optional leading single, then 2-mers, a trailing single if odd
  uint8_t out[32];
  uint32_t m = 0;
  uint32_t i = 0;
  uint32_t last_tok = 0xFFFFFFFFu;
  auto emit = [&](uint32_t a, uint32_t b, uint32_t width) {
    const uint32_t tok = a | (b << 2) | (width << 4);
    if (tok != last_tok) {
      out[m++] = static_cast<uint8_t>(a);
      if (width == 2) out[m++] = static_cast<uint8_t>(b);
    }
    last_tok = tok;
  };
  if (first_single && n > 0) {
    emit(c[0], 0, 1);
    i = 1;
  }
  for (; i + 1 < n; i += 2) emit(c[i], c[i + 1], 2);
  if (i < n) emit(c[i], 0, 1);
  for (uint32_t j = 0; j < m; ++j) c[j] = out[j];
  return m;
}

// the test of one k-mer: true iff the reference marks kmers_[p >> 4]
__device__ bool KmerPasses(const uint64_t* __restrict__ w, uint32_t len, uint32_t p,
                           uint32_t k) {
  uint8_t c[32];
  uint32_t m = 0;
  // InflateData(p, k) clamps at the read end
  for (uint32_t i = 0; i < k && p + i < len; ++i) c[m++] = static_cast<uint8_t>(BaseAt(w, p + i));
  const uint32_t need = k / 2 + 1;
  // (1) homopolymer compression
  uint32_t q = 0;
  for (uint32_t i = 0; i < m; ++i) {
    if (i == 0 || c[i] != c[i - 1]) c[q++] = c[i];
  }
  m = q;
  if (m < need) return false;
  m = CompressPairs(c, m, 0);  // (2) 2-mers at even offsets
  if (m < need) return false;
  m = CompressPairs(c, m, 1);  // (3) 2-mers at odd offsets
  return m >= need;
}

__global__ void KmerComplexityKernel(const uint64_t* __restrict__ words,
                                     const uint64_t* __restrict__ woff,
                                     const uint32_t* __restrict__ lens,
                                     const uint32_t* __restrict__ read_idx,
                                     const uint32_t* __restrict__ pos, uint64_t n,
                                     uint32_t k, uint8_t* __restrict__ keep) {
  const uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t r = read_idx[t];
  keep[t] = KmerPasses(words + woff[r], lens[r], pos[t], k) ? 1 : 0;
}

// One thread per filtered position of the flush's nr query reads (from read `first` on):
// its read by binary search in the per-read offsets, then the test and the mark.
__global__ void KmerMarksKernel(const uint64_t* __restrict__ words,
                                const uint64_t* __restrict__ woff,
                                const uint32_t* __restrict__ lens,
                                const uint32_t* __restrict__ pos,
                                const uint64_t* __restrict__ read_off, uint32_t first,
                                uint32_t nr, uint64_t n, uint32_t k,
                                const uint64_t* __restrict__ bit_off,
                                uint32_t* __restrict__ bits, uint8_t* __restrict__ touched) {
  const uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  uint32_t lo = 0, hi = nr;  // the read i with read_off[i] <= t < read_off[i + 1]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (read_off[mid] <= t) lo = mid; else hi = mid;
  }
  const uint32_t r = first + lo;
  const uint32_t p = pos[t];
  touched[r] = 1;
  if (KmerPasses(words + woff[r], lens[r], p, k)) {
    const uint32_t bin = p >> 4;
    atomicOr(bits + bit_off[r] + (bin >> 5), 1u << (bin & 31));
  }
}

// Pile::FindValidRegion(coverage) + Pile::FindMedian (pile.cc:122-172) of fresh piles
// (begin_ = 0, end_ = bins), one warp per pile. The region is the first longest run of
// bins >= coverage that is FOLLOWED by a bin below it (the reference's scan never
// records a run that reaches the last bin); it is valid from 1260 >> 4 bins on. The
// median is the element of rank size / 2 of the region (std::nth_element): the
// largest r with #{x < r} <= size / 2, found bit by bit.
__global__ void __launch_bounds__(128)
PileRegionsKernel(const uint16_t* __restrict__ data, const uint64_t* __restrict__ off,
                  uint64_t off_base, uint32_t n_piles, uint32_t coverage,
                  uint32_t* __restrict__ out_begin, uint32_t* __restrict__ out_end,
                  uint16_t* __restrict__ out_median, uint8_t* __restrict__ out_invalid) {
  const uint32_t p = (blockIdx.x * 128 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (p >= n_piles) return;
  const uint16_t* d = data + (off[p] - off_base);
  const uint32_t nb = static_cast<uint32_t>(off[p + 1] - off[p]);
  uint32_t begin = 0, end = 0;
  long long run = -1;  // start of the run the scan is in
  for (uint32_t base = 0; base < nb; base += 32) {
    const uint32_t i = base + lane;
    const uint32_t bits = min(32u, nb - base);
    const uint32_t live = bits == 32 ? 0xFFFFFFFFu : ((1u << bits) - 1u);
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, i < nb && d[i] >= coverage) & live;
    uint32_t pos = 0;
    while (pos < bits) {
      if (run < 0) {  // next bin at or above the coverage
        const uint32_t mm = m >> pos;
        if (mm == 0) break;
        const uint32_t s = __ffs(mm) - 1;
        run = static_cast<long long>(base) + pos + s;
        pos += s + 1;
      } else {  // next bin below it
        const uint32_t mm = (~m & live) >> pos;
        if (mm == 0) break;
        const uint32_t e = __ffs(mm) - 1;
        const uint32_t j = base + pos + e;
        if (end - begin < j - static_cast<uint32_t>(run)) {
          begin = static_cast<uint32_t>(run);
          end = j;
        }
        run = -1;
        pos += e + 1;
      }
    }
  }
  const bool invalid = begin >= end || end - begin < (1260u >> 4);
  uint32_t median = 0;
  if (!invalid) {
    const uint32_t size = end - begin, k = size / 2;
    uint32_t r = 0;
    for (int bit = 15; bit >= 0; --bit) {
      const uint32_t cand = r | (1u << bit);
      uint32_t c = 0;
      for (uint32_t i = begin + lane; i < end; i += 32) c += d[i] < cand;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
      if (c <= k) r = cand;
    }
    median = r;
  }
  if (lane == 0) {
    out_begin[p] = invalid ? 0 : begin;
    out_end[p] = invalid ? nb : end;
    out_median[p] = static_cast<uint16_t>(median);
    out_invalid[p] = invalid ? 1 : 0;
  }
}

}  // namespace

void KmerComplexity(Ctx& c, const uint32_t* h_read_idx, const uint32_t* h_pos,
                    uint64_t n, uint32_t k, uint8_t* h_keep) {
  if (n == 0) return;
  uint32_t* d_idx = c.m_cnt.reserve(n);
  uint32_t* d_pos = c.m_first.reserve(n);
  uint8_t* d_keep = c.m_filt.reserve(n);
  RVN_CUDA(cudaMemcpyAsync(d_idx, h_read_idx, n * 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_pos, h_pos, n * 4, cudaMemcpyHostToDevice, c.stream));
  KmerComplexityKernel<<<CeilDiv(n, 256), 256, 0, c.stream>>>(
      c.d_words.get(), c.d_woff.get(), c.d_len.get(), d_idx, d_pos, n, k, d_keep);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  RVN_CUDA(cudaMemcpyAsync(h_keep, d_keep, n, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

void Stage2KmerMarks(Ctx& c, uint32_t first, uint32_t nr, uint32_t k) {
  const uint64_t n = c.m_n_filtered;
  if (n == 0) return;
  TimerBegin(c, "stage2_kmers");
  KmerMarksKernel<<<CeilDiv(n, 256), 256, 0, c.stream>>>(
      c.d_words.get(), c.d_woff.get(), c.d_len.get(), c.m_filtered.get(), c.m_filtered_off.get(),
      first, nr, n, k, c.s2_bit_off.get(), c.s2_bits.get(), c.s2_touched.get());
  RVN_LAUNCH_CHECK();
  ++c.launches;
  TimerEnd(c);
}

// valid regions and medians of the piles of the last stage-1 call: on the device
// after a resident run; after a windowed run they are on the host and pass
// through the device in chunks of reads
void StagePileRegions(Ctx& c, uint32_t coverage, uint32_t* h_begin, uint32_t* h_end,
                      uint16_t* h_median, uint8_t* h_invalid) {
  if (!c.st_valid || !(c.st_piles_on_device || c.st_windowed)) {
    throw StateError("no stage-1 piles on the device (run rvn_find_overlaps_and_create_piles first)");
  }
  const uint32_t n = c.n_reads;
  if (n == 0) return;
  uint32_t* d_b = c.m_cnt.reserve(2ULL * n + 2);
  uint32_t* d_e = d_b + n + 1;
  uint16_t* d_m = reinterpret_cast<uint16_t*>(c.m_first.reserve(n / 2 + 2));
  uint8_t* d_i = c.m_filt.reserve(n + 1ULL);
  TimerBegin(c, "pile_regions");
  if (c.st_piles_on_device) {
    PileRegionsKernel<<<CeilDiv(n, 4), 128, 0, c.stream>>>(c.p_data.get(), c.p_off.get(), 0, n,
                                                         coverage, d_b, d_e, d_m, d_i);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  } else {
    const std::vector<uint64_t>& off = c.h_pile_off;
    uint64_t* d_off = c.p_off.reserve(n + 1ULL);
    RVN_CUDA(cudaMemcpyAsync(d_off, off.data(), (n + 1ULL) * 8, cudaMemcpyHostToDevice,
                             c.stream));
    // chunks as large as the window pile buffer of the run (one read at least)
    const uint64_t cap = std::max<uint64_t>(c.p_data.cap, 1) - 1;
    for (uint32_t r0 = 0, r1; r0 < n; r0 = r1) {
      r1 = r0 + 1;
      while (r1 < n && off[r1 + 1] - off[r0] <= cap) ++r1;
      const uint64_t bins = off[r1] - off[r0];
      uint16_t* d = c.p_data.reserve(bins + 1);
      RVN_CUDA(cudaMemcpyAsync(d, c.st_pile.get() + off[r0], bins * 2, cudaMemcpyHostToDevice,
                               c.stream));
      PileRegionsKernel<<<CeilDiv(r1 - r0, 4), 128, 0, c.stream>>>(
          d, d_off + r0, off[r0], r1 - r0, coverage, d_b + r0, d_e + r0, d_m + r0, d_i + r0);
      RVN_LAUNCH_CHECK();
      ++c.launches;
    }
  }
  TimerEnd(c);
  RVN_CUDA(cudaMemcpyAsync(h_begin, d_b, n * 4ULL, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(h_end, d_e, n * 4ULL, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(h_median, d_m, n * 2ULL, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(h_invalid, d_i, n, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

}  // namespace rvn
