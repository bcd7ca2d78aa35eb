// raven_b200 — device-wide exclusive scan (u32 counts -> u64 offsets), phase
// timers and small D2H helpers. Reduce-then-scan in three launches: chunk
// sums, one CTA scanning the chunk sums, chunk rescan with carried base.
#include "engine.cuh"

namespace rvn {

namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;
constexpr int kScanChunk = kScanThreads * kScanItems;

__global__ void __launch_bounds__(kScanThreads)
ScanChunkSums(const uint32_t* __restrict__ in, uint64_t n,
              uint64_t* __restrict__ chunk_sum) {
  __shared__ uint64_t sm[33];
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * kScanChunk;
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    uint64_t idx = base + static_cast<uint64_t>(i) * kScanThreads + threadIdx.x;
    if (idx < n) s += in[idx];
  }
  uint64_t total;
  BlockExclusiveSum<uint64_t, kScanThreads>(s, sm, &total);
  if (threadIdx.x == 0) chunk_sum[blockIdx.x] = total;
}

// one CTA: exclusive scan of chunk sums in place; grand total -> *total
__global__ void __launch_bounds__(1024)
ScanOfSums(uint64_t* __restrict__ chunk_sum, uint64_t n_chunks,
           uint64_t* __restrict__ total) {
  __shared__ uint64_t sm[33];
  uint64_t carry = 0;
  for (uint64_t b = 0; b < n_chunks; b += 1024) {
    uint64_t i = b + threadIdx.x;
    uint64_t v = i < n_chunks ? chunk_sum[i] : 0;
    uint64_t t;
    uint64_t ex = BlockExclusiveSum<uint64_t, 1024>(v, sm, &t);
    if (i < n_chunks) chunk_sum[i] = carry + ex;
    carry += t;
  }
  if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kScanThreads)
ScanChunks(const uint32_t* __restrict__ in, uint64_t n,
           const uint64_t* __restrict__ chunk_sum, uint64_t* __restrict__ out) {
  __shared__ uint64_t sm[33];
  const uint64_t base = static_cast<uint64_t>(blockIdx.x) * kScanChunk +
                        static_cast<uint64_t>(threadIdx.x) * kScanItems;
  uint32_t v[kScanItems];
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    uint64_t idx = base + i;
    v[i] = idx < n ? in[idx] : 0;
    s += v[i];
  }
  uint64_t total;
  uint64_t ex = BlockExclusiveSum<uint64_t, kScanThreads>(s, sm, &total);
  uint64_t run = chunk_sum[blockIdx.x] + ex;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    uint64_t idx = base + i;
    if (idx < n) out[idx] = run;
    run += v[i];
  }
}

}  // namespace

void ExclusiveScanU32(Ctx& c, const uint32_t* in, uint64_t* out, uint64_t n) {
  if (n == 0) {
    RVN_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), c.stream));
    return;
  }
  const uint64_t chunks = (n + kScanChunk - 1) / kScanChunk;
  uint64_t* sums = c.scan_tmp.reserve(chunks + 1);
  ScanChunkSums<<<static_cast<unsigned>(chunks), kScanThreads, 0, c.stream>>>(
      in, n, sums);
  ScanOfSums<<<1, 1024, 0, c.stream>>>(sums, chunks, out + n);
  ScanChunks<<<static_cast<unsigned>(chunks), kScanThreads, 0, c.stream>>>(
      in, n, sums, out);
  RVN_LAUNCH_CHECK();
  c.launches += 3;
}

namespace {

// h: pinned host memory, which the device addresses directly (unified addressing)
__global__ void ReadBackKernel(const uint64_t* a, const uint64_t* b, uint64_t* h) {
  h[0] = *a;
  if (b) h[1] = *b;
}

}  // namespace

// The values travel as stores of a one-thread kernel, not as a copy: a copy would queue
// behind whatever the copy engines carry for other streams (stage 1's result copies,
// megabytes, run beside its flushes). Not counted in c.launches: it stands for a copy.
uint64_t ReadU64(Ctx& c, const uint64_t* dptr, const uint64_t* dptr2, uint64_t* value2) {
  uint64_t* h = c.pin64.reserve(8);
  ReadBackKernel<<<1, 1, 0, c.stream>>>(dptr, value2 ? dptr2 : nullptr, h);
  RVN_LAUNCH_CHECK();
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  if (value2) *value2 = h[1];
  return h[0];
}

// ---- phase timers: CUDA events on the context's stream ----
static cudaEvent_t GetEvent(Ctx& c) {
  if (!c.timer.pool.empty()) {
    cudaEvent_t e = c.timer.pool.back();
    c.timer.pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  RVN_CUDA(cudaEventCreate(&e));
  return e;
}

void TimerBegin(Ctx& c, const char* name) {
  cudaEvent_t a = GetEvent(c), b = GetEvent(c);
  RVN_CUDA(cudaEventRecord(a, c.stream));
  c.timer.names.push_back(name);
  c.timer.ms.push_back(-1.f);  // open
  c.timer.pending.emplace_back(a, b);
}

void TimerEnd(Ctx& c) {
  // closes the most recently opened, still open phase
  for (std::size_t i = c.timer.pending.size(); i-- > 0;) {
    if (c.timer.ms[i] == -1.f) {
      RVN_CUDA(cudaEventRecord(c.timer.pending[i].second, c.stream));
      c.timer.ms[i] = -2.f;  // recorded, not yet read
      return;
    }
  }
}

void TimerCollect(Ctx& c) {
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  for (std::size_t i = 0; i < c.timer.pending.size(); ++i) {
    if (c.timer.ms[i] == -2.f) {
      float ms = 0;
      RVN_CUDA(cudaEventElapsedTime(&ms, c.timer.pending[i].first,
                                    c.timer.pending[i].second));
      c.timer.ms[i] = ms;
      c.timer.pool.push_back(c.timer.pending[i].first);
      c.timer.pool.push_back(c.timer.pending[i].second);
      c.timer.pending[i] = {nullptr, nullptr};
    }
  }
}

void TimerReset(Ctx& c) {
  TimerCollect(c);
  c.timer.names.clear();
  c.timer.ms.clear();
  c.timer.pending.clear();
}

}  // namespace rvn
