// raven_b200 — the window layers of racon::Polisher::Polish built on the device, and
// the window consensus over batches of windows (include/raven_b200.h,
// rvn_polish_windows; the reference call is RavenLib/src/polish.cc:43-51).
//
// The reads are on the device as 2-bit words (rvn_reads_upload) and the breaking
// points of every alignment are 16 B per window slot; a read's qualities are one
// biosoup block score per 64 bases. From these alone:
//   LayerRulesKernel   racon's per-slot rules (length, average quality, begin < end)
//                      -> per slot its window, or dropped; per window its kept layers
//                      and their bases
//   stable radix sort  of the slots by window: a window's layers stay in the order of
//                      (alignment, slot), the order racon adds them in
//   per window batch   BatchTablesKernel (sequence lengths, begin, end), a scan to the
//                      sequence offsets, PackKernel (backbone and layers as ASCII
//                      letters and Phred+33 qualities, one warp writing each sequence),
//                      then PoaRun (poa.cu) on that flat layout.
// No layer base passes through the host; device memory is bounded by a batch.
#include <algorithm>

#include "engine.cuh"

namespace rvn {

namespace {

constexpr uint32_t kStrand = 1;  // the read aligns on the target's strand
constexpr uint32_t kFlip = 2;    // Score of the aligned view reads block_quality backwards
constexpr uint32_t kQual = 4;    // the read has block qualities
constexpr int kWarpsPerBlock = 8;

struct LayerAln {  // one alignment
  uint64_t woff;          // first word of the read in c.d_words
  uint64_t bq;            // first block quality of the read in the uploaded qualities
  uint64_t slot0, slot1;  // its breaking-point slots
  uint32_t len;           // read length
  uint32_t qb;            // first aligned base, in the aligned orientation of the read
  uint32_t win0, win1;    // the windows of its target
  uint32_t flags;
  uint32_t pad;
};

struct BatchWin {  // one window of a batch
  uint64_t woff;    // first word of its target
  uint64_t lfirst;  // its first layer in the sorted slot order
  uint32_t start, len;  // backbone: target bases [start, start + len)
  uint32_t layers;
  uint32_t pad;
};

__device__ __forceinline__ uint32_t Base(const uint64_t* words, uint64_t woff, uint64_t i) {
  return static_cast<uint32_t>(words[woff + (i >> 5)] >> ((i & 31) << 1)) & 3u;
}

// One warp per alignment, lanes over its slots. Slot s gets key[s] = its window, or
// `drop` (sorts after every window), and ord[s] = alignment << 32 | s.
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
LayerRulesKernel(const LayerAln* __restrict__ aln, uint64_t n_aln, const uint4* __restrict__ bp,
                 const uint8_t* __restrict__ bq, uint32_t w, double q, uint32_t drop,
                 uint32_t* __restrict__ key, uint64_t* __restrict__ ord, uint32_t* cnt,
                 unsigned long long* bases, unsigned long long* err) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = static_cast<uint64_t>(gridDim.x) * kWarpsPerBlock;
  for (uint64_t a = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
       a < n_aln; a += warps) {
    const LayerAln r = aln[a];
    for (uint64_t s = r.slot0 + lane; s < r.slot1; s += 32) {
      uint32_t k = drop;
      const uint4 b = bp[s];
      if (b.x != 0xFFFFFFFFu) {  // else: no aligned pair in this window
        const uint32_t ft = b.x, fq = r.qb + b.y, lt = b.z, lq = r.qb + b.w;
        const uint32_t d = lq - fq;
        if (static_cast<uint64_t>(r.qb) + b.w > r.len || b.y > b.w || ft >= lt ||
            r.win0 + static_cast<uint64_t>(ft / w) >= r.win1) {
          atomicOr(err, 1ULL);
        } else if (d >= 0.02 * w) {
          bool keep = true;
          if (r.flags & kQual) {
            // sum of Score(x), x in [fq, lq), over the blocks the range covers
            uint64_t i0 = fq, i1 = lq;
            if (r.flags & kFlip) {
              i0 = r.len - lq;
              i1 = r.len - fq;
            }
            uint64_t sum = 0;
            for (uint64_t blk = i0 >> 6; blk <= (i1 - 1) >> 6; ++blk) {
              const uint64_t lo = max(i0, blk << 6), hi = min(i1, (blk + 1) << 6);
              sum += (hi - lo) * bq[r.bq + blk];
            }
            // integer scores: the sum is exactly the host's running double sum
            keep = !(static_cast<double>(sum) / d < q);
          }
          const uint32_t ws = (ft / w) * w;
          if (keep && !(ft - ws >= lt - ws - 1)) {  // racon skips begin == end
            k = r.win0 + ft / w;
            atomicAdd(cnt + k, 1u);
            atomicAdd(bases + k, static_cast<unsigned long long>(d));
          }
        }
      }
      key[s] = k;
      ord[s] = a << 32 | s;
    }
  }
}

// One warp per window of the batch: sequence lengths, begins and ends (the backbone
// first, then the window's layers in sorted order).
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
BatchTablesKernel(const BatchWin* __restrict__ win, uint32_t n_win,
                  const uint32_t* __restrict__ wf, const uint64_t* __restrict__ ord,
                  const LayerAln* __restrict__ aln, const uint4* __restrict__ bp, uint32_t w,
                  uint32_t* __restrict__ seq_len, uint32_t* __restrict__ seq_begin,
                  uint32_t* __restrict__ seq_end) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_win) return;
  const BatchWin bw = win[i];
  const uint32_t s0 = wf[i];
  if (lane == 0) {
    seq_len[s0] = bw.len;
    seq_begin[s0] = 0;
    seq_end[s0] = 0;
  }
  for (uint32_t j = lane; j < bw.layers; j += 32) {
    const uint64_t v = ord[bw.lfirst + j];
    const LayerAln& r = aln[v >> 32];
    const uint4 b = bp[v & 0xFFFFFFFFu];
    const uint32_t ws = (b.x / w) * w;
    seq_len[s0 + 1 + j] = (r.qb + b.w) - (r.qb + b.y);
    seq_begin[s0 + 1 + j] = b.x - ws;
    seq_end[s0 + 1 + j] = b.z - ws - 1;
  }
}

// One warp per window of the batch, the whole warp over one sequence at a time: letters
// and, when `quals` is not null, Phred+33 qualities at the sequence offsets.
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
PackKernel(const BatchWin* __restrict__ win, uint32_t n_win, const uint32_t* __restrict__ wf,
           const uint64_t* __restrict__ so, const uint64_t* __restrict__ ord,
           const LayerAln* __restrict__ aln, const uint4* __restrict__ bp,
           const uint64_t* __restrict__ words, const uint8_t* __restrict__ bq,
           uint8_t* __restrict__ bases, uint8_t* __restrict__ quals) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_win) return;
  const BatchWin bw = win[i];
  const uint32_t s0 = wf[i];
  {
    const uint64_t o = so[s0];
    for (uint32_t t = lane; t < bw.len; t += 32) {
      bases[o + t] = "ACGT"[Base(words, bw.woff, static_cast<uint64_t>(bw.start) + t)];
      if (quals) quals[o + t] = '!';  // the backbone weighs 0
    }
  }
  for (uint32_t j = 0; j < bw.layers; ++j) {
    const uint64_t v = ord[bw.lfirst + j];
    const LayerAln r = aln[v >> 32];
    const uint4 b = bp[v & 0xFFFFFFFFu];
    const uint32_t fq = r.qb + b.y, n = b.w - b.y;
    const uint64_t o = so[s0 + 1 + j];
    for (uint32_t t = lane; t < n; t += 32) {
      const uint32_t p = fq + t;  // position in the aligned orientation
      const uint32_t code = (r.flags & kStrand) ? Base(words, r.woff, p)
                                                : Base(words, r.woff, r.len - 1 - p) ^ 3u;
      bases[o + t] = "ACGT"[code];
      if (quals) {
        uint8_t qv = '!' + 1;  // a read without qualities weighs 1
        if (r.flags & kQual) {
          const uint32_t x = (r.flags & kFlip) ? r.len - 1 - p : p;
          qv = static_cast<uint8_t>(bq[r.bq + (x >> 6)] + '!');
        }
        quals[o + t] = qv;
      }
    }
  }
}

unsigned WarpGrid(uint64_t warps) {
  return static_cast<unsigned>((warps + kWarpsPerBlock - 1) / kWarpsPerBlock);
}

}  // namespace

void PolishWindows(Ctx& c, const PolishArgs& a) {
  c.poa_valid = false;
  if (a.gap >= 0) {
    throw InvalidArgument("[racon::Polisher::Create] error: gap penalty must be negative");
  }
  if (a.window == 0) throw InvalidArgument("window length 0");
  if (c.n_reads == 0) throw StateError("no reads uploaded (rvn_reads_upload)");
  if (a.n_targets > c.n_reads) throw InvalidArgument("more targets than uploaded reads");
  const uint32_t T = a.n_targets, W = a.window;
  std::vector<uint64_t> first_window(T + 1ULL, 0);
  for (uint32_t t = 0; t < T; ++t) {
    CheckResident(c, t, t + 1);
    first_window[t + 1] = first_window[t] + (c.h_len[t] + static_cast<uint64_t>(W) - 1) / W;
  }
  const uint64_t n_win64 = first_window[T];
  if (n_win64 >= 0xFFFFFFFFULL) throw LimitError("2^32 or more windows");
  const uint32_t n_windows = static_cast<uint32_t>(n_win64);
  // block qualities: a read has none (empty range) or one per 64 bases
  bool any_quality = false;
  uint64_t n_bq = 0;
  if (a.bq) {
    for (uint32_t r = 0; r < c.n_reads; ++r) {
      const uint64_t k = a.bq_off[r + 1] - a.bq_off[r];
      if (a.bq_off[r + 1] < a.bq_off[r] || (k && k < (c.h_len[r] + 63ULL) / 64)) {
        throw InvalidArgument("a read has fewer block qualities than 64-base blocks");
      }
      any_quality = any_quality || k;
    }
    n_bq = a.bq_off[c.n_reads];
  }
  const uint64_t A = a.n_aln;
  if (A >= 0xFFFFFFFFULL) throw LimitError("2^32 or more alignments");
  std::vector<LayerAln> h(A);
  for (uint64_t i = 0; i < A; ++i) {
    const uint32_t k = a.q_read[i], t = a.t_read[i];
    if (k >= c.n_reads || t >= T) throw InvalidArgument("read index out of bounds");
    CheckResident(c, k, k + 1);
    const uint32_t L = c.h_len[k];
    if (static_cast<uint64_t>(a.q_begin[i]) + a.q_len[i] > L) {
      throw InvalidArgument("substring beyond the end of its read");
    }
    if (a.bp_off[i + 1] < a.bp_off[i]) throw InvalidArgument("bp_off must not decrease");
    LayerAln& r = h[i];
    r.woff = c.h_woff[k];
    r.bq = a.bq ? a.bq_off[k] : 0;
    r.slot0 = a.bp_off[i];
    r.slot1 = a.bp_off[i + 1];
    r.len = L;
    // query positions are those of the aligned orientation of the read
    r.qb = a.strand[i] ? a.q_begin[i] : L - (a.q_begin[i] + a.q_len[i]);
    r.win0 = static_cast<uint32_t>(first_window[t]);
    r.win1 = static_cast<uint32_t>(first_window[t + 1]);
    const bool has_q = a.bq && a.bq_off[k + 1] > a.bq_off[k];
    const bool rc = a.rc && a.rc[k];
    r.flags = (a.strand[i] ? kStrand : 0) | ((rc != !a.strand[i]) ? kFlip : 0) |
              (has_q ? kQual : 0);
    r.pad = 0;
  }
  if (a.bp_off[0] != 0) throw InvalidArgument("bp_off must start at 0");
  const uint64_t n_slots = A ? a.bp_off[A] : 0;
  if (n_slots >= 0xFFFFFFFFULL) throw LimitError("2^32 or more breaking-point slots");

  // ---- racon's layer rules and the stable order by window ----
  TimerBegin(c, "poa_layers");
  auto* d_aln = reinterpret_cast<LayerAln*>(c.pl_aln.reserve(A * sizeof(LayerAln) + 64));
  uint32_t* d_bp = c.pl_bp.reserve(4 * n_slots + 4);
  uint8_t* d_bq = c.pl_bq.reserve(n_bq + 16);
  uint32_t* d_cnt = c.pl_cnt.reserve(n_windows + 1ULL);
  uint64_t* d_wbases = c.pl_bases.reserve(n_windows + 1ULL);
  uint64_t* d_err = c.pl_err.reserve(1);
  uint32_t* key_a = c.pl_key[0].reserve(n_slots + 1);
  uint32_t* key_b = c.pl_key[1].reserve(n_slots + 1);
  uint64_t* ord_a = c.pl_ord[0].reserve(n_slots + 1);
  uint64_t* ord_b = c.pl_ord[1].reserve(n_slots + 1);
  if (A) {
    RVN_CUDA(cudaMemcpyAsync(d_aln, h.data(), A * sizeof(LayerAln), cudaMemcpyHostToDevice, c.stream));
  }
  if (n_slots) {
    RVN_CUDA(cudaMemcpyAsync(d_bp, a.bp, 16 * n_slots, cudaMemcpyHostToDevice, c.stream));
  }
  if (n_bq) RVN_CUDA(cudaMemcpyAsync(d_bq, a.bq, n_bq, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_cnt, 0, (n_windows + 1ULL) * 4, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_wbases, 0, (n_windows + 1ULL) * 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_err, 0, 8, c.stream));
  const uint4* d_bp4 = reinterpret_cast<const uint4*>(d_bp);
  const uint64_t* ord = ord_b;
  if (A) {
    LayerRulesKernel<<<std::min<unsigned>(WarpGrid(A), c.sms * 16), kWarpsPerBlock * 32, 0,
                       c.stream>>>(d_aln, A, d_bp4, d_bq, W, a.q, n_windows, key_b, ord_b, d_cnt,
                                   reinterpret_cast<unsigned long long*>(d_wbases),
                                   reinterpret_cast<unsigned long long*>(d_err));
    RVN_LAUNCH_CHECK();
    ++c.launches;
    // keys 0 .. n_windows (dropped): the bits of n_windows
    const int bits = n_windows ? 32 - __builtin_clz(n_windows) : 1;
    const int where = RadixSortPairs(c, key_b, key_a, key_b, ord_b, ord_a, ord_b, n_slots, 0, bits);
    ord = where == 0 ? ord_a : ord_b;
  }
  std::vector<uint32_t> cnt(n_windows);
  std::vector<uint64_t> wbases(n_windows);
  RVN_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, n_windows * 4ULL, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(wbases.data(), d_wbases, n_windows * 8ULL, cudaMemcpyDeviceToHost, c.stream));
  const uint64_t bad = ReadU64(c, d_err);
  TimerEnd(c);
  if (bad) throw InvalidArgument("a breaking point lies outside its read or its target's windows");

  // ---- windows in batches: inputs, consensus slots and tables of a batch ----
  std::vector<uint64_t> lfirst(n_windows + 1ULL, 0), need(n_windows);
  std::vector<uint32_t> w_target(n_windows);
  for (uint32_t t = 0, w = 0; t < T; ++t) {
    for (; w < first_window[t + 1]; ++w) w_target[w] = t;
  }
  const uint64_t per_base = any_quality ? 3 : 2;  // letters, qualities, consensus slot
  for (uint32_t w = 0; w < n_windows; ++w) {
    lfirst[w + 1] = lfirst[w] + cnt[w];
    const uint32_t t = w_target[w];
    const uint64_t start = (w - first_window[t]) * W;
    const uint64_t bb = std::min<uint64_t>(start + W, c.h_len[t]) - start;
    need[w] = per_base * (bb + wbases[w]) + 20ULL * (1 + cnt[w]) + 64;
  }
  uint64_t budget = c.poa_batch_bytes;
  if (!budget) {
    size_t free_b = 0, total_b = 0;
    RVN_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // the buffers a batch reuses, and the POA scratch half of what is left
    budget = (free_b + c.po_bases.cap + c.po_quals.cap + c.po_cons.cap) / 4;
  }

  std::vector<uint8_t> status(n_windows, 0), cons;
  std::vector<uint64_t> cons_off(n_windows + 1ULL, 0);
  uint32_t routes[3] = {0, 0, 0}, launches[3] = {0, 0, 0};
  uint64_t cells = 0;
  c.po_batches = 0;
  std::vector<uint32_t> h_wf;
  std::vector<BatchWin> h_win;
  std::vector<uint64_t> h_so;
  std::vector<uint32_t> h_sb, h_se;
  for (uint32_t w0 = 0; w0 < n_windows;) {
    uint32_t w1 = w0;
    uint64_t bytes = 0;
    while (w1 < n_windows && (w1 == w0 || bytes + need[w1] <= budget)) bytes += need[w1++];
    const uint32_t nb = w1 - w0;
    TimerBegin(c, "poa_pack");
    h_wf.assign(nb + 1ULL, 0);
    h_win.resize(nb);
    uint64_t n_bases = 0;
    for (uint32_t i = 0; i < nb; ++i) {
      const uint32_t w = w0 + i, t = w_target[w];
      BatchWin& bw = h_win[i];
      bw.woff = c.h_woff[t];
      bw.lfirst = lfirst[w];
      bw.start = (w - static_cast<uint32_t>(first_window[t])) * W;
      bw.len = static_cast<uint32_t>(std::min<uint64_t>(bw.start + static_cast<uint64_t>(W), c.h_len[t]) -
                                     bw.start);
      bw.layers = cnt[w];
      bw.pad = 0;
      n_bases += bw.len + wbases[w];
      const uint64_t next = h_wf[i] + 1ULL + cnt[w];
      if (next >= 0xFFFFFFFFULL) throw LimitError("2^32 or more sequences in one window batch");
      h_wf[i + 1] = static_cast<uint32_t>(next);
    }
    const uint32_t n_seqs = h_wf[nb];
    uint32_t* d_wf = c.po_win_first.reserve(nb + 2ULL);
    auto* d_win = reinterpret_cast<BatchWin*>(c.pl_win.reserve(nb * sizeof(BatchWin) + 64));
    uint32_t* d_len = c.pl_seq_len.reserve(n_seqs + 2ULL);
    uint64_t* d_so = c.po_seq_off.reserve(n_seqs + 2ULL);
    uint32_t* d_sb = c.po_seq_begin.reserve(n_seqs + 2ULL);
    uint32_t* d_se = c.po_seq_end.reserve(n_seqs + 2ULL);
    uint8_t* d_bases = c.po_bases.reserve(n_bases + 16);
    uint8_t* d_quals = any_quality ? c.po_quals.reserve(n_bases + 16) : nullptr;
    RVN_CUDA(cudaMemcpyAsync(d_wf, h_wf.data(), (nb + 1ULL) * 4, cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(d_win, h_win.data(), nb * sizeof(BatchWin), cudaMemcpyHostToDevice, c.stream));
    BatchTablesKernel<<<WarpGrid(nb), kWarpsPerBlock * 32, 0, c.stream>>>(
        d_win, nb, d_wf, ord, d_aln, d_bp4, W, d_len, d_sb, d_se);
    RVN_LAUNCH_CHECK();
    ExclusiveScanU32(c, d_len, d_so, n_seqs);
    PackKernel<<<WarpGrid(nb), kWarpsPerBlock * 32, 0, c.stream>>>(
        d_win, nb, d_wf, d_so, ord, d_aln, d_bp4, c.d_words.get(), d_bq, d_bases, d_quals);
    RVN_LAUNCH_CHECK();
    c.launches += 2;
    h_so.resize(n_seqs + 1ULL);
    h_sb.resize(n_seqs);
    h_se.resize(n_seqs);
    RVN_CUDA(cudaMemcpyAsync(h_so.data(), d_so, (n_seqs + 1ULL) * 8, cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(h_sb.data(), d_sb, n_seqs * 4ULL, cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(h_se.data(), d_se, n_seqs * 4ULL, cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    TimerEnd(c);

    PoaInput d;
    d.win_first = d_wf;
    d.seq_off = d_so;
    d.bases = d_bases;
    d.quals = d_quals;
    d.seq_begin = d_sb;
    d.seq_end = d_se;
    PoaRun(c, nb, h_wf.data(), h_so.data(), h_sb.data(), h_se.data(), d, a.m, a.n, a.gap,
           a.trim, a.tgs, false);
    std::copy(c.po_h_status.begin(), c.po_h_status.end(), status.begin() + w0);
    for (uint32_t i = 0; i < nb; ++i) {
      cons_off[w0 + i + 1] = cons_off[w0] + c.po_out_off[i + 1];
    }
    cons.insert(cons.end(), c.po_out_cons.begin(), c.po_out_cons.end());
    for (int k = 0; k < 3; ++k) {
      routes[k] += c.po_route_windows[k];
      launches[k] += c.po_route_launches[k];
    }
    cells += c.po_cells;
    ++c.po_batches;
    w0 = w1;
  }
  c.po_out_cons.swap(cons);
  c.po_out_off.swap(cons_off);
  c.po_h_status.swap(status);
  for (int k = 0; k < 3; ++k) {
    c.po_route_windows[k] = routes[k];
    c.po_route_launches[k] = launches[k];
  }
  c.po_cells = cells;
  c.po_n_windows = n_windows;
  c.po_has_cov = false;
  c.poa_valid = true;
}

}  // namespace rvn
