// raven_b200 — the host drivers of the overlap stages: raven::FindOverlapsAndCreatePiles
// (RavenLib/src/construct.cc:14-121) and the device work of
// raven::FindOverlapsAndRepetetiveRegions (construct.cc:352-424), rvn_minimize, rvn_filter
// and rvn_map's flushes, with the schedule and the device-memory estimates they run by.
#include <algorithm>
#include <cstring>
#include <functional>
#include <memory>

#include <unistd.h>

#include "engine.cuh"

namespace rvn {
namespace {

// The reference's schedule (construct.cc:36-112): index batches [j, end) of >= ib
// bases, and per batch the flushes of its queries - every read up to the end of
// the batch - per >= qb bases (the truncation rule makes the flush boundaries
// observable). ib, qb 0: the reference's 2^32 and 2^30.
struct Batch {
  uint32_t j, end;
  std::vector<std::pair<uint32_t, uint32_t>> flushes;  // [k0, k1)
};

std::vector<Batch> Schedule(const Ctx& c, uint64_t ib, uint64_t qb) {
  if (ib == 0) ib = 1ULL << 32;
  if (qb == 0) qb = 1ULL << 30;
  std::vector<Batch> out;
  const std::vector<uint32_t> batches = ChunkCuts(c, 0, c.n_reads, ib);
  for (size_t i = 0; i + 1 < batches.size(); ++i) {
    Batch b{batches[i], batches[i + 1], {}};
    const std::vector<uint32_t> flushes = ChunkCuts(c, 0, b.end, qb);
    for (size_t k = 0; k + 1 < flushes.size(); ++k) {
      b.flushes.emplace_back(flushes[k], flushes[k + 1]);
    }
    out.push_back(std::move(b));
  }
  return out;
}

// Largest max_overlaps a windowed pass takes: it keeps that many records per read.
constexpr uint64_t kWindowMaxOverlaps = 1ULL << 16;
// Device working set of one index batch (sketch, tiers, bare keys, bucket table,
// self-join slots, one flush's hits, with the buffers' headroom) per base of the
// batch: a C2 pass (one 1.98 Gbp batch) holds 43.6 GB in all (DESIGN.md §3, §5).
constexpr double kBatchBytesPerBase = 21.0;
// The same for a chunked build (BuildIndexChunked), from the per-buffer breakdown of a C2
// pass (DESIGN.md §3), as three parts that grow with different sizes:
// - per base of the batch: the index the flushes probe (i_val, i_org, i_bucket, j_packed:
//   1.8 B) and the build's sort buffers and bare keys, freed before the flushes but held
//   next to the flush buffers of an earlier batch or pass (i_*_alt, t_b0, t_b1: 3.3 B);
// - per base of one chunk: its sketch in sweep 1 (sk.val, sk.org: 4.7 B);
// - per query base of the largest flush: the flush's hits, chain scratch and overlaps,
//   and on the probe path its queries' sketch and sorted micromizers. 27 B is the
//   remainder of the 59.9 GB peak of a 2^32-base batch with 2^30-base query flushes
//   (DESIGN.md §5); C2's join-only flushes hold 18.4 B.
constexpr double kIndexBytesPerBase = 1.8 + 3.3;
constexpr double kChunkSketchBytesPerBase = 4.7;
constexpr double kFlushBytesPerBase = 27.0;
// chunk size of option "index_chunk_bases" -1 (auto)
constexpr uint64_t kAutoIndexChunk = 1ULL << 30;

// Device working set of the largest index batch, one-shot (chunk 0) or in chunks of
// `chunk` bases.
double IndexFootprint(const Ctx& c, const std::vector<Batch>& batches, uint64_t chunk) {
  uint64_t batch_bases = 0, flush_bases = 0;
  for (const Batch& b : batches) {
    batch_bases = std::max(batch_bases, ReadBases(c, b.j, b.end));
    for (const auto& f : b.flushes) {
      flush_bases = std::max(flush_bases, ReadBases(c, f.first, f.second));
    }
  }
  const double bb = static_cast<double>(batch_bases);
  const double one_shot = kBatchBytesPerBase * bb;
  if (chunk == 0) return one_shot;
  // (a chunked build holds a subset of the one-shot build's buffers: below a few Gbp
  // the flush's working set dominates and chunks save little)
  return std::min(one_shot, kIndexBytesPerBase * bb +
                                kChunkSketchBytesPerBase * std::min(bb, static_cast<double>(chunk)) +
                                kFlushBytesPerBase * static_cast<double>(flush_bases));
}

// Words of the largest read range a pass sketches: an index batch, or one chunk of it
// (chunk > 0), or a query flush.
uint64_t LargestSketchWords(const Ctx& c, const std::vector<Batch>& batches, uint64_t chunk) {
  uint64_t words = 0;
  auto range = [&](uint32_t a, uint32_t b) { words = std::max(words, c.h_woff[b] - c.h_woff[a]); };
  for (const Batch& b : batches) {
    if (chunk) {
      const std::vector<uint32_t> cuts = ChunkCuts(c, b.j, b.end, chunk);
      for (size_t i = 0; i + 1 < cuts.size(); ++i) range(cuts[i], cuts[i + 1]);
    } else {
      range(b.j, b.end);
    }
    for (const auto& f : b.flushes) range(f.first, f.second);
  }
  return words;
}

// Device bytes of the packed bases during a pass: the whole set, or with the bases on the
// host the two halves of the staging window, each as large as the largest range sketched.
double BasesBytes(const Ctx& c, const std::vector<Batch>& batches, uint64_t chunk, bool host) {
  if (!host) return 8.0 * c.n_words;
  return 2.0 * 8.0 * static_cast<double>(LargestSketchWords(c, batches, chunk));
}

// Estimated memory of a stage-1 pass over the uploaded reads, in bytes.
struct Footprint {
  double resident = 0;         // device, resident pass
  double windowed_device = 0;  // device, windowed pass
  double windowed_host = 0;    // pinned host, windowed pass
};

// Both modes hold the reads (packed bases, offsets, lengths, ids, pile offsets)
// and the working set of the largest index batch. On top of that:
// - resident: all piles (u16 per bin) and their difference array (i32 per bin and
//   read), and the lists in two copies plus the staging list and its sort keys.
//   A list keeps at most kmax records; the estimate also takes one overlap per
//   other read as the most a list gathers, since the compact lists only hold what
//   was kept.
// - windowed, on the device: the same per slot of the largest window, with kmax
//   (at least 1) records per list row; on the host: the rows, counts and piles of
//   all reads.
// chunk: the index build's chunk size (0: one-shot), see IndexFootprint; host: the bases
// are on the host (BasesBytes)
Footprint Stage1Footprint(const Ctx& c, const std::vector<Batch>& batches, uint64_t kmax,
                          uint64_t chunk, bool host) {
  const uint32_t n = c.n_reads;
  const std::vector<uint64_t>& off = c.h_pile_off;
  const double bins = static_cast<double>(off[n]);
  const double stride = static_cast<double>(std::max<uint64_t>(kmax, 1));
  const double list_bytes = 3.0 * sizeof(rvn_overlap) + 8.0;  // per record
  double window = 0;  // device bytes of the largest window
  for (const Batch& b : batches) {
    for (const auto& f : b.flushes) {
      const uint32_t a0 = std::min(f.first, b.j), a1 = std::min(f.second, b.j);
      const double slots = (b.end - b.j) + (a1 - a0);
      const double wbins = static_cast<double>((off[b.end] - off[b.j]) + (off[a1] - off[a0]));
      window = std::max(window, 6.0 * wbins + 4.0 * slots + slots * stride * list_bytes);
    }
  }
  const double reads =
      BasesBytes(c, batches, chunk, host) + 32.0 * n + IndexFootprint(c, batches, chunk);
  const double kept = std::min(static_cast<double>(kmax), n > 0 ? n - 1.0 : 0.0);
  Footprint f;
  f.resident = reads + 6.0 * bins + 4.0 * n + n * kept * list_bytes;
  f.windowed_device = reads + window;
  f.windowed_host = n * stride * sizeof(rvn_overlap) + 4.0 * n + 2.0 * bins;
  return f;
}

// Option "index_chunk_bases": the chunk size of an index build, 0 = one-shot.
// -1 (auto): chunks of kAutoIndexChunk bases only when `one_shot`, the caller's estimate
// of its device memory with one-shot builds, exceeds the usable memory
// ("index_chunk_budget" replaces it when it is not 0).
uint64_t IndexChunk(const Ctx& c, double one_shot) {
  if (c.index_chunk_bases >= 0) return static_cast<uint64_t>(c.index_chunk_bases);
  return one_shot > UsableMemory(c, c.index_chunk_budget) ? kAutoIndexChunk : 0;
}

// a stage-1 pass with one-shot builds: resident, or windowed (max_overlaps permitting)
double Stage1OneShot(const Ctx& c, const std::vector<Batch>& batches, uint64_t kmax) {
  const Footprint f = Stage1Footprint(c, batches, kmax, 0, c.bases.on_host);
  return kmax <= kWindowMaxOverlaps ? std::min(f.resident, f.windowed_device) : f.resident;
}

// The untiered index rvn_minimize builds holds every record of the batch: values, origins
// and the sort's second buffers (two copies of 12 B for an estimated 0.34 records per base,
// with the buffers' headroom) and the bucket table. Estimate, not measured.
constexpr double kUntieredIndexBytesPerBase = 8.9;

// Device memory of rvn_minimize over reads [first, last): the reads, the untiered index and
// the sketch of the batch (one-shot, chunk 0) or of one chunk of `chunk` bases.
double MinimizeFootprint(const Ctx& c, uint32_t first, uint32_t last, uint64_t chunk) {
  const double bb = static_cast<double>(ReadBases(c, first, last));
  const double sketched = chunk ? std::min(bb, static_cast<double>(chunk)) : bb;
  const std::vector<Batch> batch{Batch{first, last, {}}};
  return BasesBytes(c, batch, chunk, c.bases.on_host) + 32.0 * c.n_reads +
         kUntieredIndexBytesPerBase * bb + kChunkSketchBytesPerBase * sketched;
}

// rvn_map works its query range in flushes, as the reference cuts its queries
// (construct.cc:67): at most kMapFlushCeiling bases, fewer when the device has no room for
// the per-query-base working set of a flush (kFlushBytesPerBase on the probe path,
// kJoinFlushBytesPerBase for the self-join, DESIGN.md §3). A range of up to kMapFlushFloor
// bases is never cut.
constexpr uint64_t kMapFlushCeiling = 1ULL << 30;
constexpr uint64_t kMapFlushFloor = 1ULL << 24;
constexpr double kJoinFlushBytesPerBase = 18.4;

uint64_t MapFlushBases(const Ctx& c, uint64_t range_bases, bool join) {
  if (c.map_flush_bases) return c.map_flush_bases;
  if (range_bases <= kMapFlushFloor) return kMapFlushCeiling;
  // a flush can grow into the free memory and into every buffer of the context but the
  // reads and the index
  auto bytes = [](const auto& b) { return static_cast<double>(b.cap * sizeof(*b.p)); };
  const double fixed = bytes(c.d_words) + static_cast<double>(StagedBaseBytes(c)) +
                       bytes(c.i_val) + bytes(c.i_org) + bytes(c.i_val_alt) +
                       bytes(c.i_org_alt) + bytes(c.i_bucket) + bytes(c.j_packed);
  const double room = UsableMemory(c, 0) - fixed;
  const double flush = room / (join ? kJoinFlushBytesPerBase : kFlushBytesPerBase);
  if (flush >= static_cast<double>(kMapFlushCeiling)) return kMapFlushCeiling;
  return std::max(kMapFlushFloor, static_cast<uint64_t>(std::max(flush, 0.0)));
}

// Option "stage1_window" -1 (auto): windowed only when the resident estimate exceeds
// the usable device memory ("stage1_window_budget" replaces it when it is not 0) and the
// windowed pass itself fits: it takes kmax, its own device estimate fits the same memory
// and its host rows fit the host's free physical memory. Otherwise resident, as before
// the option existed.
bool UseWindow(Ctx& c, const std::vector<Batch>& batches, uint64_t kmax, uint64_t chunk) {
  if (c.stage1_window >= 0) return c.stage1_window != 0;
  if (kmax > kWindowMaxOverlaps) return false;
  const Footprint f = Stage1Footprint(c, batches, kmax, chunk, c.bases.on_host);
  const double budget = UsableMemory(c, c.stage1_window_budget);
  if (f.resident <= budget) return false;
  const double host_free = static_cast<double>(sysconf(_SC_AVPHYS_PAGES)) *
                           static_cast<double>(sysconf(_SC_PAGESIZE));
  return f.windowed_device <= budget && f.windowed_host <= host_free;
}

// Windowed stage 1: the piles (c.st_pile) and kept lists of all reads stay on the
// host, the lists in rows of kmax records plus a count per read (c.w_rows, c.w_cnt).
// A flush brings the reads it touches - its Window - to the device: the index
// batch's piles and lists stay there for the whole batch, those of the flush's
// queries before the batch come and go with the flush. Same kernels as the
// resident pass, on window slots; results land in st_ovl / st_ovl_off / st_pile.
class WindowedStage1 {
 public:
  WindowedStage1(Ctx& c, uint64_t kmax, uint64_t total_bins)
      : c_(c), kmax_(kmax), stride_(std::max<uint64_t>(kmax, 1)) {
    if (kmax > kWindowMaxOverlaps) {
      throw LimitError("windowed stage 1 keeps max_overlaps records per read: at most 65536");
    }
    const uint64_t n = c.n_reads;
    rows_ = c.w_rows.reserve(n * stride_ + 1);
    cnt_ = c.w_cnt.reserve(n + 1);
    std::memset(cnt_, 0, (n + 1) * sizeof(uint32_t));
    pile_ = c.st_pile.reserve(total_bins + 1);
    std::memset(pile_, 0, (total_bins + 1) * sizeof(uint16_t));
  }

  // reads of [j, end) have neither piles nor lists yet: the batch part starts empty
  void BeginBatch(const Batch& b) {
    const std::vector<uint64_t>& off = c_.h_pile_off;
    j_ = b.j;
    end_ = b.end;
    nb_ = end_ - j_;
    bb_ = off[end_] - off[j_];
    uint64_t max_a = 0, max_a_bins = 0;
    for (const auto& f : b.flushes) {
      const uint32_t a0 = std::min(f.first, j_), a1 = std::min(f.second, j_);
      max_a = std::max<uint64_t>(max_a, a1 - a0);
      max_a_bins = std::max(max_a_bins, off[a1] - off[a0]);
    }
    // sized once per batch: growing a buffer does not keep its contents
    const uint64_t slots = nb_ + max_a;
    c_.g_list[0].reserve(slots * stride_ + 1);
    c_.g_list[1].reserve(slots * stride_ + 1);
    c_.g_cnt.reserve(slots + 1);
    c_.g_kept.reserve(slots + 1);
    c_.w_row_off.reserve(slots + 2);
    c_.w_pile_off.reserve(slots + 2);
    c_.p_data.reserve(bb_ + max_a_bins + 1);
    RVN_CUDA(cudaMemsetAsync(c_.g_cnt.get(), 0, nb_ * sizeof(uint32_t), c_.stream));
    RVN_CUDA(cudaMemsetAsync(c_.p_data.get(), 0, bb_ * sizeof(uint16_t), c_.stream));
  }

  // the overlaps MapRange left in c.m_ovl for the queries [k0, k1)
  void Flush(uint32_t k0, uint32_t k1) {
    if (c_.r_n_ovl == 0) return;
    const std::vector<uint64_t>& off = c_.h_pile_off;
    const Window w{j_, end_, std::min(k0, j_), std::min(k1, j_)};
    const uint32_t na = w.a1 - w.a0;
    const uint64_t a_bins = off[w.a1] - off[w.a0];
    TimerBegin(c_, "stage1_window");
    Move(w, cudaMemcpyHostToDevice);
    WindowTables(c_, w, c_.p_off.get(), stride_, c_.w_row_off.get(), c_.w_pile_off.get());
    TimerEnd(c_);
    PileAddLayersDevice(c_, c_.p_data.get(), c_.w_pile_off.get(), bb_ + a_bins, w,
                        c_.m_ovl.get(), c_.r_n_ovl);
    GatherFlush(c_, c_.m_ovl.get(), c_.m_ovl_off.get(), c_.r_n_ovl, k0, k1, kmax_, w,
                c_.w_row_off.get(), stride_);
    if (na) {
      TimerBegin(c_, "stage1_window");
      Move(w, cudaMemcpyDeviceToHost);
      TimerEnd(c_);
    }
  }

  // the batch part goes back to the host
  void EndBatch() {
    TimerBegin(c_, "stage1_window");
    Move(Window{j_, end_, 0, 0}, cudaMemcpyDeviceToHost, /*batch=*/true);
    TimerEnd(c_);
  }

  // compact lists, as the resident pass leaves them
  void Fetch() {
    RVN_CUDA(cudaStreamSynchronize(c_.stream));
    const uint32_t n = c_.n_reads;
    uint64_t* ooff = c_.st_ovl_off.reserve(n + 1ULL);
    ooff[0] = 0;
    for (uint32_t r = 0; r < n; ++r) ooff[r + 1] = ooff[r] + cnt_[r];
    rvn_overlap* o = c_.st_ovl.reserve(ooff[n] + 1);
    for (uint32_t r = 0; r < n; ++r) {
      std::memcpy(o + ooff[r], rows_ + r * stride_, cnt_[r] * sizeof(rvn_overlap));
    }
  }

 private:
  // the query part of `w` (or the batch part) between its host home and the device
  void Move(const Window& w, cudaMemcpyKind kind, bool batch = false) {
    const uint32_t r0 = batch ? w.b0 : w.a0, r1 = batch ? w.b1 : w.a1;
    if (r1 == r0) return;
    const uint64_t slot0 = batch ? 0 : nb_;
    const uint64_t bin0 = batch ? 0 : bb_;
    const std::vector<uint64_t>& off = c_.h_pile_off;
    const bool up = kind == cudaMemcpyHostToDevice;
    auto copy = [&](void* dev, void* host, uint64_t bytes) {
      if (bytes) {
        RVN_CUDA(cudaMemcpyAsync(up ? dev : host, up ? host : dev, bytes, kind, c_.stream));
      }
    };
    copy(c_.g_cnt.get() + slot0, cnt_ + r0, (r1 - r0) * sizeof(uint32_t));
    copy(c_.g_list[c_.g_cur].get() + slot0 * stride_, rows_ + r0 * stride_,
         (r1 - r0) * stride_ * sizeof(rvn_overlap));
    copy(c_.p_data.get() + bin0, pile_ + off[r0], (off[r1] - off[r0]) * sizeof(uint16_t));
  }

  Ctx& c_;
  const uint64_t kmax_, stride_;
  rvn_overlap* rows_;
  uint32_t* cnt_;
  uint16_t* pile_;
  uint32_t j_ = 0, end_ = 0, nb_ = 0;
  uint64_t bb_ = 0;
};

// Reads whose piles and lists no flush after flush i of the schedule touches (flushes in
// schedule order): every stage-1 overlap has rhs_id > lhs_id and a flush over the queries
// [k0, k1) only names reads >= k0, so after flush i that is every read below the first
// query of every flush still to run - n after the last flush, 0 before the last index
// batch (each batch's flushes start at read 0 again). Such a read's pile gets no marks
// (the coverage pass skips it), ListTotals gives its list the old count, at most kmax, which
// Truncate leaves alone, and its compact offset is a prefix of the same scan.
std::vector<uint32_t> FinalReads(const std::vector<Batch>& batches, uint32_t n) {
  std::vector<uint32_t> first;
  for (const Batch& b : batches) {
    for (const auto& f : b.flushes) first.push_back(f.first);
  }
  std::vector<uint32_t> out(first.size());
  uint32_t fin = n;
  for (size_t i = first.size(); i-- > 0;) {
    out[i] = fin;
    fin = std::min(fin, first[i]);
  }
  return out;
}

// The pinned list buffer is sized up front for min(kmax, n - 1) records per read: lists of
// more records per read than this, or more bytes in all, are not streamed.
constexpr uint64_t kStreamMaxOverlaps = 256;
constexpr uint64_t kStreamMaxListBytes = 8ULL << 30;

// Resident stage 1, option "stage1_stream": the piles and lists of the reads that are
// final (FinalReads) go to the pinned host results on c.d2h_stream while the later
// flushes run, the piles right after a flush's coverage pass, the lists after its gather.
// Sources: the final prefix of c.p_data, which no later coverage pass touches, and of
// the current list buffer and offsets, which the gather two flushes later overwrites;
// c.stream waits for all copies issued so far before every gather (BeforeGather) and at
// the end (Finish). The pinned buffers are sized before the first copy.
class ResultStream {
 public:
  ResultStream(Ctx& c, uint64_t kmax, uint64_t total_bins) : c_(c) {
    const uint32_t n = c.n_reads;
    if (!c.d2h_stream) {
      RVN_CUDA(cudaStreamCreateWithFlags(&c.d2h_stream, cudaStreamNonBlocking));
      RVN_CUDA(cudaEventCreateWithFlags(&c.d2h_ready, cudaEventDisableTiming));
      RVN_CUDA(cudaEventCreateWithFlags(&c.d2h_done, cudaEventDisableTiming));
    }
    c.st_pile.reserve(total_bins + 1);
    c.st_ovl_off.reserve(n + 1ULL)[0] = 0;
    per_read_ = std::min<uint64_t>(kmax, n ? n - 1 : 0);
    // a larger kmax: the lists go to the host after the last flush, as without streaming
    lists_ = per_read_ <= kStreamMaxOverlaps &&
             per_read_ * n * sizeof(rvn_overlap) <= kStreamMaxListBytes;
    if (lists_) c.st_ovl.reserve(per_read_ * n + 1);
  }
  // (a pass that throws leaves no copy into the pinned buffers behind)
  ~ResultStream() { cudaStreamSynchronize(c_.d2h_stream); }

  bool lists() const { return lists_; }

  // the piles of reads below `final` are final: c.p_data after the coverage pass
  void Piles(uint32_t final) {
    if (final <= pile_read_) return;
    const std::vector<uint64_t>& off = c_.h_pile_off;
    const uint64_t b0 = off[pile_read_], b1 = off[final];
    pile_read_ = final;
    if (b1 == b0) return;
    Begin();
    RVN_CUDA(cudaMemcpyAsync(c_.st_pile.get() + b0, c_.p_data.get() + b0,
                             (b1 - b0) * sizeof(uint16_t), cudaMemcpyDeviceToHost,
                             c_.d2h_stream));
    End();
  }

  // the lists of reads below `final` are final; final_off: their records (the gather's
  // compact offset of `final`)
  void Lists(uint32_t final, uint64_t final_off) {
    if (!lists_ || final <= list_read_) return;
    if (final_off + 1 > c_.st_ovl.cap) {
      // more than min(kmax, n - 1) records per read: grow once the copies are through
      RVN_CUDA(cudaStreamSynchronize(c_.d2h_stream));
      c_.st_ovl.reserve_keep(final_off + per_read_ * (c_.n_reads - final) + 1, list_off_);
    }
    Begin();
    RVN_CUDA(cudaMemcpyAsync(c_.st_ovl_off.get() + list_read_ + 1,
                             c_.g_off.get() + list_read_ + 1,
                             (final - list_read_) * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                             c_.d2h_stream));
    if (final_off > list_off_) {
      RVN_CUDA(cudaMemcpyAsync(c_.st_ovl.get() + list_off_,
                               c_.g_list[c_.g_cur].get() + list_off_,
                               (final_off - list_off_) * sizeof(rvn_overlap),
                               cudaMemcpyDeviceToHost, c_.d2h_stream));
    }
    End();
    list_read_ = final;
    list_off_ = final_off;
  }

  void BeforeGather() {
    if (issued_) RVN_CUDA(cudaStreamWaitEvent(c_.stream, c_.d2h_done, 0));
  }

  // after the last flush: c.stream waits for every copy (the lists follow when they
  // were not streamed)
  void Finish() {
    BeforeGather();
    if (!lists_) GatherFetch(c_);
  }

 private:
  void Begin() {
    RVN_CUDA(cudaEventRecord(c_.d2h_ready, c_.stream));
    RVN_CUDA(cudaStreamWaitEvent(c_.d2h_stream, c_.d2h_ready, 0));
  }
  void End() {
    RVN_CUDA(cudaEventRecord(c_.d2h_done, c_.d2h_stream));
    issued_ = true;
  }

  Ctx& c_;
  uint64_t per_read_ = 0;
  bool lists_ = false, issued_ = false;
  uint32_t pile_read_ = 0, list_read_ = 0;  // reads whose piles / lists are on their way
  uint64_t list_off_ = 0;                   // records of list_read_ reads
};

}  // namespace

// rvn_minimize: the untiered index of reads [first, last), which full sketches may probe,
// in chunks when IndexChunk says so (the build's buffers are then held until Filter)
void Minimize(Ctx& c, uint32_t first, uint32_t last, bool minhash) {
  const uint64_t chunk = IndexChunk(c, MinimizeFootprint(c, first, last, 0));
  if (chunk) {
    BuildIndexChunked(c, first, last, minhash, chunk, 0, /*tiers=*/false);
    c.i_build_held = true;
  } else {
    BuildIndex(c, first, last, minhash);
  }
}

uint32_t Filter(Ctx& c, double freq) {
  const uint32_t occ = FilterIndex(c, freq);
  if (c.i_build_held) {
    ReleaseIndexBuild(c);
    c.i_build_held = false;
  }
  return occ;
}

// rvn_map: MapRange flush by flush, each flush's overlaps, offsets and filtered positions
// appended to the pinned host results, so that they read as one MapRange over the range.
// One flush (and keep_hits, whose hits are those of one piece) is exactly that MapRange.
// each (stage 2): called with (first read, reads) after every flush, whose results it
// takes from the device (c.m_ovl, c.m_ovl_off, c.r_n_ovl, c.m_filtered); nothing is
// gathered on the host.
void MapFlushes(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal, bool avoid_symmetric,
                bool minhash, bool want_filtered,
                const std::function<void(uint32_t, uint32_t)>& each) {
  const bool join = c.self_join && minhash && avoid_equal && avoid_symmetric && !want_filtered &&
                    first >= c.i_first && last <= c.i_last;
  const std::vector<uint32_t> cuts =
      ChunkCuts(c, first, last, MapFlushBases(c, ReadBases(c, first, last), join));
  // staged bases: each probe-path flush's sketch is followed by the copy of the next flush's
  auto stage_next = [&](size_t i) {
    if (!join && i + 2 < cuts.size()) BasesNext(c, cuts[i + 1], cuts[i + 2]);
  };
  if (each) {
    for (size_t i = 0; i + 1 < cuts.size(); ++i) {
      stage_next(i);
      MapRange(c, cuts[i], cuts[i + 1], avoid_equal, avoid_symmetric, minhash, want_filtered,
               /*fetch=*/false);
      each(cuts[i], cuts[i + 1] - cuts[i]);
    }
    return;
  }
  if (c.keep_hits || cuts.size() <= 2) {
    MapRange(c, first, last, avoid_equal, avoid_symmetric, minhash, want_filtered);
    return;
  }
  const uint32_t nr = last - first;
  uint64_t* off = c.a_ovl_off.reserve(nr + 2ULL);
  uint64_t* foff = c.a_filt_off.reserve(nr + 2ULL);
  off[0] = foff[0] = 0;
  uint64_t total = 0, f_total = 0;
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    const uint32_t r0 = cuts[i], m = cuts[i + 1] - cuts[i];
    stage_next(i);
    MapRange(c, r0, r0 + m, avoid_equal, avoid_symmetric, minhash, want_filtered,
             /*fetch=*/false);
    TimerBegin(c, "map_flush");
    const uint64_t n = c.r_n_ovl;
    rvn_overlap* o = c.a_ovl.reserve_keep(total + n + 1, total);
    uint64_t* o_off = off + (r0 - first);
    RVN_CUDA(cudaMemcpyAsync(o + total, c.m_ovl.get(), n * sizeof(rvn_overlap),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(o_off + 1, c.m_ovl_off.get() + 1, m * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, c.stream));
    TimerEnd(c);
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    for (uint32_t r = 1; r <= m; ++r) o_off[r] += total;
    // (MapRange leaves the flush's filtered positions on the host)
    const uint64_t* ff = c.r_filt_off.get();
    const uint64_t nf = ff[m];
    uint32_t* f = c.a_filtered.reserve_keep(f_total + nf + 1, f_total);
    if (nf) std::memcpy(f + f_total, c.r_filtered.get(), nf * sizeof(uint32_t));
    for (uint32_t r = 1; r <= m; ++r) foff[r0 - first + r] = f_total + ff[r];
    total += n;
    f_total += nf;
  }
  c.r_ovl.swap(c.a_ovl);
  c.r_ovl_off.swap(c.a_ovl_off);
  c.r_filtered.swap(c.a_filtered);
  c.r_filt_off.swap(c.a_filt_off);
  c.r_n_ovl = total;
  c.m_first_read = first;
  c.m_last_read = last;
  c.r_valid = true;
}

// raven::FindOverlapsAndRepetetiveRegions' device work (construct.cc:352-424) over the
// first n valid reads of the uploaded set, in the reference's sorted order: index
// batches [j, end) cut by the reference's rule (bytes < 1U << 30; option
// "stage2_batch_bases" forces a smaller batch), each an untiered full-sketch index
// filtered at freq, then every read of [0, end) mapped with (avoid equal, avoid
// symmetric, no minhash, filtered positions) in rvn_map's flushes. Per flush, on the
// device: the filtered positions mark the k-mer bitmaps (Pile::AddKmers), and with
// identity != 0 the overlaps are clipped to the valid regions (rbeg, rend: Pile::begin()
// and end() per valid read) and filtered by edit distance. Only the final overlaps, and
// at the end the bitmaps and touched flags, go to the pinned host results.
void Stage2(Ctx& c, double freq, double identity, uint32_t n, const uint32_t* h_rbeg,
            const uint32_t* h_rend) {
  if (n > c.n_reads) throw InvalidArgument("more valid reads than uploaded reads");
  if (n && (!h_rbeg || !h_rend)) throw InvalidArgument("null regions");
  CheckResident(c, 0, n);
  c.s2_valid = false;
  uint32_t max_id = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (h_rbeg[i] > h_rend[i] || h_rend[i] > c.h_len[i]) {
      throw InvalidArgument("region outside its read");
    }
    max_id = std::max(max_id, c.h_ids[i]);
  }
  // read id -> position in the uploaded set (construct.cc:331-337's sequences_map)
  std::vector<uint32_t> pos_of(max_id + 1ULL, 0);
  for (uint32_t i = 0; i < n; ++i) pos_of[c.h_ids[i]] = i;
  uint64_t* boff = c.s2_bit_off_h.reserve(n + 1ULL);
  boff[0] = 0;
  for (uint32_t i = 0; i < n; ++i) boff[i + 1] = boff[i] + ((c.h_len[i] >> 4) + 1 + 31) / 32;
  uint32_t* d_pos_of = c.s2_pos_of.reserve(pos_of.size());
  uint32_t* d_rbeg = c.s2_rbeg.reserve(n + 1ULL);
  uint32_t* d_rend = c.s2_rend.reserve(n + 1ULL);
  uint64_t* d_boff = c.s2_bit_off.reserve(n + 1ULL);
  uint32_t* d_bits = c.s2_bits.reserve(boff[n] + 1);
  uint8_t* d_touched = c.s2_touched.reserve(n + 1ULL);
  RVN_CUDA(cudaMemcpyAsync(d_pos_of, pos_of.data(), pos_of.size() * 4, cudaMemcpyHostToDevice,
                           c.stream));
  if (n) {
    RVN_CUDA(cudaMemcpyAsync(d_rbeg, h_rbeg, n * 4ULL, cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(d_rend, h_rend, n * 4ULL, cudaMemcpyHostToDevice, c.stream));
  }
  RVN_CUDA(cudaMemcpyAsync(d_boff, boff, (n + 1ULL) * 8, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_bits, 0, (boff[n] + 1) * 4, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_touched, 0, n + 1ULL, c.stream));

  uint64_t* ooff = c.s2_ovl_off.reserve(n + 1ULL);
  ooff[0] = 0;
  c.s2_ovl.reserve_keep(1, 0);
  uint64_t total = 0, mapped = 0;
  auto flush = [&](uint32_t r0, uint32_t m) {
    Stage2KmerMarks(c, r0, m, c.prm.k);
    const uint64_t nm = c.r_n_ovl;
    mapped += nm;
    const rvn_overlap* src = c.m_ovl.get();
    uint64_t kept = nm;
    if (identity != 0) {  // with identity 0 the overlaps pass unchanged (construct.cc:385)
      rvn_overlap* dst = c.s2_kept.reserve(nm + 1);
      uint64_t* dst_off = c.s2_kept_off.reserve(m + 1ULL);
      kept = Stage2ClipFilter(c, c.m_ovl.get(), c.m_ovl_off.get(), m, nm, identity, dst, dst_off);
      src = dst;
    }
    rvn_overlap* o = c.s2_ovl.reserve_keep(total + kept + 1, total);
    RVN_CUDA(cudaMemcpyAsync(o + total, src, kept * sizeof(rvn_overlap), cudaMemcpyDeviceToHost,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    total += kept;
  };
  struct HostFiltered {  // the filtered positions stay on the device for the whole call
    Ctx& c;
    explicit HostFiltered(Ctx& x) : c(x) { c.m_filtered_host = false; }
    ~HostFiltered() { c.m_filtered_host = true; }
  } keep_on_device(c);
  const std::vector<uint32_t> cuts =
      ChunkCuts(c, 0, n, c.stage2_batch_bases ? c.stage2_batch_bases : (1ULL << 30));
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    const uint32_t j = cuts[i], end = cuts[i + 1];
    // a read that does not end a batch: the empty range at the total before its batch
    std::fill(ooff + j + 1, ooff + end, total);
    Minimize(c, j, end, false);
    Filter(c, freq);
    MapFlushes(c, 0, end, true, true, false, true, flush);
    ooff[end] = total;
  }
  uint32_t* bits = c.s2_bits_h.reserve(boff[n] + 1);
  uint8_t* touched = c.s2_touched_h.reserve(n + 1ULL);
  RVN_CUDA(cudaMemcpyAsync(bits, d_bits, boff[n] * 4, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(touched, d_touched, n, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  c.s2_n_valid = n;
  c.s2_mapped = mapped;
  c.s2_valid = true;
}

// raven::FindOverlapsAndCreatePiles, same batch / flush schedule as the
// reference; every step runs on the GPU (Minimize, Filter, Map, AddLayers,
// gather, truncation); the host only drives the schedule (and, windowed, keeps
// the piles and lists of the reads a flush does not touch).
void Stage1(Ctx& c, double freq, uint64_t kmax, bool minhash, uint64_t ib,
            uint64_t qb) {
  if (!(0 <= freq && freq <= 1)) {
    throw InvalidArgument(
        "[ram::MinimizerEngine::Filter] error: invalid frequency");
  }
  if (!c.ids_identity) {
    throw StateError("stage 1 needs read ids equal to their index");
  }
  c.st_valid = false;
  c.st_piles_on_device = false;
  c.own_mod = 1;
  c.own_rem = 0;
  // a stage-1 pass owns its intermediates: nothing is carried over from an
  // earlier call (sketches, micromizers and the index are rebuilt)
  MarkStale(c, Stale::kIndex);
  TimerReset(c);
  std::memset(&c.stats, 0, sizeof(c.stats));
  const uint64_t launches0 = c.launches;
  const uint32_t n = c.n_reads;
  const uint64_t total_bins = c.h_pile_off[n];
  const std::vector<Batch> batches = Schedule(c, ib, qb);
  const uint64_t chunk = IndexChunk(c, Stage1OneShot(c, batches, kmax));
  const bool windowed = UseWindow(c, batches, kmax, chunk);
  c.st_windowed = false;
  uint16_t* d_pile = nullptr;
  if (!windowed) {
    d_pile = c.p_data.reserve(total_bins + 1);
    RVN_CUDA(cudaMemsetAsync(d_pile, 0, (total_bins + 1) * sizeof(uint16_t), c.stream));
  }
  uint64_t* d_poff = c.p_off.reserve(n + 1ULL);
  if (!c.p_off_uploaded) {  // (an asynchronous upload has sent them ahead of the bases)
    RVN_CUDA(cudaMemcpyAsync(d_poff, c.h_pile_off.data(), (n + 1ULL) * 8,
                             cudaMemcpyHostToDevice, c.stream));
  }

  GatherReset(c);
  c.st_mapped = 0;
  std::unique_ptr<WindowedStage1> win;
  if (windowed) win.reset(new WindowedStage1(c, kmax, total_bins));
  std::unique_ptr<ResultStream> out;
  if (!windowed && c.stage1_stream) out.reset(new ResultStream(c, kmax, total_bins));
  const std::vector<uint32_t> final_reads = FinalReads(batches, n);
  size_t flush = 0;  // index of the flush in the schedule

  // Staged bases: the range sketched after each sketch, copied beside the kernels that read
  // no bases - the batch's first range (itself, or its first chunk), then the flushes that
  // probe (those that are not inside the batch, or all of them with minhash), then the
  // next batch's first range. next_sketch[i]: the first such range from batch i's flushes on.
  auto probes = [&](const Batch& b, const std::pair<uint32_t, uint32_t>& f) {
    return !(c.self_join && !minhash && f.first >= b.j && f.second <= b.end);
  };
  auto first_range = [&](const Batch& b) {
    const std::vector<uint32_t> cuts = ChunkCuts(c, b.j, b.end, chunk ? chunk : ~0ULL);
    return std::make_pair(cuts[0], cuts[1]);
  };
  auto stage_after = [&](size_t bi, size_t fi) {  // the range after flush fi - 1 of batch bi
    if (!c.bases.on_host) return;
    for (size_t i = fi; i < batches[bi].flushes.size(); ++i) {
      if (probes(batches[bi], batches[bi].flushes[i])) {
        BasesNext(c, batches[bi].flushes[i].first, batches[bi].flushes[i].second);
        return;
      }
    }
    if (bi + 1 < batches.size()) {
      const auto r = first_range(batches[bi + 1]);
      BasesNext(c, r.first, r.second);
    }
  };

  uint64_t tmax = 0;  // largest micromizer value of the reads sketched so far
  for (size_t bi = 0; bi < batches.size(); ++bi) {
    const Batch& b = batches[bi];
    stage_after(bi, 0);
    // Queries are micromizers only (construct.cc:62): no record above the largest
    // micromizer value of any read so far can be hit - those are counted for the
    // occurrence threshold but stay out of the index (index.cu, tiers)
    if (chunk) {
      tmax = BuildIndexChunked(c, b.j, b.end, minhash, chunk, tmax);
      FilterIndex(c, freq);
      ReleaseIndexBuild(c);
    } else {
      uint64_t limit = ~0ULL;
      if (!minhash) {
        tmax = std::max(tmax, MaxMicromizerValue(c, b.j, b.end));
        limit = tmax;
      }
      BuildIndex(c, b.j, b.end, minhash, limit);
      FilterIndex(c, freq);
    }
    if (win) win->BeginBatch(b);

    for (size_t fi = 0; fi < b.flushes.size(); ++fi) {
      const auto& f = b.flushes[fi];
      stage_after(bi, fi + 1);
      MapRange(c, f.first, f.second, true, true, true, false, /*fetch=*/false);
      const uint32_t final = final_reads[flush++];
      if (win) {
        win->Flush(f.first, f.second);
      } else {
        // (the flush names no read below f.first)
        PileAddLayersDevice(c, d_pile, d_poff, total_bins, Window::All(n), c.m_ovl.get(),
                            c.r_n_ovl, f.first);
        uint64_t final_off = 0;
        if (out) {
          out->BeforeGather();
          out->Piles(final);
        }
        GatherFlush(c, c.m_ovl.get(), c.m_ovl_off.get(), c.r_n_ovl, f.first, f.second, kmax,
                    Window::All(n), nullptr, 0, final,
                    out && out->lists() ? &final_off : nullptr);
        if (out) out->Lists(final, final_off);
      }
      c.st_mapped += c.r_n_ovl;
    }
    if (win) win->EndBatch();
  }

  if (win) {
    win->Fetch();
  } else {
    // what of the copy to the host still runs after the last kernel
    TimerBegin(c, "results");
    if (out) {
      out->Finish();
    } else {
      GatherFetch(c);
      RVN_CUDA(cudaMemcpyAsync(c.st_pile.reserve(total_bins + 1), d_pile,
                               total_bins * sizeof(uint16_t), cudaMemcpyDeviceToHost,
                               c.stream));
    }
    TimerEnd(c);
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  TimerCollect(c);
  c.stats.kernel_launches = c.launches - launches0;
  c.stats.occurrence = c.occurrence;
  c.st_valid = true;
  c.st_windowed = windowed;
  c.st_piles_on_device = !windowed;
}

bool UseHostBases(const Ctx& c) {
  if (c.bases.host_bases >= 0) return c.bases.host_bases != 0;
  if (c.n_reads == 0) return false;
  // the windowed, chunked pass of the reference's schedule at its default max_overlaps
  const std::vector<Batch> batches = Schedule(c, 0, 0);
  const double usable = UsableMemory(c, c.bases.host_bases_budget);
  if (Stage1Footprint(c, batches, 32, kAutoIndexChunk, false).windowed_device <= usable) {
    return false;
  }
  return Stage1Footprint(c, batches, 32, kAutoIndexChunk, true).windowed_device <= usable;
}

double UsableMemory(const Ctx& c, uint64_t budget) {
  if (budget) return static_cast<double>(budget);
  size_t free_b = 0, total_b = 0;
  RVN_CUDA(cudaMemGetInfo(&free_b, &total_b));
  return static_cast<double>(free_b) + static_cast<double>(c.held_bytes);
}

void Stage1Footprints(const Ctx& c, uint64_t kmax, uint64_t ib, uint64_t qb,
                      uint64_t* resident, uint64_t* windowed_device, uint64_t* windowed_host) {
  const std::vector<Batch> batches = Schedule(c, ib, qb);
  const Footprint f = Stage1Footprint(
      c, batches, kmax, IndexChunk(c, Stage1OneShot(c, batches, kmax)), c.bases.on_host);
  if (resident) *resident = static_cast<uint64_t>(f.resident);
  if (windowed_device) *windowed_device = static_cast<uint64_t>(f.windowed_device);
  if (windowed_host) *windowed_host = static_cast<uint64_t>(f.windowed_host);
}

void IndexFootprints(const Ctx& c, uint64_t ib, uint64_t* one_shot, uint64_t* chunked) {
  const std::vector<Batch> batches = Schedule(c, ib, 0);
  const uint64_t chunk =
      c.index_chunk_bases > 0 ? static_cast<uint64_t>(c.index_chunk_bases) : kAutoIndexChunk;
  if (one_shot) *one_shot = static_cast<uint64_t>(IndexFootprint(c, batches, 0));
  if (chunked) *chunked = static_cast<uint64_t>(IndexFootprint(c, batches, chunk));
}

void MinimizeFootprints(const Ctx& c, uint32_t first, uint32_t last, uint64_t* one_shot,
                        uint64_t* chunked, uint64_t* chunk) {
  const uint64_t size =
      c.index_chunk_bases > 0 ? static_cast<uint64_t>(c.index_chunk_bases) : kAutoIndexChunk;
  const double fit = MinimizeFootprint(c, first, last, 0);
  if (one_shot) *one_shot = static_cast<uint64_t>(fit);
  if (chunked) *chunked = static_cast<uint64_t>(MinimizeFootprint(c, first, last, size));
  if (chunk) *chunk = IndexChunk(c, fit);
}

}  // namespace rvn
