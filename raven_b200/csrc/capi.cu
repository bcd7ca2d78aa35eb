// raven_b200 — the C ABI (include/raven_b200.h) over the overlap engine, and
// the stage-1 driver that replaces raven::FindOverlapsAndCreatePiles
// (RavenLib/src/construct.cc:14-121).
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>

#include <unistd.h>

#include "engine.cuh"

using namespace rvn;

struct rvn_ctx {
  Ctx c;
};

namespace {

template <typename F>
int Guard(rvn_ctx* ctx, F&& f, bool sketches_first = false) {
  if (!ctx) return RVN_ERR_INVALID;
  // buffers allocated during the call are charged to this context
  struct Owner {
    uint64_t* prev;
    explicit Owner(uint64_t* o) : prev(g_devbuf_owner) { g_devbuf_owner = o; }
    ~Owner() { g_devbuf_owner = prev; }
  } owner(&ctx->c.held_bytes);
  try {
    RVN_CUDA(cudaSetDevice(ctx->c.device));
    // an asynchronous upload in flight: calls that begin with the sketch kernel
    // consume it chunk by chunk (EnsureSketch), everything else waits for all of it
    if (!sketches_first) WaitUpload(ctx->c);
    f(ctx->c);
    ctx->c.err.clear();
    return RVN_OK;
  } catch (const InvalidArgument& e) {
    ctx->c.err = e.what();
    return RVN_ERR_INVALID;
  } catch (const StateError& e) {
    ctx->c.err = e.what();
    return RVN_ERR_STATE;
  } catch (const LimitError& e) {
    ctx->c.err = e.what();
    return RVN_ERR_LIMIT;
  } catch (const CudaError& e) {
    ctx->c.err = e.what();
    return RVN_ERR_CUDA;
  } catch (const std::exception& e) {
    ctx->c.err = e.what();
    return RVN_ERR_CUDA;
  }
}

}  // namespace

namespace rvn {
void WaitUpload(Ctx& c) {
  if (!c.up_pending) return;
  RVN_CUDA(cudaStreamWaitEvent(c.stream, c.up_events[c.up_chunks - 1], 0));
  c.up_pending = false;
}
}  // namespace rvn

namespace {

void CheckRange(const Ctx& c, uint32_t first, uint32_t last) {
  if (first > last || last > c.n_reads) {
    throw InvalidArgument("read range out of bounds");
  }
}

// The reference's schedule (construct.cc:36-112): index batches [j, end) of >= ib
// bases, and per batch the flushes of its queries - every read up to the end of
// the batch - per >= qb bases (the truncation rule makes the flush boundaries
// observable).
struct Batch {
  uint32_t j, end;
  std::vector<std::pair<uint32_t, uint32_t>> flushes;  // [k0, k1)
};

std::vector<Batch> Schedule(const Ctx& c, uint64_t ib, uint64_t qb) {
  std::vector<Batch> out;
  const uint32_t n = c.n_reads;
  uint64_t bases = 0;
  for (uint32_t i = 0, j = 0; i < n; ++i) {
    bases += c.h_len[i];
    if (i != n - 1 && bases < ib) continue;
    bases = 0;
    Batch b{j, i + 1, {}};
    for (uint32_t k = 0, k0 = 0; k < i + 1; ++k) {
      bases += c.h_len[k];
      if (k != i && bases < qb) continue;
      bases = 0;
      b.flushes.emplace_back(k0, k + 1);
      k0 = k + 1;
    }
    out.push_back(std::move(b));
    j = i + 1;
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
// - per base of one chunk: its sketch in sweep 1 (s_val, s_org: 4.7 B);
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
    uint64_t bases = 0;
    for (uint32_t r = b.j; r < b.end; ++r) bases += c.h_len[r];
    batch_bases = std::max(batch_bases, bases);
    for (const auto& f : b.flushes) {
      uint64_t q = 0;
      for (uint32_t r = f.first; r < f.second; ++r) q += c.h_len[r];
      flush_bases = std::max(flush_bases, q);
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
// off: pile offsets of the reads (len >> 4 bins each, n + 1 entries)
// chunk: the index build's chunk size (0: one-shot), see IndexFootprint
Footprint Stage1Footprint(const Ctx& c, const std::vector<uint64_t>& off,
                          const std::vector<Batch>& batches, uint64_t kmax, uint64_t chunk) {
  const uint32_t n = c.n_reads;
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
  const double reads = 8.0 * c.n_words + 32.0 * n + IndexFootprint(c, batches, chunk);
  const double kept = std::min(static_cast<double>(kmax), n > 0 ? n - 1.0 : 0.0);
  Footprint f;
  f.resident = reads + 6.0 * bins + 4.0 * n + n * kept * list_bytes;
  f.windowed_device = reads + window;
  f.windowed_host = n * stride * sizeof(rvn_overlap) + 4.0 * n + 2.0 * bins;
  return f;
}

// device memory a pass can use: `budget`, or when that is 0 the free memory plus the
// buffers this context already holds (a pass re-uses them)
double UsableMemory(const Ctx& c, uint64_t budget) {
  if (budget) return static_cast<double>(budget);
  size_t free_b = 0, total_b = 0;
  RVN_CUDA(cudaMemGetInfo(&free_b, &total_b));
  return static_cast<double>(free_b) + static_cast<double>(c.held_bytes);
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
double Stage1OneShot(const Ctx& c, const std::vector<uint64_t>& off,
                     const std::vector<Batch>& batches, uint64_t kmax) {
  const Footprint f = Stage1Footprint(c, off, batches, kmax, 0);
  return kmax <= kWindowMaxOverlaps ? std::min(f.resident, f.windowed_device) : f.resident;
}

// The untiered index rvn_minimize builds holds every record of the batch: values, origins
// and the sort's second buffers (two copies of 12 B for an estimated 0.34 records per base,
// with the buffers' headroom) and the bucket table. Estimate, not measured.
constexpr double kUntieredIndexBytesPerBase = 8.9;

// Device memory of rvn_minimize over reads [first, last): the reads, the untiered index and
// the sketch of the batch (one-shot, chunk 0) or of one chunk of `chunk` bases.
double MinimizeFootprint(const Ctx& c, uint32_t first, uint32_t last, uint64_t chunk) {
  uint64_t bases = 0;
  for (uint32_t r = first; r < last; ++r) bases += c.h_len[r];
  const double bb = static_cast<double>(bases);
  const double sketched = chunk ? std::min(bb, static_cast<double>(chunk)) : bb;
  return 8.0 * c.n_words + 32.0 * c.n_reads + kUntieredIndexBytesPerBase * bb +
         kChunkSketchBytesPerBase * sketched;
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
  const double fixed = bytes(c.d_words) + bytes(c.i_val) + bytes(c.i_org) + bytes(c.i_val_alt) +
                       bytes(c.i_org_alt) + bytes(c.i_bucket) + bytes(c.j_packed);
  const double room = UsableMemory(c, 0) - fixed;
  const double flush = room / (join ? kJoinFlushBytesPerBase : kFlushBytesPerBase);
  if (flush >= static_cast<double>(kMapFlushCeiling)) return kMapFlushCeiling;
  return std::max(kMapFlushFloor, static_cast<uint64_t>(std::max(flush, 0.0)));
}

// rvn_map: MapRange flush by flush, each flush's overlaps, offsets and filtered positions
// appended to the pinned host results, so that they read as one MapRange over the range.
// One flush (and keep_hits, whose hits are those of one piece) is exactly that MapRange.
// each (stage 2): called with (first read, reads) after every flush, whose results it
// takes from the device (c.m_ovl, c.m_ovl_off, c.r_n_ovl, c.m_filtered); nothing is
// gathered on the host.
void MapFlushes(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal, bool avoid_symmetric,
                bool minhash, bool want_filtered,
                const std::function<void(uint32_t, uint32_t)>& each = nullptr) {
  uint64_t bases = 0;
  for (uint32_t r = first; r < last; ++r) bases += c.h_len[r];
  const bool join = c.self_join && minhash && avoid_equal && avoid_symmetric && !want_filtered &&
                    first >= c.i_first && last <= c.i_last;
  const std::vector<uint32_t> cuts = ChunkCuts(c, first, last, MapFlushBases(c, bases, join));
  if (each) {
    for (size_t i = 0; i + 1 < cuts.size(); ++i) {
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
// batches [j, i + 1) cut by the reference's rule (bytes < 1U << 30; option
// "stage2_batch_bases" forces a smaller batch), each an untiered full-sketch index
// filtered at freq, then every read of [0, i + 1) mapped with (avoid equal, avoid
// symmetric, no minhash, filtered positions) in rvn_map's flushes. Per flush, on the
// device: the filtered positions mark the k-mer bitmaps (Pile::AddKmers), and with
// identity != 0 the overlaps are clipped to the valid regions (rbeg, rend: Pile::begin()
// and end() per valid read) and filtered by edit distance. Only the final overlaps, and
// at the end the bitmaps and touched flags, go to the pinned host results.
void Stage2(Ctx& c, double freq, double identity, uint32_t n, const uint32_t* h_rbeg,
            const uint32_t* h_rend) {
  if (n > c.n_reads) throw InvalidArgument("more valid reads than uploaded reads");
  if (n && (!h_rbeg || !h_rend)) throw InvalidArgument("null regions");
  if (n && (c.res_first > 0 || c.res_last < n)) {
    throw StateError("the bases of the valid reads were not uploaded");
  }
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
  const uint64_t cut = c.stage2_batch_bases ? c.stage2_batch_bases : (1ULL << 30);
  struct HostFiltered {  // the filtered positions stay on the device for the whole call
    Ctx& c;
    explicit HostFiltered(Ctx& x) : c(x) { c.m_filtered_host = false; }
    ~HostFiltered() { c.m_filtered_host = true; }
  } keep_on_device(c);
  uint64_t bytes = 0;
  for (uint32_t i = 0, j = 0; i < n; ++i) {
    bytes += c.h_len[i];
    ooff[i + 1] = total;
    if (i != n - 1 && bytes < cut) continue;
    bytes = 0;
    // rvn_minimize(j, i + 1, 0) and rvn_filter(freq)
    const uint64_t chunk = IndexChunk(c, MinimizeFootprint(c, j, i + 1, 0));
    if (chunk) {
      BuildIndexChunked(c, j, i + 1, false, chunk, 0, /*tiers=*/false);
    } else {
      BuildIndex(c, j, i + 1, false);
    }
    FilterIndex(c, freq);
    if (chunk) ReleaseIndexBuild(c);
    MapFlushes(c, 0, i + 1, true, true, false, true, flush);
    ooff[i + 1] = total;
    j = i + 1;
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

// Option "stage1_window" -1 (auto): windowed only when the resident estimate exceeds
// the usable device memory ("stage1_window_budget" replaces it when it is not 0) and the
// windowed pass itself fits: it takes kmax, its own device estimate fits the same memory
// and its host rows fit the host's free physical memory. Otherwise resident, as before
// the option existed.
bool UseWindow(Ctx& c, const std::vector<Batch>& batches, uint64_t kmax, uint64_t chunk) {
  if (c.stage1_window >= 0) return c.stage1_window != 0;
  if (kmax > kWindowMaxOverlaps) return false;
  const Footprint f = Stage1Footprint(c, c.st_pile_off, batches, kmax, chunk);
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
    const std::vector<uint64_t>& off = c_.st_pile_off;
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
    const std::vector<uint64_t>& off = c_.st_pile_off;
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
    const std::vector<uint64_t>& off = c_.st_pile_off;
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
    const std::vector<uint64_t>& off = c_.st_pile_off;
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

// raven::FindOverlapsAndCreatePiles, same batch / flush schedule as the
// reference; every step runs on the GPU (Minimize, Filter, Map, AddLayers,
// gather, truncation); the host only drives the schedule (and, windowed, keeps
// the piles and lists of the reads a flush does not touch).
void Stage1(Ctx& c, double freq, uint64_t kmax, bool minhash, uint64_t ib,
            uint64_t qb) {
  if (ib == 0) ib = 1ULL << 32;
  if (qb == 0) qb = 1ULL << 30;
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
  c.s_valid = c.q_valid = c.qt_valid = c.i_valid = c.r_valid = false;
  TimerReset(c);
  std::memset(&c.stats, 0, sizeof(c.stats));
  const uint64_t launches0 = c.launches;
  const uint32_t n = c.n_reads;

  // piles: len >> 4 bins each (pile.cc:19-31)
  c.st_pile_off.assign(n + 1ULL, 0);
  for (uint32_t i = 0; i < n; ++i) {
    c.st_pile_off[i + 1] = c.st_pile_off[i] + (c.h_len[i] >> 4);
  }
  const uint64_t total_bins = c.st_pile_off[n];
  const std::vector<Batch> batches = Schedule(c, ib, qb);
  const uint64_t chunk = IndexChunk(c, Stage1OneShot(c, c.st_pile_off, batches, kmax));
  const bool windowed = UseWindow(c, batches, kmax, chunk);
  c.st_windowed = false;
  uint16_t* d_pile = nullptr;
  if (!windowed) {
    d_pile = c.p_data.reserve(total_bins + 1);
    RVN_CUDA(cudaMemsetAsync(d_pile, 0, (total_bins + 1) * sizeof(uint16_t), c.stream));
  }
  uint64_t* d_poff = c.p_off.reserve(n + 1ULL);
  if (!c.p_off_uploaded) {  // (an asynchronous upload has sent them ahead of the bases)
    RVN_CUDA(cudaMemcpyAsync(d_poff, c.st_pile_off.data(), (n + 1ULL) * 8,
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

  uint64_t tmax = 0;  // largest micromizer value of the reads sketched so far
  for (const Batch& b : batches) {
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

    for (const auto& f : b.flushes) {
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

void SetOption(Ctx& c, const char* name, int64_t value) {
  if (name && std::strcmp(name, "keep_hits") == 0) {
    c.keep_hits = value != 0;
  } else if (name && std::strcmp(name, "async_upload") == 0) {
    c.async_upload = value != 0;
  } else if (name && std::strcmp(name, "self_join") == 0) {
    c.self_join = value != 0;
  } else if (name && std::strcmp(name, "bare_count") == 0) {
    if (value != 0 && value != 1 && value != 8 && value != 16) {
      throw InvalidArgument("bare_count: 0, 1, 8 or 16");
    }
    c.bare_count = value;
    c.bare_cluster = 0;  // (chosen again at the next build)
  } else if (name && std::strcmp(name, "tier_min_records") == 0) {
    c.tier_min_records = value < 0 ? 0 : static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "stage1_window") == 0) {
    if (value < -1 || value > 1) throw InvalidArgument("stage1_window: -1 (auto), 0 or 1");
    c.stage1_window = value;
  } else if (name && std::strcmp(name, "stage1_stream") == 0) {
    if (value != 0 && value != 1) throw InvalidArgument("stage1_stream: 0 or 1");
    c.stage1_stream = value;
  } else if (name && std::strcmp(name, "stage1_window_budget") == 0) {
    c.stage1_window_budget = value < 0 ? 0 : static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "index_chunk_bases") == 0) {
    if (value < -1) throw InvalidArgument("index_chunk_bases: -1 (auto), 0 or a chunk size");
    c.index_chunk_bases = value;
  } else if (name && std::strcmp(name, "index_chunk_budget") == 0) {
    if (value < 0) throw InvalidArgument("index_chunk_budget: bytes, 0 = the free memory");
    c.index_chunk_budget = static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "map_flush_bases") == 0) {
    if (value < 0) throw InvalidArgument("map_flush_bases: bases, 0 = from the device memory");
    c.map_flush_bases = static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "stage2_batch_bases") == 0) {
    if (value < 0) throw InvalidArgument("stage2_batch_bases: bases, 0 = the reference's 2^30");
    c.stage2_batch_bases = static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "poa_wide") == 0) {
    if (value < 0 || value > 2) throw InvalidArgument("poa_wide: 0, 1 or 2");
    c.poa_wide = value;
  } else if (name && std::strcmp(name, "poa_scratch_budget") == 0) {
    if (value < 0) throw InvalidArgument("poa_scratch_budget: bytes, 0 = from the device memory");
    c.poa_scratch_budget = static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "poa_batch_bytes") == 0) {
    if (value < 0) throw InvalidArgument("poa_batch_bytes: bytes, 0 = from the device memory");
    c.poa_batch_bytes = static_cast<uint64_t>(value);
  } else if (name && std::strcmp(name, "radix_portion_tiles") == 0) {
    if (value < 0) throw InvalidArgument("radix_portion_tiles: tiles, 0 = the longest portion");
    c.radix_portion_tiles = value;
  } else if (name && std::strcmp(name, "reset_stats") == 0) {
    std::memset(&c.stats, 0, sizeof(c.stats));
    c.launches = 0;
    TimerReset(c);
  } else {
    throw InvalidArgument("unknown option");
  }
}

// RVN_SET_OPTIONS="name=value,...": options of every context the process creates, for
// programs that reach the library only through a facade (the reference's own executable)
void EnvOptions(Ctx& c) {
  const char* env = std::getenv("RVN_SET_OPTIONS");
  if (!env) return;
  std::string all(env);
  for (size_t b = 0; b < all.size();) {
    const size_t e = std::min(all.find(',', b), all.size());
    const std::string item = all.substr(b, e - b);
    const size_t eq = item.find('=');
    if (eq == std::string::npos) throw InvalidArgument("RVN_SET_OPTIONS: name=value,...");
    SetOption(c, item.substr(0, eq).c_str(), std::stoll(item.substr(eq + 1)));
    b = e + 1;
  }
}

}  // namespace

extern "C" {

#define RVN_API __attribute__((visibility("default")))

RVN_API int rvn_version(void) { return 100; }

RVN_API int rvn_ctx_create(int device, void* stream, rvn_ctx** out) {
  if (!out) return RVN_ERR_INVALID;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
    return RVN_ERR_CUDA;  // no CPU fallback: a usable device is mandatory
  }
  cudaDeviceProp prop;
  // the library holds sm_90a code only, which loads on compute capability 9.0 alone
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 ||
      prop.minor != 0) {
    return RVN_ERR_CUDA;
  }
  auto* ctx = new rvn_ctx();
  ctx->c.device = device;
  ctx->c.sms = prop.multiProcessorCount;
  int rc = Guard(ctx, [&](Ctx& c) {
    if (stream) {
      c.stream = static_cast<cudaStream_t>(stream);
    } else {
      RVN_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
      c.own_stream = true;
    }
    EnvOptions(c);
  });
  if (rc != RVN_OK) {
    delete ctx;
    return rc;
  }
  *out = ctx;
  return RVN_OK;
}

RVN_API void rvn_ctx_destroy(rvn_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->c.device);
  cudaStreamSynchronize(ctx->c.stream);
  for (auto& p : ctx->c.timer.pending) {
    if (p.first) cudaEventDestroy(p.first);
    if (p.second) cudaEventDestroy(p.second);
  }
  for (auto e : ctx->c.timer.pool) cudaEventDestroy(e);
  ArenaRelease(ctx->c);
  if (ctx->c.copy_stream) {
    cudaStreamSynchronize(ctx->c.copy_stream);
    cudaStreamDestroy(ctx->c.copy_stream);
  }
  if (ctx->c.d2h_stream) {
    cudaStreamSynchronize(ctx->c.d2h_stream);
    cudaStreamDestroy(ctx->c.d2h_stream);
    cudaEventDestroy(ctx->c.d2h_ready);
    cudaEventDestroy(ctx->c.d2h_done);
  }
  for (auto e : ctx->c.up_events) cudaEventDestroy(e);
  if (ctx->c.up_fence) cudaEventDestroy(ctx->c.up_fence);
  if (ctx->c.own_stream) cudaStreamDestroy(ctx->c.stream);
  delete ctx;
}

RVN_API const char* rvn_last_error(const rvn_ctx* ctx) {
  return ctx ? ctx->c.err.c_str() : "null context";
}

RVN_API int rvn_engine_configure(rvn_ctx* ctx, uint32_t k, uint32_t w,
                                 uint32_t bandwidth, uint32_t chain,
                                 uint32_t matches, uint32_t gap) {
  return Guard(ctx, [&](Ctx& c) {
    if (w == 0) throw InvalidArgument("window length must be positive");
    if (w > kMaxWindow) throw LimitError("window length above 256");
    c.prm.k = std::min(std::max(k, 1u), 31u);
    c.prm.w = w;
    c.prm.bandwidth = bandwidth;
    c.prm.chain = chain;
    c.prm.matches = matches;
    c.prm.gap = gap;
    c.s_valid = c.q_valid = c.qt_valid = c.i_valid = c.r_valid = false;
    c.tiles_k = 0;  // the tile table depends on (k, w)
    c.occurrence = 0xFFFFFFFFu;
  });
}

static void UploadReads(Ctx& c, const uint64_t* words, const uint64_t* word_off,
                        const uint32_t* lens, const uint32_t* ids,
                        uint32_t n_reads, uint32_t res_first = 0,
                        uint32_t res_last = 0xFFFFFFFFu) {
  if (n_reads && (!word_off || !lens)) throw InvalidArgument("null read set");
  res_last = std::min(res_last, n_reads);
  if (res_first > res_last) throw InvalidArgument("resident range out of bounds");
  if (n_reads == 0xFFFFFFFFu) throw LimitError("too many reads");
  c.s_valid = c.q_valid = c.qt_valid = c.i_valid = c.r_valid = c.st_valid = false;
  c.st_piles_on_device = false;
  c.tiles_k = 0;
  c.n_reads = n_reads;
  c.h_woff.assign(1, 0);
  if (n_reads) c.h_woff.assign(word_off, word_off + n_reads + 1);
  c.h_len.assign(lens, lens + n_reads);
  c.h_ids.resize(n_reads);
  c.ids_identity = true;
  c.ids_ascending = true;
  for (uint32_t i = 0; i < n_reads; ++i) {
    const uint64_t have = c.h_woff[i + 1] - c.h_woff[i];
    if (have < ((static_cast<uint64_t>(lens[i]) + 31) >> 5)) {
      throw InvalidArgument("read shorter than its declared length");
    }
    if (lens[i] >= (1u << 31)) throw LimitError("read of 2^31 or more bases");
    c.h_ids[i] = ids ? ids[i] : i;
    if (c.h_ids[i] != i) c.ids_identity = false;
    if (i > 0 && c.h_ids[i] < c.h_ids[i - 1]) c.ids_ascending = false;
  }
  c.n_words = c.h_woff[n_reads];
  // one spare slot everywhere: an external query read rides at index n_reads
  uint64_t* dw = c.d_words.reserve(c.n_words + 2);
  uint64_t* dwo = c.d_woff.reserve(n_reads + 2ULL);
  uint32_t* dl = c.d_len.reserve(n_reads + 2ULL);
  uint32_t* di = c.d_ids.reserve(n_reads + 2ULL);
  // bases of the resident reads only (a rank of a partitioned run sketches its
  // own range; lengths and ids of all reads are always resident)
  c.res_first = res_first;
  c.res_last = res_last;
  // offsets, lengths, ids first (small, from pageable memory: behind the bases they
  // would wait for the copy engine)
  RVN_CUDA(cudaMemcpyAsync(dwo, c.h_woff.data(), (n_reads + 1ULL) * 8,
                           cudaMemcpyHostToDevice, c.stream));
  if (n_reads) {
    RVN_CUDA(cudaMemcpyAsync(dl, c.h_len.data(), n_reads * 4ULL,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(di, c.h_ids.data(), n_reads * 4ULL,
                             cudaMemcpyHostToDevice, c.stream));
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  const uint64_t w0 = c.h_woff[res_first], w1 = c.h_woff[res_last];
  c.up_pending = false;
  c.p_off_uploaded = false;
  if (w1 > w0 && c.async_upload && res_last - res_first >= 1024) {
    // everything small the next call would send host-to-device goes first: behind the
    // bases it would wait for the copy engine (tile tables, pile offsets of stage 1)
    EnsureTiles(c);
    {
      c.st_pile_off.assign(n_reads + 1ULL, 0);
      for (uint32_t i = 0; i < n_reads; ++i) c.st_pile_off[i + 1] = c.st_pile_off[i] + (lens[i] >> 4);
      uint64_t* d_poff = c.p_off.reserve(n_reads + 1ULL);
      RVN_CUDA(cudaMemcpyAsync(d_poff, c.st_pile_off.data(), (n_reads + 1ULL) * 8,
                               cudaMemcpyHostToDevice, c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));
      c.p_off_uploaded = true;
    }
    // chunks that end at read boundaries, on the copy stream; the caller keeps
    // `words` alive until the next call on this context has returned
    constexpr uint32_t kChunks = 8;
    if (!c.copy_stream) {
      RVN_CUDA(cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking));
      RVN_CUDA(cudaEventCreateWithFlags(&c.up_fence, cudaEventDisableTiming));
    }
    while (c.up_events.size() < kChunks) {
      cudaEvent_t ev;
      RVN_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      c.up_events.push_back(ev);
    }
    // (kernels of earlier calls may still read the old bases)
    RVN_CUDA(cudaEventRecord(c.up_fence, c.stream));
    RVN_CUDA(cudaStreamWaitEvent(c.copy_stream, c.up_fence, 0));
    c.up_read_end.clear();
    uint32_t r_prev = res_first;
    for (uint32_t i = 1; i <= kChunks && r_prev < res_last; ++i) {
      const uint64_t target = w0 + (w1 - w0) * i / kChunks;
      uint32_t r = static_cast<uint32_t>(
          std::lower_bound(c.h_woff.begin() + r_prev + 1, c.h_woff.begin() + res_last + 1, target) -
          c.h_woff.begin());
      if (i == kChunks || r > res_last) r = res_last;
      const uint64_t a = c.h_woff[r_prev], b = c.h_woff[r];
      if (b > a) {
        RVN_CUDA(cudaMemcpyAsync(dw + a, words + a, (b - a) * 8, cudaMemcpyHostToDevice,
                                 c.copy_stream));
      }
      RVN_CUDA(cudaEventRecord(c.up_events[c.up_read_end.size()], c.copy_stream));
      c.up_read_end.push_back(r);
      r_prev = r;
    }
    c.up_chunks = static_cast<uint32_t>(c.up_read_end.size());
    c.up_pending = c.up_chunks > 0;
  } else if (w1 > w0) {
    RVN_CUDA(cudaMemcpyAsync(dw + w0, words + w0, (w1 - w0) * 8, cudaMemcpyHostToDevice,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  }
}

RVN_API int rvn_reads_upload(rvn_ctx* ctx, const uint64_t* words,
                             const uint64_t* word_off, const uint32_t* lens,
                             uint32_t n_reads) {
  return Guard(ctx, [&](Ctx& c) {
    UploadReads(c, words, word_off, lens, nullptr, n_reads);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_reads_upload_range(rvn_ctx* ctx, const uint64_t* words,
                                   const uint64_t* word_off, const uint32_t* lens,
                                   uint32_t n_reads, uint32_t first, uint32_t last) {
  return Guard(ctx, [&](Ctx& c) {
    UploadReads(c, words, word_off, lens, nullptr, n_reads, first, last);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_reads_upload_ids(rvn_ctx* ctx, const uint64_t* words,
                                 const uint64_t* word_off, const uint32_t* lens,
                                 const uint32_t* ids, uint32_t n_reads) {
  return Guard(ctx, [&](Ctx& c) {
    UploadReads(c, words, word_off, lens, ids, n_reads);
  }, /*sketches_first=*/true);
}

// Map one read that is not part of the uploaded set (it rides in the spare
// slot behind the set for the duration of the call)
RVN_API int rvn_map_external(rvn_ctx* ctx, const uint64_t* words, uint32_t len,
                             uint32_t id, int avoid_equal, int avoid_symmetric,
                             int minhash, int want_filtered) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.i_valid) throw StateError("Map before Minimize");
    if (len >= (1u << 31)) throw LimitError("read of 2^31 or more bases");
    const uint32_t n = c.n_reads;
    const uint64_t nw = (static_cast<uint64_t>(len) + 31) >> 5;
    if (nw && !words) throw InvalidArgument("null read");
    uint64_t* dw = c.d_words.reserve_keep(c.n_words + nw + 2, c.n_words, c.stream);
    if (nw) {
      RVN_CUDA(cudaMemcpyAsync(dw + c.n_words, words, nw * 8,
                               cudaMemcpyHostToDevice, c.stream));
    }
    EnsureTiles(c);
    // extend the host/device tables by the spare slot
    const uint64_t woff_tail[2] = {c.n_words, c.n_words + nw};
    uint64_t tiles = 0;
    if (len >= c.prm.k && len - c.prm.k + 1 >= c.prm.w) {
      tiles = (len - c.prm.k + 1 + kSketchTile - 1) / kSketchTile;
    }
    const uint64_t tile_tail[2] = {c.h_tile_off[n], c.h_tile_off[n] + tiles};
    RVN_CUDA(cudaMemcpyAsync(c.d_woff.get() + n, woff_tail, 16,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(c.d_tile_off.get() + n, tile_tail, 16,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(c.d_len.get() + n, &len, 4, cudaMemcpyHostToDevice,
                             c.stream));
    RVN_CUDA(cudaMemcpyAsync(c.d_ids.get() + n, &id, 4, cudaMemcpyHostToDevice,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    c.h_woff.push_back(c.n_words + nw);
    c.h_len.push_back(len);
    c.h_ids.push_back(id);
    c.h_tile_off.push_back(tile_tail[1]);
    c.n_reads = n + 1;
    c.s_valid = c.q_valid = c.qt_valid = false;
    // the rider's bases are resident for the duration of the call (EnsureSketch
    // refuses reads outside [res_first, res_last))
    const uint32_t res_first0 = c.res_first, res_last0 = c.res_last;
    c.res_first = n;
    c.res_last = n + 1;
    auto restore = [&]() {
      c.res_first = res_first0;
      c.res_last = res_last0;
      c.n_reads = n;
      c.h_woff.pop_back(); c.h_len.pop_back(); c.h_ids.pop_back();
      c.h_tile_off.pop_back();
      c.s_valid = c.q_valid = c.qt_valid = false;
    };
    try {
      // an id below an indexed id breaks the "kept postings are a suffix" shortcut
      // only through avoid_symmetric, which compares ids, not indices: fine
      MapRange(c, n, n + 1, avoid_equal != 0, avoid_symmetric != 0, minhash != 0,
               want_filtered != 0);
    } catch (...) {
      restore();
      throw;
    }
    restore();
    TimerCollect(c);
  });
}

RVN_API int rvn_minimize(rvn_ctx* ctx, uint32_t first, uint32_t last,
                         int minhash) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    const uint64_t chunk = IndexChunk(c, MinimizeFootprint(c, first, last, 0));
    if (chunk) {
      // untiered: a later rvn_map may probe with full sketches
      BuildIndexChunked(c, first, last, minhash != 0, chunk, 0, /*tiers=*/false);
      c.i_build_held = true;
    } else {
      BuildIndex(c, first, last, minhash != 0);
    }
  }, /*sketches_first=*/true);
}

RVN_API int rvn_filter(rvn_ctx* ctx, double frequency, uint32_t* occurrence) {
  return Guard(ctx, [&](Ctx& c) {
    uint32_t occ = FilterIndex(c, frequency);
    if (c.i_build_held) {
      ReleaseIndexBuild(c);
      c.i_build_held = false;
    }
    if (occurrence) *occurrence = occ;
  });
}

RVN_API int rvn_map(rvn_ctx* ctx, uint32_t first, uint32_t last,
                    int avoid_equal, int avoid_symmetric, int minhash,
                    int want_filtered) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    MapFlushes(c, first, last, avoid_equal != 0, avoid_symmetric != 0, minhash != 0,
               want_filtered != 0);
    TimerCollect(c);
  });
}

RVN_API int rvn_map_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                            const uint64_t** ovl_off, uint64_t* n_overlaps,
                            const uint32_t** filtered,
                            const uint64_t** filt_off) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.r_valid) throw StateError("no map results");
    if (overlaps) *overlaps = c.r_ovl.get();
    if (ovl_off) *ovl_off = c.r_ovl_off.get();
    if (n_overlaps) *n_overlaps = c.r_n_ovl;
    if (filtered) *filtered = c.r_filtered.get();
    if (filt_off) *filt_off = c.r_filt_off.get();
  });
}

RVN_API int rvn_pile_add_layers(rvn_ctx* ctx, uint16_t* data,
                                const uint64_t* bin_off, uint32_t n_piles,
                                const rvn_overlap* overlaps,
                                uint64_t n_overlaps) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_piles == 0) return;
    if (!data || !bin_off) throw InvalidArgument("null piles");
    const uint64_t bins = bin_off[n_piles];
    uint16_t* d = c.p_data.reserve(bins + 1);
    c.p_off_uploaded = false;
    c.st_piles_on_device = false;
    uint64_t* off = c.p_off.reserve(n_piles + 1ULL);
    rvn_overlap* o = c.p_ovl.reserve(n_overlaps + 1);
    RVN_CUDA(cudaMemcpyAsync(d, data, bins * 2, cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(off, bin_off, (n_piles + 1ULL) * 8,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(o, overlaps, n_overlaps * sizeof(rvn_overlap),
                             cudaMemcpyHostToDevice, c.stream));
    PileAddLayersDevice(c, d, off, bins, Window::All(n_piles), o, n_overlaps);
    RVN_CUDA(cudaMemcpyAsync(data, d, bins * 2, cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    TimerCollect(c);
  });
}

RVN_API int rvn_poa_batch(rvn_ctx* ctx, uint32_t n_windows, const uint32_t* win_first,
                          const uint64_t* seq_off, const char* bases,
                          const char* quals, const uint32_t* seq_begin,
                          const uint32_t* seq_end, int8_t m, int8_t n, int8_t g,
                          int trim, int tgs, int want_coverage) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_windows && (!win_first || !seq_off || !bases || !seq_begin || !seq_end)) {
      throw InvalidArgument("null window batch");
    }
    TimerReset(c);
    PoaBatch(c, n_windows, win_first, seq_off, reinterpret_cast<const uint8_t*>(bases),
             reinterpret_cast<const uint8_t*>(quals), seq_begin, seq_end, m, n, g,
             trim != 0, tgs != 0, want_coverage != 0);
    TimerCollect(c);
  });
}

RVN_API int rvn_poa_results(rvn_ctx* ctx, const char** consensus,
                            const uint64_t** cons_off, const uint8_t** status,
                            const uint32_t** coverage, uint64_t* cells) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.poa_valid) throw StateError("no POA results");
    if (consensus) *consensus = reinterpret_cast<const char*>(c.po_out_cons.data());
    if (cons_off) *cons_off = c.po_out_off.data();
    if (status) *status = c.po_h_status.data();
    if (coverage) *coverage = c.po_has_cov ? c.po_out_cov.data() : nullptr;
    if (cells) *cells = c.po_cells;
  });
}

RVN_API int rvn_poa_routes(rvn_ctx* ctx, uint32_t* windows, uint32_t* launches) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.poa_valid) throw StateError("no POA results");
    for (int k = 0; k < 3; ++k) {
      if (windows) windows[k] = c.po_route_windows[k];
      if (launches) launches[k] = c.po_route_launches[k];
    }
  });
}

RVN_API int rvn_polish_windows(rvn_ctx* ctx, uint64_t n_alignments, const uint32_t* q_read,
                               const uint32_t* q_begin, const uint32_t* q_len,
                               const uint8_t* strand, const uint32_t* t_read,
                               const uint64_t* bp_off, const uint32_t* breaking_points,
                               uint32_t n_targets, uint32_t window,
                               const uint8_t* block_quality, const uint64_t* bq_off,
                               const uint8_t* reverse_complement, double q, int8_t m, int8_t n,
                               int8_t g, int trim, int tgs, uint32_t* window_batches) {
  return Guard(ctx, [&](Ctx& c) {
    if (!bp_off || (block_quality && !bq_off)) throw InvalidArgument("null argument");
    if (n_alignments && (!q_read || !q_begin || !q_len || !strand || !t_read ||
                         (bp_off[n_alignments] && !breaking_points))) {
      throw InvalidArgument("null argument");
    }
    TimerReset(c);
    PolishArgs a{n_alignments, q_read, q_begin, q_len, strand, t_read, bp_off, breaking_points,
                 n_targets, window, block_quality, bq_off, reverse_complement, q, m, n, g,
                 trim != 0, tgs != 0};
    PolishWindows(c, a);
    if (window_batches) *window_batches = c.po_batches;
    TimerCollect(c);
  });
}

RVN_API int rvn_kmer_complexity(rvn_ctx* ctx, const uint32_t* read_index,
                                const uint32_t* positions, uint64_t n,
                                uint32_t kmer_len, uint8_t* keep) {
  return Guard(ctx, [&](Ctx& c) {
    if (n && (!read_index || !positions || !keep)) throw InvalidArgument("null argument");
    if (kmer_len == 0 || kmer_len > 31) throw InvalidArgument("k-mer length outside [1, 31]");
    for (uint64_t i = 0; i < n; ++i) {
      if (read_index[i] >= c.n_reads) throw InvalidArgument("read index out of bounds");
    }
    KmerComplexity(c, read_index, positions, n, kmer_len, keep);
  });
}

RVN_API int rvn_find_overlaps_and_create_piles(rvn_ctx* ctx, double frequency,
                                               uint64_t max_overlaps,
                                               int minhash,
                                               uint64_t index_batch_bases,
                                               uint64_t query_batch_bases) {
  return Guard(ctx, [&](Ctx& c) {
    Stage1(c, frequency, max_overlaps, minhash != 0, index_batch_bases,
           query_batch_bases);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_find_overlaps_and_repetitive_regions(rvn_ctx* ctx, double frequency,
                                                     double identity, uint32_t n_valid,
                                                     const uint32_t* region_begin,
                                                     const uint32_t* region_end) {
  return Guard(ctx, [&](Ctx& c) {
    Stage2(c, frequency, identity, n_valid, region_begin, region_end);
    TimerCollect(c);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_stage2_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                               const uint64_t** overlap_off, const uint32_t** kmer_bits,
                               const uint64_t** kmer_off, const uint8_t** kmer_touched,
                               uint64_t* n_mapped) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.s2_valid) throw StateError("no stage-2 results");
    if (overlaps) *overlaps = c.s2_ovl.get();
    if (overlap_off) *overlap_off = c.s2_ovl_off.get();
    if (kmer_bits) *kmer_bits = c.s2_bits_h.get();
    if (kmer_off) *kmer_off = c.s2_bit_off_h.get();
    if (kmer_touched) *kmer_touched = c.s2_touched_h.get();
    if (n_mapped) *n_mapped = c.s2_mapped;
  });
}

RVN_API int rvn_stage1_footprint(rvn_ctx* ctx, uint64_t max_overlaps,
                                 uint64_t index_batch_bases, uint64_t query_batch_bases,
                                 uint64_t* resident, uint64_t* windowed_device,
                                 uint64_t* windowed_host) {
  return Guard(ctx, [&](Ctx& c) {
    const uint32_t n = c.n_reads;
    std::vector<uint64_t> off(n + 1ULL, 0);
    for (uint32_t i = 0; i < n; ++i) off[i + 1] = off[i] + (c.h_len[i] >> 4);
    const std::vector<Batch> batches =
        Schedule(c, index_batch_bases ? index_batch_bases : 1ULL << 32,
                 query_batch_bases ? query_batch_bases : 1ULL << 30);
    const Footprint f = Stage1Footprint(c, off, batches, max_overlaps,
                                        IndexChunk(c, Stage1OneShot(c, off, batches, max_overlaps)));
    if (resident) *resident = static_cast<uint64_t>(f.resident);
    if (windowed_device) *windowed_device = static_cast<uint64_t>(f.windowed_device);
    if (windowed_host) *windowed_host = static_cast<uint64_t>(f.windowed_host);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_index_footprint(rvn_ctx* ctx, uint64_t index_batch_bases, uint64_t* one_shot,
                                uint64_t* chunked) {
  return Guard(ctx, [&](Ctx& c) {
    const std::vector<Batch> batches =
        Schedule(c, index_batch_bases ? index_batch_bases : 1ULL << 32, 1ULL << 30);
    const uint64_t chunk =
        c.index_chunk_bases > 0 ? static_cast<uint64_t>(c.index_chunk_bases) : kAutoIndexChunk;
    if (one_shot) *one_shot = static_cast<uint64_t>(IndexFootprint(c, batches, 0));
    if (chunked) *chunked = static_cast<uint64_t>(IndexFootprint(c, batches, chunk));
  }, /*sketches_first=*/true);
}

RVN_API int rvn_minimize_footprint(rvn_ctx* ctx, uint32_t first, uint32_t last,
                                   uint64_t* one_shot, uint64_t* chunked, uint64_t* chunk) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    const uint64_t size =
        c.index_chunk_bases > 0 ? static_cast<uint64_t>(c.index_chunk_bases) : kAutoIndexChunk;
    const double fit = MinimizeFootprint(c, first, last, 0);
    if (one_shot) *one_shot = static_cast<uint64_t>(fit);
    if (chunked) *chunked = static_cast<uint64_t>(MinimizeFootprint(c, first, last, size));
    if (chunk) *chunk = IndexChunk(c, fit);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_stage1_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                               const uint64_t** ovl_off, const uint16_t** pile,
                               const uint64_t** pile_off, uint64_t* n_mapped) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.st_valid) throw StateError("no stage-1 results");
    if (overlaps) *overlaps = c.st_ovl.get();
    if (ovl_off) *ovl_off = c.st_ovl_off.get();
    if (pile) *pile = c.st_pile.get();
    if (pile_off) *pile_off = c.st_pile_off.data();
    if (n_mapped) *n_mapped = c.st_mapped;
  });
}

RVN_API int rvn_sketch(rvn_ctx* ctx, uint32_t first, uint32_t last, int minhash,
                       const uint64_t** value, const uint64_t** origin,
                       const uint64_t** offsets, uint64_t* n_records) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    const uint32_t nr = last - first;
    const uint64_t *dv, *dorg;
    const std::vector<uint64_t>* hoff;
    uint64_t total;
    EnsureSketch(c, first, last);
    if (minhash) {
      EnsureMicromizers(c, first, last);
      dv = c.q_val.get();
      dorg = c.q_org.get();
      hoff = &c.h_q_off;
      total = c.q_n;
    } else {
      dv = c.s_val.get();
      dorg = c.s_org.get();
      hoff = &c.h_s_off;
      total = c.s_n;
    }
    uint64_t* hv = c.x_val.reserve(total + 1);
    uint64_t* ho = c.x_org.reserve(total + 1);
    uint64_t* hf = c.x_off.reserve(nr + 2ULL);
    const bool v32 = minhash ? c.q_is32 : c.s_is32;  // k <= 15: u32 values
    RVN_CUDA(cudaMemcpyAsync(hv, dv, total * (v32 ? 4 : 8), cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(ho, dorg, total * 8, cudaMemcpyDeviceToHost, c.stream));
    for (uint32_t i = 0; i <= nr; ++i) hf[i] = (*hoff)[i];
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    if (v32) {  // widen in place, back to front
      const uint32_t* h32 = reinterpret_cast<const uint32_t*>(hv);
      for (uint64_t i = total; i-- > 0;) hv[i] = h32[i];
    }
    TimerCollect(c);
    if (value) *value = hv;
    if (origin) *origin = ho;
    if (offsets) *offsets = hf;
    if (n_records) *n_records = total;
  }, /*sketches_first=*/true);
}

RVN_API int rvn_index_records(rvn_ctx* ctx, const uint64_t** value,
                              const uint64_t** origin, uint64_t* n_records,
                              uint64_t* n_keys) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.i_valid) throw StateError("no index");
    uint64_t* hv = c.x_val.reserve(c.i_n + 1);
    uint64_t* ho = c.x_org.reserve(c.i_n + 1);
    RVN_CUDA(cudaMemcpyAsync(hv, c.i_val.get(), c.i_n * (c.i_is32 ? 4 : 8),
                             cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaMemcpyAsync(ho, c.i_org.get(), c.i_n * 8, cudaMemcpyDeviceToHost,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    if (c.i_is32) {  // widen in place, back to front
      const uint32_t* h32 = reinterpret_cast<const uint32_t*>(hv);
      for (uint64_t i = c.i_n; i-- > 0;) hv[i] = h32[i];
    }
    if (value) *value = hv;
    if (origin) *origin = ho;
    if (n_records) *n_records = c.i_n;
    if (n_keys) *n_keys = c.i_keys;
  });
}

RVN_API int rvn_map_hits(rvn_ctx* ctx, const uint64_t** group,
                         const uint64_t** positions, const uint64_t** hit_off,
                         uint64_t* n_hits) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.r_valid || !c.keep_hits) throw StateError("hits were not kept");
    if (group) *group = c.r_hit_grp.get();
    if (positions) *positions = c.r_hit_pos.get();
    if (hit_off) *hit_off = c.r_hit_off.get();
    if (n_hits) *n_hits = c.r_n_hits;
  });
}

RVN_API int rvn_edit_distance_batch(rvn_ctx* ctx, uint64_t n_pairs, const uint32_t* lhs_read,
                                    const uint32_t* lhs_begin, const uint32_t* lhs_len,
                                    const uint32_t* rhs_read, const uint32_t* rhs_begin,
                                    const uint32_t* rhs_len, const uint8_t* strand,
                                    const int32_t* limit, int32_t* distance) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_pairs && (!lhs_read || !lhs_begin || !lhs_len || !rhs_read || !rhs_begin || !rhs_len ||
                    !strand || !distance)) {
      throw InvalidArgument("null argument");
    }
    EditDistanceBatch(c, n_pairs, lhs_read, lhs_begin, lhs_len, rhs_read, rhs_begin, rhs_len,
                      strand, limit, distance);
    TimerCollect(c);
  });
}

RVN_API int rvn_stage1_pile_regions(rvn_ctx* ctx, uint32_t coverage, uint32_t* begin,
                                    uint32_t* end, uint16_t* median, uint8_t* invalid) {
  return Guard(ctx, [&](Ctx& c) {
    if (c.n_reads && (!begin || !end || !median || !invalid)) throw InvalidArgument("null argument");
    if (coverage > 0xFFFF) throw InvalidArgument("coverage beyond 65535");
    StagePileRegions(c, coverage, begin, end, median, invalid);
    TimerCollect(c);
  });
}

RVN_API int rvn_align_breaking_points(rvn_ctx* ctx, uint64_t n_pairs, const uint32_t* q_read,
                                      const uint32_t* q_begin, const uint32_t* q_len,
                                      const uint8_t* strand, const uint32_t* t_read,
                                      const uint32_t* t_begin, const uint32_t* t_len,
                                      uint32_t window, const uint64_t* bp_off, int32_t* distance,
                                      uint32_t* breaking_points) {
  return Guard(ctx, [&](Ctx& c) {
    if (!bp_off) throw InvalidArgument("null argument");
    if (n_pairs && (!q_read || !q_begin || !q_len || !strand || !t_read || !t_begin || !t_len ||
                    !distance || (bp_off[n_pairs] && !breaking_points))) {
      throw InvalidArgument("null argument");
    }
    AlignBreakingPoints(c, n_pairs, q_read, q_begin, q_len, strand, t_read, t_begin, t_len, window,
                        bp_off, distance, breaking_points);
    TimerCollect(c);
  });
}

// whether p is device memory: the debug entry points below take host or device arrays
static bool OnDevice(const void* p) {
  cudaPointerAttributes a{};
  if (!p || cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();  // (clears the error of a pointer CUDA does not know)
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// the engine's radix sort, in place (parity tests of radix.cu). Host arrays travel
// through three device buffers per array; device arrays are the sort's source and its
// buffer b, so that only buffer a is allocated.
RVN_API int rvn_debug_sort_pairs(rvn_ctx* ctx, int key_bytes, int val_bytes, void* keys,
                                 void* vals, uint64_t n, int begin_bit, int end_bit,
                                 int descending) {
  return Guard(ctx, [&](Ctx& c) {
    if ((key_bytes != 4 && key_bytes != 8) || (val_bytes != 0 && val_bytes != 4 && val_bytes != 8)) {
      throw InvalidArgument("key of 4 or 8 bytes, value of 0, 4 or 8 bytes");
    }
    if (val_bytes == 0 && key_bytes != 4) throw InvalidArgument("keys-only sort takes u32 keys");
    if (begin_bit < 0 || end_bit > 8 * key_bytes || begin_bit > end_bit) {
      throw InvalidArgument("bit range out of bounds");
    }
    if (n >= 0xFFFFFFFFULL) throw LimitError("radix sort of 2^32 or more records");
    if (n && (!keys || (val_bytes && !vals))) throw InvalidArgument("null arrays");
    const bool dev = n && OnDevice(keys);
    if (val_bytes && n && OnDevice(vals) != dev) {
      throw InvalidArgument("keys and values both on the device or both on the host");
    }
    const size_t kbytes = static_cast<size_t>(key_bytes) * n, vbytes = static_cast<size_t>(val_bytes) * n;
    DevBuf<uint8_t> ks, ka, kb, vs, va, vb;
    uint8_t *k_src, *k_a, *k_b, *v_src, *v_a, *v_b;
    k_a = ka.reserve(kbytes + 16);
    v_a = va.reserve(vbytes + 16);
    if (dev) {
      k_src = k_b = static_cast<uint8_t*>(keys);
      v_src = v_b = val_bytes ? static_cast<uint8_t*>(vals) : vb.reserve(16);
    } else {
      k_src = ks.reserve(kbytes + 16);
      k_b = kb.reserve(kbytes + 16);
      v_src = vs.reserve(vbytes + 16);
      v_b = vb.reserve(vbytes + 16);
      RVN_CUDA(cudaMemcpyAsync(k_src, keys, kbytes, cudaMemcpyHostToDevice, c.stream));
      if (val_bytes) RVN_CUDA(cudaMemcpyAsync(v_src, vals, vbytes, cudaMemcpyHostToDevice, c.stream));
    }
    int where;
    const bool desc = descending != 0;
    if (val_bytes == 0) {
      where = RadixSortKeys(c, (const uint32_t*)k_src, (uint32_t*)k_a, (uint32_t*)k_b, n,
                            begin_bit, end_bit);
    } else if (key_bytes == 4 && val_bytes == 8) {
      where = RadixSortPairs(c, (const uint32_t*)k_src, (uint32_t*)k_a, (uint32_t*)k_b,
                             (const uint64_t*)v_src, (uint64_t*)v_a, (uint64_t*)v_b, n,
                             begin_bit, end_bit, desc);
    } else if (key_bytes == 8 && val_bytes == 8) {
      where = RadixSortPairs(c, (const uint64_t*)k_src, (uint64_t*)k_a, (uint64_t*)k_b,
                             (const uint64_t*)v_src, (uint64_t*)v_a, (uint64_t*)v_b, n,
                             begin_bit, end_bit, desc);
    } else if (key_bytes == 4 && val_bytes == 4) {
      where = RadixSortPairs(c, (const uint32_t*)k_src, (uint32_t*)k_a, (uint32_t*)k_b,
                             (const uint32_t*)v_src, (uint32_t*)v_a, (uint32_t*)v_b, n,
                             begin_bit, end_bit, desc);
    } else {
      where = RadixSortPairs(c, (const uint64_t*)k_src, (uint64_t*)k_a, (uint64_t*)k_b,
                             (const uint32_t*)v_src, (uint32_t*)v_a, (uint32_t*)v_b, n,
                             begin_bit, end_bit, desc);
    }
    const uint8_t* rk = where < 0 ? k_src : (where == 0 ? k_a : k_b);
    const uint8_t* rv = where < 0 ? v_src : (where == 0 ? v_a : v_b);
    if (rk != keys) {  // (device arrays: only a result in buffer a moves)
      RVN_CUDA(cudaMemcpyAsync(keys, rk, kbytes, cudaMemcpyDefault, c.stream));
      if (val_bytes) RVN_CUDA(cudaMemcpyAsync(vals, rv, vbytes, cudaMemcpyDefault, c.stream));
    }
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  });
}

// the engine's unstable radix partition (RadixPartitionKeys), in place: keys (u32) and
// bin_start (1024 entries) on the host or on the device, each on its own
RVN_API int rvn_debug_partition_keys(rvn_ctx* ctx, uint32_t* keys, uint64_t n, int begin_bit,
                                     int end_bit, uint32_t* bin_start) {
  return Guard(ctx, [&](Ctx& c) {
    if (begin_bit < 0 || end_bit > 32 || end_bit - begin_bit < 1 || end_bit - begin_bit > 10) {
      throw InvalidArgument("1 to 10 key bits inside 32");
    }
    if (n >= 0xFFFFFFFFULL) throw LimitError("radix partition of 2^32 or more records");
    if ((n && !keys) || !bin_start) throw InvalidArgument("null arrays");
    const size_t bytes = sizeof(uint32_t) * n;
    DevBuf<uint32_t> src_buf, dst_buf, start_buf;
    const bool dev = n && OnDevice(keys);
    uint32_t* src = dev ? keys : src_buf.reserve(n + 1);
    uint32_t* dst = dst_buf.reserve(n + 1);  // (the pass cannot write over its source)
    uint32_t* start = OnDevice(bin_start) ? bin_start : start_buf.reserve(1024);
    if (!dev && n) RVN_CUDA(cudaMemcpyAsync(src, keys, bytes, cudaMemcpyHostToDevice, c.stream));
    RadixPartitionKeys(c, src, dst, n, begin_bit, end_bit, start);
    if (n) RVN_CUDA(cudaMemcpyAsync(keys, dst, bytes, cudaMemcpyDefault, c.stream));
    if (start != bin_start) {
      RVN_CUDA(cudaMemcpyAsync(bin_start, start, 1024 * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                               c.stream));
    }
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  });
}

// the engine's exclusive scan (ExclusiveScanU32): out[i] = in[0] + ... + in[i - 1] for
// i in [0, n]; in and out on the host or on the device, each on its own
RVN_API int rvn_debug_exclusive_scan(rvn_ctx* ctx, const uint32_t* in, uint64_t n,
                                     uint64_t* out) {
  return Guard(ctx, [&](Ctx& c) {
    if ((n && !in) || !out) throw InvalidArgument("null arrays");
    DevBuf<uint32_t> in_buf;
    DevBuf<uint64_t> out_buf;
    const uint32_t* d_in = in;
    if (n && !OnDevice(in)) {
      d_in = in_buf.reserve(n);
      RVN_CUDA(cudaMemcpyAsync(const_cast<uint32_t*>(d_in), in, sizeof(uint32_t) * n,
                               cudaMemcpyHostToDevice, c.stream));
    }
    uint64_t* d_out = OnDevice(out) ? out : out_buf.reserve(n + 1);
    ExclusiveScanU32(c, d_in, d_out, n);
    if (d_out != out) {
      RVN_CUDA(cudaMemcpyAsync(out, d_out, sizeof(uint64_t) * (n + 1), cudaMemcpyDeviceToHost,
                               c.stream));
    }
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  });
}

RVN_API int rvn_get_stats(rvn_ctx* ctx, rvn_stats* out) {
  return Guard(ctx, [&](Ctx& c) {
    if (!out) throw InvalidArgument("null stats");
    *out = c.stats;
    out->occurrence = c.occurrence;
    out->kernel_launches = c.launches;
  }, /*sketches_first=*/true);
}

RVN_API int rvn_set_option(rvn_ctx* ctx, const char* name, int64_t value) {
  return Guard(ctx, [&](Ctx& c) { SetOption(c, name, value); }, /*sketches_first=*/true);
}

RVN_API int rvn_get_timings(rvn_ctx* ctx, const char* const** names,
                            const float** ms, uint32_t* n) {
  return Guard(ctx, [&](Ctx& c) {
    TimerCollect(c);
    if (names) *names = c.timer.names.data();
    if (ms) *ms = c.timer.ms.data();
    if (n) *n = static_cast<uint32_t>(c.timer.names.size());
  }, /*sketches_first=*/true);
}

// ---- multi-GPU building blocks (dist.cu); device pointers in and out ----
RVN_API int rvn_dist_sketch_split(rvn_ctx* ctx, uint32_t first, uint32_t last,
                                  int minhash, uint32_t n_parts,
                                  const uint64_t** d_value, const uint64_t** d_origin,
                                  uint64_t* counts) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    if (!d_value || !d_origin || !counts) throw InvalidArgument("null output");
    DistSketchSplit(c, first, last, minhash ? 1 : 0, n_parts, d_value, d_origin, counts);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_dist_index_limited(rvn_ctx* ctx, const uint64_t* d_value,
                                   const uint64_t* d_origin, uint64_t n_records,
                                   uint64_t index_bases, uint64_t value_limit) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_records && (!d_value || !d_origin)) throw InvalidArgument("null records");
    c.i_first = c.i_last = 0;
    // (a rank owns 1/N of the keys of every group of equal upper bits: from about four
    //  ranks on, counting inside groups costs more than a third pass over the bare keys)
    c.group_count_min = n_records >= (1ULL << 22) ? 256 : 0;  // (small slices: not worth deciding)
    try {
      BuildIndexFrom(c, ValView{d_value, 0}, d_origin, n_records, index_bases, value_limit);
    } catch (...) {
      c.group_count_min = 0;
      throw;
    }
    c.group_count_min = 0;
    // (records of a partitioned run arrive in read order: the caller's contract)
    c.i_sorted_ids = c.ids_ascending;
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  });
}

RVN_API int rvn_dist_index(rvn_ctx* ctx, const uint64_t* d_value,
                           const uint64_t* d_origin, uint64_t n_records,
                           uint64_t index_bases) {
  return rvn_dist_index_limited(ctx, d_value, d_origin, n_records, index_bases, ~0ULL);
}

RVN_API int rvn_dist_max_threshold(rvn_ctx* ctx, uint32_t first, uint32_t last,
                                   uint64_t* value) {
  return Guard(ctx, [&](Ctx& c) {
    if (!value) throw InvalidArgument("null output");
    if (first > last) throw InvalidArgument("empty range");
    *value = 0;
    if (first == last) return;
    CheckRange(c, first, last);
    *value = MaxMicromizerValue(c, first, last);
  });
}

RVN_API int rvn_dist_histogram(rvn_ctx* ctx, const uint64_t** d_hist, uint32_t* n_bins,
                               uint64_t* n_keys) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.i_valid) throw StateError("Filter before Minimize");
    if (!d_hist) throw InvalidArgument("null output");
    *d_hist = IndexHistogram(c);
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    if (n_bins) *n_bins = 65536;
    if (n_keys) *n_keys = c.i_keys;
  });
}

RVN_API int rvn_dist_set_occurrence(rvn_ctx* ctx, const uint64_t* hist, uint64_t n_keys,
                                    double frequency, uint32_t* occurrence) {
  return Guard(ctx, [&](Ctx& c) {
    if (!(0 <= frequency && frequency <= 1)) {
      throw InvalidArgument("[ram::MinimizerEngine::Filter] error: invalid frequency");
    }
    if (!c.i_valid) throw StateError("Filter before Minimize");
    if (frequency == 0 || n_keys == 0) {
      c.occurrence = 0xFFFFFFFFu;
    } else {
      if (!hist) throw InvalidArgument("null histogram");
      bool long_runs = false;
      const uint32_t occ = ThresholdFromHistogram(c, hist, n_keys, frequency, &long_runs);
      if (long_runs) throw LimitError("occurrence threshold above 65534 postings");
      c.occurrence = occ;
    }
    if (occurrence) *occurrence = c.occurrence;
  });
}

RVN_API int rvn_dist_hits_split(rvn_ctx* ctx, const uint64_t* d_qvalue,
                                const uint64_t* d_qorigin, uint64_t n_queries,
                                int avoid_equal, int avoid_symmetric, uint32_t n_parts,
                                uint32_t n_query_reads, const uint64_t** d_group,
                                const uint64_t** d_positions, const uint32_t** d_lhs,
                                uint64_t* counts) {
  return Guard(ctx, [&](Ctx& c) {
    if (!d_group || !d_positions || !d_lhs || !counts) throw InvalidArgument("null argument");
    if (n_queries && (!d_qvalue || !d_qorigin)) throw InvalidArgument("null queries");
    DistHitsSplit(c, d_qvalue, d_qorigin, n_queries, avoid_equal != 0,
                  avoid_symmetric != 0, n_parts, n_query_reads, d_group, d_positions, d_lhs,
                  counts);
  });
}

RVN_API int rvn_dist_chain(rvn_ctx* ctx, const uint64_t* d_group,
                           const uint64_t* d_positions, const uint32_t* d_lhs,
                           uint64_t n_hits, uint32_t n_runs, const uint64_t* run_off,
                           uint32_t n_parts, uint32_t rank, uint32_t n_query_reads,
                           const rvn_overlap** d_overlaps, uint64_t* n_overlaps) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_hits && (!d_group || !d_positions || !d_lhs)) throw InvalidArgument("null hits");
    if (!d_overlaps || !n_overlaps || !run_off) throw InvalidArgument("null argument");
    DistChainOwned(c, d_group, d_positions, d_lhs, n_hits, n_runs, run_off, n_parts, rank,
                   n_query_reads, d_overlaps, n_overlaps);
  });
}

RVN_API int rvn_dist_overlaps_split(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank,
                                    const rvn_overlap** d_overlaps, uint64_t* counts) {
  return Guard(ctx, [&](Ctx& c) {
    if (!d_overlaps || !counts) throw InvalidArgument("null output");
    DistOverlapsSplit(c, n_parts, rank, d_overlaps, counts);
  });
}

RVN_API int rvn_dist_stage1_begin(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank) {
  return Guard(ctx, [&](Ctx& c) {
    c.s_valid = c.q_valid = c.qt_valid = c.i_valid = c.r_valid = false;
    TimerReset(c);
    std::memset(&c.stats, 0, sizeof(c.stats));
    DistStage1Begin(c, n_parts, rank);
  });
}

RVN_API int rvn_dist_stage1_add(rvn_ctx* ctx, const rvn_overlap* d_overlaps,
                                uint64_t n_overlaps, uint32_t n_runs,
                                const uint64_t* run_off, uint32_t n_query_reads,
                                uint64_t max_overlaps, uint64_t query_batch_bases) {
  return Guard(ctx, [&](Ctx& c) {
    if (!run_off) throw InvalidArgument("null run offsets");
    if (n_overlaps && !d_overlaps) throw InvalidArgument("null overlaps");
    DistStage1Add(c, d_overlaps, n_overlaps, n_runs, run_off, n_query_reads, max_overlaps,
                  query_batch_bases);
  });
}

RVN_API int rvn_dist_stage1_end(rvn_ctx* ctx) {
  return Guard(ctx, [&](Ctx& c) { DistStage1End(c); });
}

RVN_API int rvn_dist_stage1_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                                    const uint64_t** overlap_off, const uint16_t** pile,
                                    const uint64_t** pile_off, uint32_t* n_owned,
                                    uint64_t* n_mapped) {
  return Guard(ctx, [&](Ctx& c) {
    if (!c.ds_results_valid) throw StateError("no partitioned stage-1 results");
    if (overlaps) *overlaps = c.ds_r_ovl.get();
    if (overlap_off) *overlap_off = c.ds_r_ovl_off.get();
    if (pile) *pile = c.ds_r_pile.get();
    if (pile_off) *pile_off = c.ds_r_pile_off.get();
    if (n_owned) *n_owned = c.ds_n_own;
    if (n_mapped) *n_mapped = c.st_mapped;
  });
}

// ---- peer-memory exchange (dist.cu) ----
RVN_API int rvn_dist_arena_export(rvn_ctx* ctx, uint64_t bytes, void* handle64) {
  return Guard(ctx, [&](Ctx& c) {
    if (!handle64) throw InvalidArgument("null handle");
    ArenaExport(c, bytes, handle64);
  });
}

RVN_API int rvn_dist_arena_import(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank,
                                  const void* handles) {
  return Guard(ctx, [&](Ctx& c) {
    if (!handles) throw InvalidArgument("null handles");
    ArenaImport(c, n_parts, rank, handles);
  });
}

RVN_API int rvn_dist_arena_close_peers(rvn_ctx* ctx) {
  return Guard(ctx, [&](Ctx& c) { ArenaClosePeers(c); });
}

RVN_API int rvn_dist_arena(rvn_ctx* ctx, void** d_arena, uint64_t* bytes) {
  return Guard(ctx, [&](Ctx& c) {
    if (d_arena) *d_arena = c.x_arena;
    if (bytes) *bytes = c.x_cap;
  });
}

RVN_API int rvn_dist_put(rvn_ctx* ctx, uint32_t dest, uint64_t dst_offset,
                         const void* d_src, uint64_t bytes) {
  return Guard(ctx, [&](Ctx& c) {
    if (dst_offset + bytes > c.x_cap) throw LimitError("arena overflow");
    ArenaPut(c, dest, dst_offset, d_src, bytes);
  });
}

RVN_API int rvn_dist_put_flush(rvn_ctx* ctx) {
  return Guard(ctx, [&](Ctx& c) { ArenaFlush(c); });
}

}  // extern "C"
