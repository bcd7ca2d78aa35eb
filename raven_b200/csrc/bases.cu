// raven_b200 — where the packed bases of the uploaded reads are (Ctx::bases): the upload
// (to d_words, at once or in pieces on the copy stream behind which the next sketch starts;
// or, option host_bases, to the context's pinned host copy), the staging window that brings
// the range a sketch reads to the device, the residency check of the calls that read bases,
// rvn_map_external's rider read, and the teardown.
#include <algorithm>
#include <cstring>

#include "engine.cuh"

namespace rvn {

namespace {

// A range of kPiecewiseReads reads or more (an asynchronous upload always is) is copied in
// this many pieces of about equal words, cut at read boundaries: the sketch of the reads of a
// piece starts when it has arrived. A smaller staged range is one piece.
constexpr uint32_t kCopyPieces = 8;
constexpr uint32_t kPiecewiseReads = 1024;

void EnsureCopyStream(Ctx& c) {
  Bases& b = c.bases;
  if (b.copy_stream) return;
  RVN_CUDA(cudaStreamCreateWithFlags(&b.copy_stream, cudaStreamNonBlocking));
  RVN_CUDA(cudaEventCreateWithFlags(&b.up_fence, cudaEventDisableTiming));
}

// Copy of the words of reads [first, last) from src to dst (both pointing at the first read's
// first word) on the copy stream, in pieces that end at read boundaries, with an event
// recorded behind each.
void CopyReads(Ctx& c, CopyPieces& p, uint32_t first, uint32_t last, uint64_t* dst,
               const uint64_t* src) {
  const uint64_t w0 = c.h_woff[first], w1 = c.h_woff[last];
  const uint32_t pieces = last - first >= kPiecewiseReads ? kCopyPieces : 1;
  while (p.events.size() < pieces) {
    cudaEvent_t ev;
    RVN_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    p.events.push_back(ev);
  }
  p.read_end.clear();
  uint32_t r_prev = first;
  for (uint32_t i = 1; i <= pieces && r_prev < last; ++i) {
    const uint64_t target = w0 + (w1 - w0) * i / pieces;
    uint32_t r = static_cast<uint32_t>(
        std::lower_bound(c.h_woff.begin() + r_prev + 1, c.h_woff.begin() + last + 1, target) -
        c.h_woff.begin());
    if (i == pieces) r = last;
    const uint64_t a = c.h_woff[r_prev], e = c.h_woff[r];
    if (e > a) {
      RVN_CUDA(cudaMemcpyAsync(dst + (a - w0), src + (a - w0), (e - a) * 8,
                               cudaMemcpyHostToDevice, c.bases.copy_stream));
    }
    RVN_CUDA(cudaEventRecord(p.events[p.read_end.size()], c.bases.copy_stream));
    p.read_end.push_back(r);
    r_prev = r;
  }
  p.n = static_cast<uint32_t>(p.read_end.size());
}

// the half that holds every read of [first, last), -1 = none
int HalfWith(const Ctx& c, uint32_t first, uint32_t last) {
  for (int i = 0; i < 2; ++i) {
    const BaseHalf& h = c.bases.half[i];
    if (h.valid && h.first <= first && last <= h.last) return i;
  }
  return -1;
}

// Copy of the words of reads [first, last) (src: their words on the host, from the first
// read's first word) into half i, on the copy stream behind every kernel that read the half.
void StageRange(Ctx& c, int i, uint32_t first, uint32_t last, const uint64_t* src) {
  Bases& b = c.bases;
  BaseHalf& h = b.half[i];
  const uint64_t nw = c.h_woff[last] - c.h_woff[first];
  h.valid = false;
  EnsureCopyStream(c);
  if (!h.used) RVN_CUDA(cudaEventCreateWithFlags(&h.used, cudaEventDisableTiming));
  if (nw + 2 > h.words.cap) {  // (growth frees the buffer: its readers must be done)
    if (h.used_recorded) RVN_CUDA(cudaEventSynchronize(h.used));
    RVN_CUDA(cudaStreamSynchronize(b.copy_stream));
    h.words.reserve(nw + 2);
  }
  if (h.used_recorded) RVN_CUDA(cudaStreamWaitEvent(b.copy_stream, h.used, 0));
  CopyReads(c, h.copy, first, last, h.words.get(), src);
  h.first = first;
  h.last = last;
  h.valid = true;
}

// the halves holding reads >= `from` forget them; release: every half frees its memory
void DropStagedBases(Ctx& c, uint32_t from, bool release) {
  Bases& b = c.bases;
  for (BaseHalf& h : b.half) {
    if (h.valid && h.last > from) h.valid = false;
    if (release && h.words.cap) {
      if (h.used_recorded) RVN_CUDA(cudaEventSynchronize(h.used));
      if (b.copy_stream) RVN_CUDA(cudaStreamSynchronize(b.copy_stream));
      h.words.release();
      h.valid = false;
    }
  }
  b.next_first = b.next_last = 0;
}

// the set before rvn_map_external's rider joined it
void RestoreSet(const RiderRead& r) {
  Ctx& c = r.c;
  if (c.bases.on_host) DropStagedBases(c, r.n, /*release=*/false);
  c.bases.res_first = r.res_first;
  c.bases.res_last = r.res_last;
  c.n_reads = r.n;
  c.h_woff.pop_back();
  c.h_len.pop_back();
  c.h_ids.pop_back();
  c.h_tile_off.pop_back();
  MarkStale(c, Stale::kThresholds);
}

// The host read tables of a new set (offsets, lengths, pile offsets, ids); the device
// buffers of the old set are idle when this returns.
void SetReadTables(Ctx& c, const uint64_t* word_off, const uint32_t* lens, const uint32_t* ids,
                   uint32_t n_reads) {
  if (n_reads && (!word_off || !lens)) throw InvalidArgument("null read set");
  if (n_reads == 0xFFFFFFFFu) throw LimitError("too many reads");
  MarkStale(c, Stale::kStage1);
  c.st_piles_on_device = false;
  c.reads_unset = c.fx_valid = false;
  c.tiles_k = 0;
  c.n_reads = n_reads;
  c.h_woff.assign(1, 0);
  if (n_reads) c.h_woff.assign(word_off, word_off + n_reads + 1);
  c.h_len.assign(lens, lens + n_reads);
  // piles: len >> 4 bins each (pile.cc:19-31)
  c.h_pile_off.assign(n_reads + 1ULL, 0);
  for (uint32_t i = 0; i < n_reads; ++i) c.h_pile_off[i + 1] = c.h_pile_off[i] + (lens[i] >> 4);
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
  // (kernels and copies of earlier calls may still use the buffers of the old bases)
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  if (c.bases.copy_stream) RVN_CUDA(cudaStreamSynchronize(c.bases.copy_stream));
}

// offsets, lengths, ids to the device (small, from pageable memory: behind the bases they
// would wait for the copy engine); one spare slot everywhere: an external query read rides
// at index n_reads
void UploadReadTables(Ctx& c) {
  const uint32_t n_reads = c.n_reads;
  uint64_t* dwo = c.d_woff.reserve(n_reads + 2ULL);
  uint32_t* dl = c.d_len.reserve(n_reads + 2ULL);
  uint32_t* di = c.d_ids.reserve(n_reads + 2ULL);
  RVN_CUDA(cudaMemcpyAsync(dwo, c.h_woff.data(), (n_reads + 1ULL) * 8,
                           cudaMemcpyHostToDevice, c.stream));
  if (n_reads) {
    RVN_CUDA(cudaMemcpyAsync(dl, c.h_len.data(), n_reads * 4ULL,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaMemcpyAsync(di, c.h_ids.data(), n_reads * 4ULL,
                             cudaMemcpyHostToDevice, c.stream));
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));
}

}  // namespace

void UploadReads(Ctx& c, const uint64_t* words, const uint64_t* word_off, const uint32_t* lens,
                 const uint32_t* ids, uint32_t n_reads, uint32_t res_first, uint32_t res_last,
                 bool whole_set) {
  Bases& b = c.bases;
  res_last = std::min(res_last, n_reads);
  if (res_first > res_last) throw InvalidArgument("resident range out of bounds");
  SetReadTables(c, word_off, lens, ids, n_reads);
  b.on_host = whole_set && UseHostBases(c);
  if (b.on_host) {
    // the context's own pinned copy (the caller may change its words once this returns);
    // the sketch kernels read it through the staging window
    if (c.n_words && !words) throw InvalidArgument("null read set");
    DropStagedBases(c, 0, /*release=*/false);
    uint64_t* hw = b.h_words.reserve(c.n_words + 2);
    if (c.n_words) std::memcpy(hw, words, c.n_words * sizeof(uint64_t));
    c.d_words.release();
  } else {
    DropStagedBases(c, 0, /*release=*/true);
  }
  uint64_t* dw = b.on_host ? nullptr : c.d_words.reserve(c.n_words + 2);
  // bases of the resident reads only (a rank of a partitioned run sketches its
  // own range; lengths and ids of all reads are always resident)
  b.res_first = res_first;
  b.res_last = res_last;
  UploadReadTables(c);
  const uint64_t w0 = c.h_woff[res_first], w1 = c.h_woff[res_last];
  b.upload.n = 0;
  c.p_off_uploaded = false;
  if (b.on_host) return;  // (async_upload has nothing left to do)
  if (w1 > w0 && c.bases.async_upload && res_last - res_first >= kPiecewiseReads) {
    // everything small the next call would send host-to-device goes first: behind the
    // bases it would wait for the copy engine (tile tables, pile offsets of stage 1)
    EnsureTiles(c);
    uint64_t* d_poff = c.p_off.reserve(n_reads + 1ULL);
    RVN_CUDA(cudaMemcpyAsync(d_poff, c.h_pile_off.data(), (n_reads + 1ULL) * 8,
                             cudaMemcpyHostToDevice, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    c.p_off_uploaded = true;
    // pieces on the copy stream, behind the kernels of earlier calls that may still read the
    // old bases; the caller keeps `words` alive until the next call on this context has
    // returned
    EnsureCopyStream(c);
    RVN_CUDA(cudaEventRecord(b.up_fence, c.stream));
    RVN_CUDA(cudaStreamWaitEvent(b.copy_stream, b.up_fence, 0));
    CopyReads(c, b.upload, res_first, res_last, dw + w0, words + w0);
  } else if (w1 > w0) {
    RVN_CUDA(cudaMemcpyAsync(dw + w0, words + w0, (w1 - w0) * 8, cudaMemcpyHostToDevice,
                             c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));
  }
}

void AdoptParsedReads(Ctx& c, const uint64_t* word_off, const uint32_t* lens, uint32_t n_reads) {
  Bases& b = c.bases;
  SetReadTables(c, word_off, lens, nullptr, n_reads);
  b.on_host = UseHostBases(c);
  if (b.on_host) {
    DropStagedBases(c, 0, /*release=*/false);
    uint64_t* hw = b.h_words.reserve(c.n_words + 2);
    if (c.n_words) {
      RVN_CUDA(cudaMemcpyAsync(hw, c.d_words.get(), c.n_words * sizeof(uint64_t),
                               cudaMemcpyDeviceToHost, c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));
    }
    c.d_words.release();
  } else {
    DropStagedBases(c, 0, /*release=*/true);
  }
  b.res_first = 0;
  b.res_last = n_reads;
  UploadReadTables(c);
  b.upload.n = 0;
  c.p_off_uploaded = false;
}

void CheckResident(const Ctx& c, uint32_t first, uint32_t last) {
  const Bases& b = c.bases;
  if (first < last && !b.on_host && (first < b.res_first || last > b.res_last)) {
    throw StateError("the bases of these reads were not uploaded (rvn_reads_upload_range)");
  }
}

void WaitUpload(Ctx& c) {
  CopyPieces& p = c.bases.upload;
  if (!p.n) return;
  RVN_CUDA(cudaStreamWaitEvent(c.stream, p.events[p.n - 1], 0));
  p.n = 0;
}

BaseView SketchBases(Ctx& c, uint32_t first, uint32_t last) {
  Bases& b = c.bases;
  if (!b.on_host) {
    // (an asynchronous upload in flight: its pieces are this launch's to wait for)
    const BaseView v{c.d_words.get(), 0, b.upload.events.data(), b.upload.read_end.data(),
                     b.upload.n, -1};
    b.upload.n = 0;
    return v;
  }
  int i = HalfWith(c, first, last);
  if (i < 0) {
    i = 1 - b.cur;
    StageRange(c, i, first, last, b.h_words.get() + c.h_woff[first]);
  }
  b.cur = i;
  const BaseHalf& h = b.half[i];
  return BaseView{h.words.get(), c.h_woff[h.first], h.copy.events.data(),
                  h.copy.read_end.data(), h.copy.n, i};
}

void BasesLaunched(Ctx& c, const BaseView& v) {
  if (v.half < 0) return;
  Bases& b = c.bases;
  BaseHalf& h = b.half[v.half];
  RVN_CUDA(cudaEventRecord(h.used, c.stream));
  h.used_recorded = true;
  const uint32_t first = b.next_first, last = b.next_last;
  b.next_first = b.next_last = 0;
  if (first < last && last <= c.n_reads && HalfWith(c, first, last) < 0) {
    StageRange(c, 1 - v.half, first, last, b.h_words.get() + c.h_woff[first]);
  }
}

void BasesNext(Ctx& c, uint32_t first, uint32_t last) {
  if (!c.bases.on_host) return;
  c.bases.next_first = first;
  c.bases.next_last = last;
}

uint64_t StagedBaseBytes(const Ctx& c) {
  return (c.bases.half[0].words.cap + c.bases.half[1].words.cap) * sizeof(uint64_t);
}

void EnsureDeviceBases(Ctx& c) {
  Bases& b = c.bases;
  if (!b.on_host) return;
  const uint64_t bytes = (c.n_words + 2) * sizeof(uint64_t);
  const double usable = UsableMemory(c, c.bases.host_bases_budget);
  if (static_cast<double>(bytes) > usable) {
    throw LimitError("the packed bases of the whole read set (" + std::to_string(bytes) +
                     " bytes) do not fit the device (" +
                     std::to_string(static_cast<uint64_t>(usable)) + " bytes usable)");
  }
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  DropStagedBases(c, 0, /*release=*/true);
  uint64_t* dw = c.d_words.reserve(c.n_words + 2);
  RVN_CUDA(cudaMemcpyAsync(dw, b.h_words.get(), c.n_words * sizeof(uint64_t),
                           cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  b.on_host = false;
  b.res_first = 0;
  b.res_last = c.n_reads;
}

RiderRead::RiderRead(Ctx& ctx, const uint64_t* words, uint32_t len, uint32_t id)
    : c(ctx), n(ctx.n_reads), res_first(ctx.bases.res_first), res_last(ctx.bases.res_last) {
  const uint64_t nw = (static_cast<uint64_t>(len) + 31) >> 5;
  if (!c.bases.on_host) {
    uint64_t* dw = c.d_words.reserve_keep(c.n_words + nw + 2, c.n_words, c.stream);
    if (nw) {
      RVN_CUDA(cudaMemcpyAsync(dw + c.n_words, words, nw * 8, cudaMemcpyHostToDevice, c.stream));
    }
  }
  EnsureTiles(c);
  // extend the host/device tables by the spare slot
  const uint64_t woff_tail[2] = {c.n_words, c.n_words + nw};
  uint64_t tiles = 0;
  if (len >= c.prm.k && len - c.prm.k + 1 >= c.prm.w) {
    tiles = (len - c.prm.k + 1 + kSketchTile - 1) / kSketchTile;
  }
  const uint64_t tile_tail[2] = {c.h_tile_off[n], c.h_tile_off[n] + tiles};
  RVN_CUDA(cudaMemcpyAsync(c.d_woff.get() + n, woff_tail, 16, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(c.d_tile_off.get() + n, tile_tail, 16, cudaMemcpyHostToDevice,
                           c.stream));
  RVN_CUDA(cudaMemcpyAsync(c.d_len.get() + n, &len, 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(c.d_ids.get() + n, &id, 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  c.h_woff.push_back(c.n_words + nw);
  c.h_len.push_back(len);
  c.h_ids.push_back(id);
  c.h_tile_off.push_back(tile_tail[1]);
  c.n_reads = n + 1;
  MarkStale(c, Stale::kThresholds);
  // the rider's bases are the only resident ones while it rides
  c.bases.res_first = n;
  c.bases.res_last = n + 1;
  if (!c.bases.on_host) return;
  try {
    StageRange(c, 1 - c.bases.cur, n, n + 1, words);
  } catch (...) {
    RestoreSet(*this);  // (no destructor runs after a constructor throws)
    throw;
  }
}

RiderRead::~RiderRead() { RestoreSet(*this); }

void ReleaseBases(Ctx& c) {
  Bases& b = c.bases;
  if (b.copy_stream) {
    cudaStreamSynchronize(b.copy_stream);
    cudaStreamDestroy(b.copy_stream);
  }
  for (auto e : b.upload.events) cudaEventDestroy(e);
  for (auto& h : b.half) {
    for (auto e : h.copy.events) cudaEventDestroy(e);
    if (h.used) cudaEventDestroy(h.used);
  }
  if (b.up_fence) cudaEventDestroy(b.up_fence);
}

}  // namespace rvn
