// raven_b200 — the C ABI (include/raven_b200.h) over the overlap engine, and
// the stage-1 driver that replaces raven::FindOverlapsAndCreatePiles
// (RavenLib/src/construct.cc:14-121).
#include <algorithm>
#include <cstring>

#include "engine.cuh"

using namespace rvn;

struct rvn_ctx {
  Ctx c;
};

namespace {

template <typename F>
int Guard(rvn_ctx* ctx, F&& f, bool sketches_first = false) {
  if (!ctx) return RVN_ERR_INVALID;
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

// raven::FindOverlapsAndCreatePiles, same batch / flush schedule as the
// reference; every step runs on the GPU (Minimize, Filter, Map, AddLayers,
// gather, truncation); the host only drives the schedule.
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
  uint16_t* d_pile = c.p_data.reserve(total_bins + 1);
  uint64_t* d_poff = c.p_off.reserve(n + 1ULL);
  RVN_CUDA(cudaMemsetAsync(d_pile, 0, (total_bins + 1) * sizeof(uint16_t), c.stream));
  if (!c.p_off_uploaded) {  // (an asynchronous upload has sent them ahead of the bases)
    RVN_CUDA(cudaMemcpyAsync(d_poff, c.st_pile_off.data(), (n + 1ULL) * 8,
                             cudaMemcpyHostToDevice, c.stream));
  }

  GatherReset(c);
  c.st_mapped = 0;

  uint64_t bases = 0;
  uint64_t tmax = 0;  // largest micromizer value of the reads sketched so far
  for (uint32_t i = 0, j = 0; i < n; ++i) {
    bases += c.h_len[i];
    if (i != n - 1 && bases < ib) continue;
    bases = 0;

    // Queries are micromizers only (construct.cc:62): no record above the largest
    // micromizer value of any read so far can be hit - those are counted for the
    // occurrence threshold but stay out of the index (index.cu, tiers)
    uint64_t limit = ~0ULL;
    if (!minhash) {
      tmax = std::max(tmax, MaxMicromizerValue(c, j, i + 1));
      limit = tmax;
    }
    BuildIndex(c, j, i + 1, minhash, limit);
    FilterIndex(c, freq);

    // every read up to the end of this index batch is a query, flushed per
    // >= qb bases exactly like the reference (the truncation rule makes the
    // flush boundaries observable)
    for (uint32_t k = 0, k0 = 0; k < i + 1; ++k) {
      bases += c.h_len[k];
      if (k != i && bases < qb) continue;
      bases = 0;

      MapRange(c, k0, k + 1, true, true, true, false, /*fetch=*/false);
      PileAddLayersDevice(c, d_pile, d_poff, c.st_pile_off.data(), n,
                          c.m_ovl.get(), c.r_n_ovl);
      GatherFlush(c, c.m_ovl.get(), c.m_ovl_off.get(), c.r_n_ovl, k0, k + 1, kmax);
      c.st_mapped += c.r_n_ovl;
      k0 = k + 1;
    }
    j = i + 1;
  }

  GatherFetch(c);
  RVN_CUDA(cudaMemcpyAsync(c.st_pile.reserve(total_bins + 1), d_pile, total_bins * sizeof(uint16_t),
                           cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaStreamSynchronize(c.stream));
  TimerCollect(c);
  c.stats.kernel_launches = c.launches - launches0;
  c.stats.occurrence = c.occurrence;
  c.st_valid = true;
  c.st_piles_on_device = true;
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
    BuildIndex(c, first, last, minhash != 0);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_filter(rvn_ctx* ctx, double frequency, uint32_t* occurrence) {
  return Guard(ctx, [&](Ctx& c) {
    uint32_t occ = FilterIndex(c, frequency);
    if (occurrence) *occurrence = occ;
  });
}

RVN_API int rvn_map(rvn_ctx* ctx, uint32_t first, uint32_t last,
                    int avoid_equal, int avoid_symmetric, int minhash,
                    int want_filtered) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    MapRange(c, first, last, avoid_equal != 0, avoid_symmetric != 0,
             minhash != 0, want_filtered != 0);
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
    PileAddLayersDevice(c, d, off, bin_off, n_piles, o, n_overlaps);
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

// the engine's radix sort on host arrays (parity tests of radix.cu)
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
    if (n && (!keys || (val_bytes && !vals))) throw InvalidArgument("null arrays");
    DevBuf<uint8_t> ks, ka, kb, vs, va, vb;
    const size_t kb_ = static_cast<size_t>(key_bytes) * n + 16, vb_ = static_cast<size_t>(val_bytes) * n + 16;
    ks.reserve(kb_); ka.reserve(kb_); kb.reserve(kb_);
    vs.reserve(vb_); va.reserve(vb_); vb.reserve(vb_);
    RVN_CUDA(cudaMemcpyAsync(ks.get(), keys, static_cast<size_t>(key_bytes) * n, cudaMemcpyHostToDevice, c.stream));
    if (val_bytes) {
      RVN_CUDA(cudaMemcpyAsync(vs.get(), vals, static_cast<size_t>(val_bytes) * n, cudaMemcpyHostToDevice, c.stream));
    }
    int where;
    const bool desc = descending != 0;
    if (val_bytes == 0) {
      where = RadixSortKeys(c, (const uint32_t*)ks.get(), (uint32_t*)ka.get(), (uint32_t*)kb.get(), n,
                            begin_bit, end_bit);
    } else if (key_bytes == 4 && val_bytes == 8) {
      where = RadixSortPairs(c, (const uint32_t*)ks.get(), (uint32_t*)ka.get(), (uint32_t*)kb.get(),
                             (const uint64_t*)vs.get(), (uint64_t*)va.get(), (uint64_t*)vb.get(), n,
                             begin_bit, end_bit, desc);
    } else if (key_bytes == 8 && val_bytes == 8) {
      where = RadixSortPairs(c, (const uint64_t*)ks.get(), (uint64_t*)ka.get(), (uint64_t*)kb.get(),
                             (const uint64_t*)vs.get(), (uint64_t*)va.get(), (uint64_t*)vb.get(), n,
                             begin_bit, end_bit, desc);
    } else if (key_bytes == 4 && val_bytes == 4) {
      where = RadixSortPairs(c, (const uint32_t*)ks.get(), (uint32_t*)ka.get(), (uint32_t*)kb.get(),
                             (const uint32_t*)vs.get(), (uint32_t*)va.get(), (uint32_t*)vb.get(), n,
                             begin_bit, end_bit, desc);
    } else {
      where = RadixSortPairs(c, (const uint64_t*)ks.get(), (uint64_t*)ka.get(), (uint64_t*)kb.get(),
                             (const uint32_t*)vs.get(), (uint32_t*)va.get(), (uint32_t*)vb.get(), n,
                             begin_bit, end_bit, desc);
    }
    const uint8_t* rk = where < 0 ? ks.get() : (where == 0 ? ka.get() : kb.get());
    const uint8_t* rv = where < 0 ? vs.get() : (where == 0 ? va.get() : vb.get());
    RVN_CUDA(cudaMemcpyAsync(keys, rk, static_cast<size_t>(key_bytes) * n, cudaMemcpyDeviceToHost, c.stream));
    if (val_bytes) {
      RVN_CUDA(cudaMemcpyAsync(vals, rv, static_cast<size_t>(val_bytes) * n, cudaMemcpyDeviceToHost, c.stream));
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
  return Guard(ctx, [&](Ctx& c) {
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
    } else if (name && std::strcmp(name, "reset_stats") == 0) {
      std::memset(&c.stats, 0, sizeof(c.stats));
      c.launches = 0;
      TimerReset(c);
    } else {
      throw InvalidArgument("unknown option");
    }
  }, /*sketches_first=*/true);
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
