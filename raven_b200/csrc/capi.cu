// raven_b200 — the C ABI (include/raven_b200.h) over the overlap engine: argument
// checks and dispatch to the engine (the stage drivers are in stage.cu).
#include <algorithm>
#include <cstdlib>
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

// the calls that work on the uploaded reads
void CheckReadSet(const Ctx& c) {
  if (c.reads_unset) throw StateError("no read set: the last rvn_reads_upload_files failed");
}

void CheckRange(const Ctx& c, uint32_t first, uint32_t last) {
  CheckReadSet(c);
  if (first > last || last > c.n_reads) {
    throw InvalidArgument("read range out of bounds");
  }
}

void SetOption(Ctx& c, const char* name, int64_t value) {
  if (name && std::strcmp(name, "keep_hits") == 0) {
    c.keep_hits = value != 0;
  } else if (name && std::strcmp(name, "async_upload") == 0) {
    c.bases.async_upload = value != 0;
  } else if (name && std::strcmp(name, "host_bases") == 0) {
    if (value < -1 || value > 1) throw InvalidArgument("host_bases: -1 (auto), 0 or 1");
    c.bases.host_bases = value;
  } else if (name && std::strcmp(name, "host_bases_budget") == 0) {
    if (value < 0) throw InvalidArgument("host_bases_budget: bytes, 0 = the free memory");
    c.bases.host_bases_budget = static_cast<uint64_t>(value);
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
  } else if (name && std::strcmp(name, "fastx_chunk_bytes") == 0) {
    if (value < 0) throw InvalidArgument("fastx_chunk_bytes: bytes, 0 = 256 MiB");
    c.fastx_chunk_bytes = static_cast<uint64_t>(value);
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
  ReleaseBases(ctx->c);
  if (ctx->c.d2h_stream) {
    cudaStreamSynchronize(ctx->c.d2h_stream);
    cudaStreamDestroy(ctx->c.d2h_stream);
    cudaEventDestroy(ctx->c.d2h_ready);
    cudaEventDestroy(ctx->c.d2h_done);
  }
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
    MarkStale(c, Stale::kIndex);
    c.tiles_k = 0;  // the tile table depends on (k, w)
    c.occurrence = 0xFFFFFFFFu;
  });
}

RVN_API int rvn_reads_upload(rvn_ctx* ctx, const uint64_t* words,
                             const uint64_t* word_off, const uint32_t* lens,
                             uint32_t n_reads) {
  return Guard(ctx, [&](Ctx& c) {
    UploadReads(c, words, word_off, lens, nullptr, n_reads, 0, 0xFFFFFFFFu, /*whole_set=*/true);
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
    UploadReads(c, words, word_off, lens, ids, n_reads, 0, 0xFFFFFFFFu, /*whole_set=*/true);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_reads_upload_files(rvn_ctx* ctx, const char* const* paths, uint32_t n_paths,
                                   uint64_t sizes[4]) {
  return Guard(ctx, [&](Ctx& c) {
    if (n_paths && !paths) throw InvalidArgument("null paths");
    UploadFiles(c, paths, n_paths);
    TimerCollect(c);
    if (sizes) {
      sizes[0] = c.n_reads;
      sizes[1] = c.n_words;
      sizes[2] = c.fx_bq.size();
      sizes[3] = c.fx_names.size();
    }
  });
}

RVN_API int rvn_reads_parsed(rvn_ctx* ctx, uint64_t* words, uint64_t* word_off, uint32_t* lens,
                             uint8_t* block_quality, uint64_t* bq_off, char* names,
                             uint64_t* name_off) {
  return Guard(ctx, [&](Ctx& c) {
    ParsedReads(c, words, word_off, lens, block_quality, bq_off, names, name_off);
  });
}

// Map one read that is not part of the uploaded set (it rides in the spare
// slot behind the set for the duration of the call)
RVN_API int rvn_map_external(rvn_ctx* ctx, const uint64_t* words, uint32_t len,
                             uint32_t id, int avoid_equal, int avoid_symmetric,
                             int minhash, int want_filtered) {
  return Guard(ctx, [&](Ctx& c) {
    CheckReadSet(c);
    if (!c.i_valid) throw StateError("Map before Minimize");
    if (len >= (1u << 31)) throw LimitError("read of 2^31 or more bases");
    if (len && !words) throw InvalidArgument("null read");
    const uint32_t n = c.n_reads;
    RiderRead rider(c, words, len, id);
    // an id below an indexed id breaks the "kept postings are a suffix" shortcut
    // only through avoid_symmetric, which compares ids, not indices: fine
    MapRange(c, n, n + 1, avoid_equal != 0, avoid_symmetric != 0, minhash != 0,
             want_filtered != 0);
    TimerCollect(c);
  });
}

RVN_API int rvn_minimize(rvn_ctx* ctx, uint32_t first, uint32_t last,
                         int minhash) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    Minimize(c, first, last, minhash != 0);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_filter(rvn_ctx* ctx, double frequency, uint32_t* occurrence) {
  return Guard(ctx, [&](Ctx& c) {
    const uint32_t occ = Filter(c, frequency);
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
    EnsureDeviceBases(c);
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
    EnsureDeviceBases(c);
    KmerComplexity(c, read_index, positions, n, kmer_len, keep);
  });
}

RVN_API int rvn_find_overlaps_and_create_piles(rvn_ctx* ctx, double frequency,
                                               uint64_t max_overlaps,
                                               int minhash,
                                               uint64_t index_batch_bases,
                                               uint64_t query_batch_bases) {
  return Guard(ctx, [&](Ctx& c) {
    CheckReadSet(c);
    Stage1(c, frequency, max_overlaps, minhash != 0, index_batch_bases,
           query_batch_bases);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_find_overlaps_and_repetitive_regions(rvn_ctx* ctx, double frequency,
                                                     double identity, uint32_t n_valid,
                                                     const uint32_t* region_begin,
                                                     const uint32_t* region_end) {
  return Guard(ctx, [&](Ctx& c) {
    CheckReadSet(c);
    EnsureDeviceBases(c);
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
    Stage1Footprints(c, max_overlaps, index_batch_bases, query_batch_bases, resident,
                     windowed_device, windowed_host);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_index_footprint(rvn_ctx* ctx, uint64_t index_batch_bases, uint64_t* one_shot,
                                uint64_t* chunked) {
  return Guard(ctx, [&](Ctx& c) {
    IndexFootprints(c, index_batch_bases, one_shot, chunked);
  }, /*sketches_first=*/true);
}

RVN_API int rvn_minimize_footprint(rvn_ctx* ctx, uint32_t first, uint32_t last,
                                   uint64_t* one_shot, uint64_t* chunked, uint64_t* chunk) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    MinimizeFootprints(c, first, last, one_shot, chunked, chunk);
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
    if (pile_off) *pile_off = c.h_pile_off.data();
    if (n_mapped) *n_mapped = c.st_mapped;
  });
}

RVN_API int rvn_sketch(rvn_ctx* ctx, uint32_t first, uint32_t last, int minhash,
                       const uint64_t** value, const uint64_t** origin,
                       const uint64_t** offsets, uint64_t* n_records) {
  return Guard(ctx, [&](Ctx& c) {
    CheckRange(c, first, last);
    const uint32_t nr = last - first;
    EnsureSketch(c, first, last);
    if (minhash) EnsureMicromizers(c, first, last);
    const RecordSet& set = minhash ? c.mm : c.sk;
    const uint64_t total = set.n;
    uint64_t* hv = c.x_val.reserve(total + 1);
    uint64_t* ho = c.x_org.reserve(total + 1);
    uint64_t* hf = c.x_off.reserve(nr + 2ULL);
    const bool v32 = set.is32;  // k <= 15: u32 values
    RVN_CUDA(cudaMemcpyAsync(hv, set.val.get(), total * (v32 ? 4 : 8), cudaMemcpyDeviceToHost,
                             c.stream));
    RVN_CUDA(cudaMemcpyAsync(ho, set.org.get(), total * 8, cudaMemcpyDeviceToHost, c.stream));
    for (uint32_t i = 0; i <= nr; ++i) hf[i] = set.h_off[i];
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
    EnsureDeviceBases(c);
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
    EnsureDeviceBases(c);
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

RVN_API int rvn_reads_residency(rvn_ctx* ctx, int* on_host, uint64_t* device_word_bytes) {
  return Guard(ctx, [&](Ctx& c) {
    if (on_host) *on_host = c.bases.on_host ? 1 : 0;
    if (device_word_bytes) {
      *device_word_bytes =
          c.bases.on_host ? StagedBaseBytes(c) : c.d_words.cap * sizeof(uint64_t);
    }
  }, /*sketches_first=*/true);
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
    MarkStale(c, Stale::kIndex);
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
