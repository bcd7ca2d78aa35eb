// raven_b200 — ram::MinimizerEngine facade over the C ABI (include/raven_b200.h).
// Same signatures, argument meaning and error behaviour as the reference's
// dependency (call sites: RavenLib/src/construct.cc:42-44,62,363,372,377-381,
// 661-662; assemble.cc:753-780).
#include "ram/minimizer_engine.hpp"

#include <algorithm>
#include <stdexcept>
#include <string>

#include "raven_b200.h"

namespace ram {

namespace {

void Check(rvn_ctx* ctx, int rc, const char* what) {
  if (rc == RVN_OK) return;
  std::string msg = std::string("[ram::MinimizerEngine::") + what + "] error: " +
                    (ctx ? rvn_last_error(ctx) : "no context");
  if (rc == RVN_ERR_INVALID) throw std::invalid_argument(msg);
  throw std::runtime_error(msg);
}

}  // namespace

MinimizerEngine::MinimizerEngine(
    std::shared_ptr<thread_pool::ThreadPool> thread_pool, std::uint32_t k,
    std::uint32_t w, std::uint32_t bandwidth, std::uint32_t chain,
    std::uint32_t matches, std::uint32_t gap)
    : ctx_(nullptr),
      mutex_(new std::mutex()),
      occurrence_(-1),
      counters_{0, 0, 0},
      thread_pool_(thread_pool) {
  int rc = rvn_ctx_create(0, nullptr, &ctx_);
  if (rc != RVN_OK) {
    // no CPU fallback: the GPU engine is the only implementation
    throw std::runtime_error(
        "[ram::MinimizerEngine::MinimizerEngine] error: no usable CUDA device");
  }
  Check(ctx_, rvn_engine_configure(ctx_, k, w, bandwidth, chain, matches, gap),
        "MinimizerEngine");
}

MinimizerEngine::MinimizerEngine(MinimizerEngine&& o) noexcept
    : ctx_(o.ctx_),
      mutex_(std::move(o.mutex_)),
      occurrence_(o.occurrence_),
      resident_(std::move(o.resident_)),
      batches_(std::move(o.batches_)),
      counters_(o.counters_),
      thread_pool_(std::move(o.thread_pool_)) {
  o.ctx_ = nullptr;
}

MinimizerEngine& MinimizerEngine::operator=(MinimizerEngine&& o) noexcept {
  if (this != &o) {
    if (ctx_) rvn_ctx_destroy(ctx_);
    ctx_ = o.ctx_;
    o.ctx_ = nullptr;
    mutex_ = std::move(o.mutex_);
    occurrence_ = o.occurrence_;
    resident_ = std::move(o.resident_);
    batches_ = std::move(o.batches_);
    counters_ = o.counters_;
    thread_pool_ = std::move(o.thread_pool_);
  }
  return *this;
}

MinimizerEngine::~MinimizerEngine() {
  if (ctx_) rvn_ctx_destroy(ctx_);
}

void MinimizerEngine::Append(Resident& r, Iterator first, Iterator last) {
  for (auto it = first; it != last; ++it) {
    if ((*it)->is_reverse_complement) {
      throw std::invalid_argument(
          "[ram::MinimizerEngine::Minimize] error: reverse-complemented view");
    }
  }
  // deflated_data is already the device format: concatenate, never repack
  for (auto it = first; it != last; ++it) {
    const auto& s = **it;
    r.position[s.id] = static_cast<std::uint32_t>(r.lens.size());
    r.words.insert(r.words.end(), s.deflated_data.begin(), s.deflated_data.end());
    r.off.push_back(r.words.size());
    r.lens.push_back(s.inflated_len);
    r.ids.push_back(s.id);
    r.objects.push_back(&s);
  }
}

void MinimizerEngine::UploadResident(const Resident& r) {
  Check(ctx_,
        rvn_reads_upload_ids(ctx_, r.words.data(), r.off.data(), r.lens.data(),
                             r.ids.data(), static_cast<std::uint32_t>(r.lens.size())),
        "Minimize");
}

void MinimizerEngine::UploadRange(Iterator first, Iterator last) {
  resident_.batch_first = 0;
  resident_.next = nullptr;
  // the same objects as last time (stage 1 -> identity filter): nothing to move
  {
    const std::size_t n = static_cast<std::size_t>(last - first);
    bool same = n > 0 && n == resident_.lens.size();
    std::size_t pos = 0;
    for (auto it = first; same && it != last; ++it, ++pos) {
      same = resident_.objects[pos] == it->get() && resident_.ids[pos] == (*it)->id;
    }
    if (same) return;
  }
  resident_ = Resident();
  Resident r;
  Append(r, first, last);
  UploadResident(r);
  resident_ = std::move(r);
}

void MinimizerEngine::Upload(
    const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences) {
  std::lock_guard<std::mutex> lock(*mutex_);
  batches_.clear();
  UploadRange(sequences.begin(), sequences.end());
}

void MinimizerEngine::Upload(Iterator first, Iterator last) {
  std::lock_guard<std::mutex> lock(*mutex_);
  batches_.clear();
  UploadRange(first, last);
}

void MinimizerEngine::Minimize(Iterator first, Iterator last, bool minhash) {
  std::lock_guard<std::mutex> lock(*mutex_);
  occurrence_ = -1;
  batches_.clear();
  if (first >= last) {
    UploadRange(first, first);
  } else if (resident_.next == &*first) {
    // the next index batch of a pass (construct.cc:32-43): the earlier batches
    // stay on the device as queries, the index covers this batch alone
    Resident r = std::move(resident_);
    resident_ = Resident();
    const auto j = static_cast<std::uint32_t>(r.lens.size());
    Append(r, first, last);
    UploadResident(r);
    r.batch_first = j;
    resident_ = std::move(r);
  } else {
    UploadRange(first, last);
  }
  if (first < last) resident_.next = &*(last - 1) + 1;
  Check(ctx_,
        rvn_minimize(ctx_, resident_.batch_first,
                     static_cast<std::uint32_t>(resident_.lens.size()), minhash),
        "Minimize");
}

void MinimizerEngine::Filter(double frequency) {
  std::lock_guard<std::mutex> lock(*mutex_);
  batches_.clear();
  Check(ctx_, rvn_filter(ctx_, frequency, &occurrence_), "Filter");
}

MinimizerEngine::MapCounters MinimizerEngine::map_counters() const {
  std::lock_guard<std::mutex> lock(*mutex_);
  return counters_;
}

std::int64_t MinimizerEngine::ResidentPosition(const biosoup::NucleicAcid& s) const {
  if (s.is_reverse_complement) return -1;
  const auto it = resident_.position.find(s.id);
  if (it == resident_.position.end()) return -1;
  const std::uint32_t p = it->second;
  if (resident_.lens[p] != s.inflated_len) return -1;
  const auto w = resident_.words.begin();
  if (!std::equal(w + resident_.off[p], w + resident_.off[p + 1], s.deflated_data.begin(),
                  s.deflated_data.end())) {
    return -1;  // changed since it was uploaded
  }
  return p;
}

MinimizerEngine::BatchResults& MinimizerEngine::Results(bool avoid_equal,
                                                        bool avoid_symmetric,
                                                        bool minhash,
                                                        bool want_filtered) const {
  for (auto& b : batches_) {
    if (b.avoid_equal == avoid_equal && b.avoid_symmetric == avoid_symmetric &&
        b.minhash == minhash && b.want_filtered == want_filtered) {
      return b;
    }
  }
  const auto n = static_cast<std::uint32_t>(resident_.lens.size());
  const std::uint32_t j = resident_.batch_first;
  BatchResults b{avoid_equal, avoid_symmetric, minhash, want_filtered, {}, {0}, {}, {0},
                 std::vector<bool>(n, false), n};
  // the earlier batches' reads take the probe path; the batch's own reads keep
  // the self-join, which needs a range inside the index batch
  for (const auto& range : {std::make_pair(0u, j), std::make_pair(j, n)}) {
    if (range.first == range.second) continue;
    Check(ctx_,
          rvn_map(ctx_, range.first, range.second, avoid_equal, avoid_symmetric, minhash,
                  want_filtered),
          "Map");
    ++counters_.batch_maps;
    const rvn_overlap* o = nullptr;
    const std::uint64_t* off = nullptr;
    const std::uint32_t* f = nullptr;
    const std::uint64_t* foff = nullptr;
    std::uint64_t total = 0;
    Check(ctx_, rvn_map_results(ctx_, &o, &off, &total, &f, &foff), "Map");
    const std::uint32_t m = range.second - range.first;
    const std::uint64_t base = b.overlaps.size();
    b.overlaps.insert(b.overlaps.end(), o + off[0], o + off[m]);
    for (std::uint32_t r = 1; r <= m; ++r) b.overlap_off.push_back(base + off[r] - off[0]);
    const std::uint64_t fbase = b.filtered.size();
    if (want_filtered) b.filtered.insert(b.filtered.end(), f + foff[0], f + foff[m]);
    for (std::uint32_t r = 1; r <= m; ++r) {
      b.filtered_off.push_back(want_filtered ? fbase + foff[r] - foff[0] : fbase);
    }
  }
  batches_.emplace_back(std::move(b));
  return batches_.back();
}

std::vector<biosoup::Overlap> MinimizerEngine::Map(
    const std::unique_ptr<biosoup::NucleicAcid>& sequence, bool avoid_equal,
    bool avoid_symmetric, bool minhash,
    std::vector<std::uint32_t>* filtered) const {
  std::lock_guard<std::mutex> lock(*mutex_);
  const auto& s = *sequence;
  std::vector<biosoup::Overlap> dst;
  const std::int64_t pos = ResidentPosition(s);
  if (pos >= 0) {
    // a read on the device: from the results of the whole resident set
    auto& b = Results(avoid_equal, avoid_symmetric, minhash, filtered != nullptr);
    const auto p = static_cast<std::size_t>(pos);
    dst.reserve(b.overlap_off[p + 1] - b.overlap_off[p]);
    for (std::uint64_t i = b.overlap_off[p]; i < b.overlap_off[p + 1]; ++i) {
      const auto& o = b.overlaps[i];
      dst.emplace_back(o.lhs_id, o.lhs_begin, o.lhs_end, o.rhs_id, o.rhs_begin, o.rhs_end,
                       o.score, o.strand != 0);
    }
    if (filtered) {
      filtered->insert(filtered->end(), b.filtered.begin() + b.filtered_off[p],
                       b.filtered.begin() + b.filtered_off[p + 1]);
    }
    ++counters_.served;
    if (!b.served[p]) {
      b.served[p] = true;
      if (--b.unserved == 0) batches_.erase(batches_.begin() + (&b - batches_.data()));
    }
    return dst;
  }
  // a read that is not on the device (never minimized in this pass, changed
  // since, or a reverse-complemented view): it rides in the spare device slot
  std::vector<std::uint64_t> rc_words;
  const std::uint64_t* words = s.deflated_data.data();
  if (s.is_reverse_complement) {
    rc_words.assign((static_cast<std::uint64_t>(s.inflated_len) + 31) >> 5, 0);
    for (std::uint32_t i = 0; i < s.inflated_len; ++i) {
      rc_words[i >> 5] |= s.Code(i) << ((i << 1) & 63);
    }
    words = rc_words.data();
  }
  Check(ctx_,
        rvn_map_external(ctx_, words, s.inflated_len, s.id, avoid_equal,
                         avoid_symmetric, minhash, filtered != nullptr),
        "Map");
  ++counters_.single_maps;
  const rvn_overlap* o = nullptr;
  const std::uint64_t* off = nullptr;
  const std::uint32_t* f = nullptr;
  const std::uint64_t* foff = nullptr;
  std::uint64_t n = 0;
  Check(ctx_, rvn_map_results(ctx_, &o, &off, &n, &f, &foff), "Map");
  dst.reserve(n);
  for (std::uint64_t i = 0; i < n; ++i) {
    dst.emplace_back(o[i].lhs_id, o[i].lhs_begin, o[i].lhs_end, o[i].rhs_id,
                     o[i].rhs_begin, o[i].rhs_end, o[i].score, o[i].strand != 0);
  }
  if (filtered) {
    filtered->insert(filtered->end(), f + foff[0], f + foff[1]);
  }
  return dst;
}

}  // namespace ram
