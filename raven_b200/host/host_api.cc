// raven_b200 — C entry points over the C++ facades (bench.py and the tests drive
// the racon::Polisher facade through this; RavenLib links the facades directly).
//   rvnh_polish  racon::Polisher::Create(...)->Polish(targets, sequences, false)
//                (RavenLib/src/polish.cc:43-51) on flat biosoup-format read sets
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "biosoup/nucleic_acid.hpp"
#include "racon/polisher.hpp"
#include "thread_pool/thread_pool.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace {

std::vector<std::unique_ptr<biosoup::NucleicAcid>> Unflatten(
    const std::uint64_t* words, const std::uint64_t* woff, const std::uint32_t* lens,
    const std::uint8_t* bq, const std::uint64_t* bq_off, std::uint32_t n, const char* prefix) {
  std::vector<std::unique_ptr<biosoup::NucleicAcid>> v;
  v.reserve(n);
  for (std::uint32_t i = 0; i < n; ++i) {
    auto s = std::make_unique<biosoup::NucleicAcid>();
    s->id = i;
    s->name = std::string(prefix) + std::to_string(i);
    s->deflated_data.assign(words + woff[i], words + woff[i + 1]);
    s->inflated_len = lens[i];
    s->is_reverse_complement = false;
    if (bq) s->block_quality.assign(bq + bq_off[i], bq + bq_off[i + 1]);
    v.emplace_back(std::move(s));
  }
  return v;
}

struct PolishResult {
  std::vector<std::uint64_t> words, woff;
  std::vector<std::uint32_t> lens;
  std::string names, error;
  // windows, polished windows, POA seconds, total seconds, then the phases of
  // Polish: map, alignment paths, window packing, consensus, stitch, layer rules;
  // then the windows that ran on the wide consensus kernel, the window batches
  double stats[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
};

}  // namespace

extern "C" {

#define RVNH_API __attribute__((visibility("default")))

// returns a handle (never null); rvnh_polish_error(h) is "" on success
RVNH_API void* rvnh_polish(const std::uint64_t* t_words, const std::uint64_t* t_woff,
                           const std::uint32_t* t_lens, std::uint32_t n_targets,
                           const std::uint64_t* s_words, const std::uint64_t* s_woff,
                           const std::uint32_t* s_lens, const std::uint8_t* s_bq,
                           const std::uint64_t* s_bq_off, std::uint32_t n_sequences, double q,
                           double e, std::uint32_t w, int trim, int m, int n, int g,
                           std::uint32_t threads) {
  auto* res = new PolishResult();
  try {
    const auto t0 = std::chrono::steady_clock::now();
    auto targets = Unflatten(t_words, t_woff, t_lens, nullptr, nullptr, n_targets, "Utg");
    auto sequences = Unflatten(s_words, s_woff, s_lens, s_bq, s_bq_off, n_sequences, "r");
    auto pool = std::make_shared<thread_pool::ThreadPool>(threads ? threads : 1);
    auto polisher = racon::Polisher::Create(pool, q, e, w, trim != 0, static_cast<std::int8_t>(m),
                                            static_cast<std::int8_t>(n),
                                            static_cast<std::int8_t>(g), 0, false, 0);
    auto polished = polisher->Polish(targets, sequences, false);
    res->woff.push_back(0);
    for (const auto& p : polished) {
      res->words.insert(res->words.end(), p->deflated_data.begin(), p->deflated_data.end());
      res->woff.push_back(res->words.size());
      res->lens.push_back(p->inflated_len);
      res->names += p->name + "\n";
    }
    res->stats[0] = static_cast<double>(polisher->num_windows());
    res->stats[1] = static_cast<double>(polisher->num_polished_windows());
    res->stats[2] = polisher->poa_seconds();
    res->stats[3] =
        std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (int i = 0; i < 6; ++i) res->stats[4 + i] = polisher->phase_seconds()[i];
    res->stats[10] = static_cast<double>(polisher->num_wide_windows());
    res->stats[11] = static_cast<double>(polisher->num_window_batches());
  } catch (const std::exception& ex) {
    res->error = ex.what();
    if (res->error.empty()) res->error = "error";
  }
  return res;
}

RVNH_API const char* rvnh_polish_error(void* h) { return static_cast<PolishResult*>(h)->error.c_str(); }
RVNH_API std::uint32_t rvnh_polish_count(void* h) {
  return static_cast<std::uint32_t>(static_cast<PolishResult*>(h)->lens.size());
}
RVNH_API const std::uint64_t* rvnh_polish_words(void* h) { return static_cast<PolishResult*>(h)->words.data(); }
RVNH_API const std::uint64_t* rvnh_polish_word_off(void* h) { return static_cast<PolishResult*>(h)->woff.data(); }
RVNH_API const std::uint32_t* rvnh_polish_lens(void* h) { return static_cast<PolishResult*>(h)->lens.data(); }
RVNH_API const char* rvnh_polish_names(void* h) { return static_cast<PolishResult*>(h)->names.c_str(); }
RVNH_API const double* rvnh_polish_stats(void* h) { return static_cast<PolishResult*>(h)->stats; }
RVNH_API void rvnh_polish_free(void* h) { delete static_cast<PolishResult*>(h); }

}  // extern "C"
