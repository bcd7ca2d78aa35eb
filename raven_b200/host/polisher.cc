// raven_b200 — racon::Polisher facade (include/racon/polisher.hpp).
// Reference contract: RavenLib/src/polish.cc:43-51; behaviour of the stages:
// SURVEY.md App. A.4. GPU: mapping (rvn_minimize/rvn_filter/rvn_map), the global
// alignment paths of the reads (edlibAlign NW PATH) cut at the windows
// (rvn_align_breaking_points), racon's per-layer rules, the window layers and their
// consensus (rvn_polish_windows). Host: best overlap per read, stitching.
#include "racon/polisher.hpp"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

#include "raven_b200.h"

namespace racon {

namespace {

void Check(rvn_ctx* ctx, int rc) {
  if (rc == RVN_OK) return;
  std::string msg = std::string("[racon::Polisher::Polish] error: ") + rvn_last_error(ctx);
  if (rc == RVN_ERR_INVALID) throw std::invalid_argument(msg);
  throw std::runtime_error(msg);
}

// whether RVN_SET_OPTIONS ("name=value,...") sets option `name`
bool EnvNamesOption(const std::string& name) {
  const char* env = std::getenv("RVN_SET_OPTIONS");
  if (!env) return false;
  const std::string all(env);
  for (size_t b = 0; b < all.size();) {
    const size_t e = std::min(all.find(',', b), all.size());
    if (all.compare(b, std::min(all.find('=', b), e) - b, name) == 0) return true;
    b = e + 1;
  }
  return false;
}

struct Hit {  // the overlap kept for one read
  bool valid = false;
  rvn_overlap o{};
};

}  // namespace

Polisher::Polisher(std::shared_ptr<thread_pool::ThreadPool> thread_pool, double q,
                   double e, std::uint32_t w, bool trim, std::int8_t m, std::int8_t n,
                   std::int8_t g)
    : thread_pool_(thread_pool ? thread_pool
                               : std::make_shared<thread_pool::ThreadPool>(1)),
      q_(q), e_(e), w_(w), trim_(trim), m_(m), n_(n), g_(g), ctx_(nullptr) {
  if (rvn_ctx_create(0, nullptr, &ctx_) != RVN_OK) {
    throw std::runtime_error(
        "[racon::Polisher::Create] error: no usable CUDA device (no CPU fallback)");
  }
  // windows of any depth, like racon: the ones past the 16-bit consensus kernels run
  // on the wide kernel. RVN_SET_OPTIONS=poa_wide=... (applied by rvn_ctx_create) wins.
  if (!EnvNamesOption("poa_wide")) Check(ctx_, rvn_set_option(ctx_, "poa_wide", 1));
}

Polisher::~Polisher() {
  if (ctx_) rvn_ctx_destroy(ctx_);
}

std::unique_ptr<Polisher> Polisher::Create(
    std::shared_ptr<thread_pool::ThreadPool> thread_pool, double q, double e,
    std::uint32_t w, bool trim, std::int8_t m, std::int8_t n, std::int8_t g,
    std::uint32_t /*cuda_poa_batches*/, bool /*cuda_banded_alignment*/,
    std::uint32_t /*cuda_alignment_batches*/) {
  if (w == 0) {
    throw std::invalid_argument("[racon::Polisher::Create] error: invalid window length");
  }
  if (g >= 0) {
    throw std::invalid_argument(
        "[racon::Polisher::Create] error: gap penalty must be negative");
  }
  return std::unique_ptr<Polisher>(new Polisher(thread_pool, q, e, w, trim, m, n, g));
}

std::vector<std::unique_ptr<biosoup::NucleicAcid>> Polisher::Polish(
    const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& targets,
    const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences,
    bool drop_unpolished) {
  num_windows_ = num_polished_windows_ = num_wide_windows_ = num_window_batches_ = 0;
  poa_seconds_ = 0;
  if (targets.empty() || sequences.empty()) {
    return {};
  }
  const std::uint32_t T = targets.size(), S = sequences.size();
  auto t_phase = std::chrono::steady_clock::now();
  const auto Seconds = [](std::chrono::steady_clock::time_point& since) {
    const auto now = std::chrono::steady_clock::now();
    const double s = std::chrono::duration<double>(now - since).count();
    since = now;
    return s;
  };

  // ---- 1. GPU: index the targets, map every read (ram k=15 w=5 f=0.001) ----
  // device set = targets (ids 0..T-1) followed by reads (ids T..T+S-1)
  std::vector<std::uint64_t> words, off{0};
  std::vector<std::uint32_t> lens;
  std::uint64_t total_len = 0;
  auto append = [&](const biosoup::NucleicAcid& s) {
    if (s.is_reverse_complement) {
      std::vector<std::uint64_t> w((static_cast<std::uint64_t>(s.inflated_len) + 31) >> 5, 0);
      for (std::uint32_t i = 0; i < s.inflated_len; ++i) w[i >> 5] |= s.Code(i) << ((i << 1) & 63);
      words.insert(words.end(), w.begin(), w.end());
    } else {
      words.insert(words.end(), s.deflated_data.begin(), s.deflated_data.end());
    }
    off.push_back(words.size());
    lens.push_back(s.inflated_len);
  };
  for (const auto& t : targets) append(*t);
  for (const auto& s : sequences) {
    append(*s);
    total_len += s->inflated_len;
  }
  const bool tgs = static_cast<double>(total_len) / S > 1000;
  Check(ctx_, rvn_engine_configure(ctx_, 15, 5, 500, 4, 100, 10000));
  Check(ctx_, rvn_reads_upload(ctx_, words.data(), off.data(), lens.data(), T + S));

  std::vector<Hit> best(S);
  std::uint64_t bytes = 0;
  for (std::uint32_t i = 0, j = 0; i < T; ++i) {
    bytes += targets[i]->inflated_len;
    if (i != T - 1 && bytes < (1ULL << 32)) continue;
    bytes = 0;
    Check(ctx_, rvn_minimize(ctx_, j, i + 1, 0));
    std::uint32_t occ = 0;
    Check(ctx_, rvn_filter(ctx_, 0.001, &occ));
    Check(ctx_, rvn_map(ctx_, T, T + S, 0, 0, 0, 0));
    const rvn_overlap* o = nullptr;
    const std::uint64_t* ooff = nullptr;
    std::uint64_t n = 0;
    Check(ctx_, rvn_map_results(ctx_, &o, &ooff, &n, nullptr, nullptr));
    for (std::uint32_t k = 0; k < S; ++k) {
      for (std::uint64_t x = ooff[k]; x < ooff[k + 1]; ++x) {
        const auto span = [](const rvn_overlap& v) {
          return std::max(v.lhs_end - v.lhs_begin, v.rhs_end - v.rhs_begin);
        };
        if (!best[k].valid || span(best[k].o) < span(o[x])) {
          best[k].o = o[x];
          best[k].valid = true;
        }
      }
    }
    j = i + 1;
  }

  phase_seconds_[0] = Seconds(t_phase);

  // ---- 2. GPU: alignment paths cut at the windows (rvn_align_breaking_points) ----
  std::vector<std::uint64_t> first_window(T + 1ULL, 0);
  for (std::uint32_t i = 0; i < T; ++i) {
    first_window[i + 1] = first_window[i] + (targets[i]->inflated_len + w_ - 1) / w_;
  }
  std::vector<std::uint32_t> coverage(T, 0);
  std::vector<std::uint32_t> a_qread, a_qbegin, a_qlen, a_tread, a_tbegin, a_tlen;
  std::vector<std::uint8_t> a_strand;
  std::vector<std::uint64_t> bp_off{0};
  for (std::uint32_t k = 0; k < S; ++k) {
    if (!best[k].valid) continue;
    const rvn_overlap o = best[k].o;
    const double ql = o.lhs_end - o.lhs_begin, tl = o.rhs_end - o.rhs_begin;
    if (1 - std::min(ql, tl) / std::max(ql, tl) > e_) continue;
    ++coverage[o.rhs_id];
    a_qread.push_back(T + k);
    a_qbegin.push_back(o.lhs_begin);
    a_qlen.push_back(o.lhs_end - o.lhs_begin);
    a_strand.push_back(o.strand ? 1 : 0);
    a_tread.push_back(o.rhs_id);
    a_tbegin.push_back(o.rhs_begin);
    a_tlen.push_back(o.rhs_end - o.rhs_begin);
    const std::uint64_t windows =
        o.rhs_end > o.rhs_begin ? (o.rhs_end - 1) / w_ - o.rhs_begin / w_ + 1 : 0;
    bp_off.push_back(bp_off.back() + windows);
  }
  const std::size_t A = a_qread.size();
  std::vector<std::int32_t> a_dist(A);
  std::vector<std::uint32_t> bp(4 * bp_off.back() + 4);
  // (batches of about 2^29 query bases bound the device scratch of the alignment:
  //  score columns, match masks and stored leaf columns grow with the bases in flight)
  std::uint64_t batch_bases = 1ULL << 29;
  if (const char* env = std::getenv("RVN_POLISH_BATCH_BASES")) {  // (tests: several batches)
    batch_bases = std::max<std::uint64_t>(1, std::strtoull(env, nullptr, 10));
  }
  for (std::size_t a0 = 0; a0 < A;) {
    std::size_t a1 = a0;
    std::uint64_t bases = 0;
    while (a1 < A && (a1 == a0 || bases + a_qlen[a1] <= batch_bases)) bases += a_qlen[a1++];
    std::vector<std::uint64_t> off(bp_off.begin() + a0, bp_off.begin() + a1 + 1);
    for (auto& x : off) x -= bp_off[a0];
    Check(ctx_, rvn_align_breaking_points(
                    ctx_, a1 - a0, a_qread.data() + a0, a_qbegin.data() + a0, a_qlen.data() + a0,
                    a_strand.data() + a0, a_tread.data() + a0, a_tbegin.data() + a0,
                    a_tlen.data() + a0, w_, off.data(), a_dist.data() + a0,
                    bp.data() + 4 * bp_off[a0]));
    a0 = a1;
  }
  phase_seconds_[1] = Seconds(t_phase);

  // ---- 3. GPU: racon's layer rules, the layers of every window and their consensus,
  //         in batches of windows (rvn_polish_windows) ----
  std::vector<std::uint8_t> bq, rc(T + S, 0);
  std::vector<std::uint64_t> bq_off(T + S + 1ULL, 0);
  for (std::uint32_t i = 0; i < T + S; ++i) {
    const auto& s = i < T ? *targets[i] : *sequences[i - T];
    rc[i] = s.is_reverse_complement ? 1 : 0;
    if (i >= T) bq.insert(bq.end(), s.block_quality.begin(), s.block_quality.end());
    bq_off[i + 1] = bq.size();
  }
  const auto t0 = std::chrono::steady_clock::now();
  std::uint32_t batches = 0;
  Check(ctx_, rvn_polish_windows(ctx_, A, a_qread.data(), a_qbegin.data(), a_qlen.data(),
                                 a_strand.data(), a_tread.data(), bp_off.data(), bp.data(), T, w_,
                                 bq.empty() ? nullptr : bq.data(), bq_off.data(), rc.data(), q_,
                                 m_, n_, g_, trim_, tgs, &batches));
  const char* cons = nullptr;
  const std::uint64_t* cons_off = nullptr;
  const std::uint8_t* status = nullptr;
  Check(ctx_, rvn_poa_results(ctx_, &cons, &cons_off, &status, nullptr, nullptr));
  std::uint32_t routes[3] = {0, 0, 0};
  Check(ctx_, rvn_poa_routes(ctx_, routes, nullptr));
  num_wide_windows_ = routes[2];
  num_window_batches_ = batches;
  poa_seconds_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  // the device time of the layer rules and of the packing (rvn_get_timings)
  double layers_s = 0, pack_s = 0;
  const char* const* names = nullptr;
  const float* ms = nullptr;
  std::uint32_t n_phases = 0;
  Check(ctx_, rvn_get_timings(ctx_, &names, &ms, &n_phases));
  for (std::uint32_t i = 0; i < n_phases; ++i) {
    if (std::strcmp(names[i], "poa_layers") == 0) layers_s += ms[i] / 1000;
    if (std::strcmp(names[i], "poa_pack") == 0) pack_s += ms[i] / 1000;
  }
  const double consensus_s = Seconds(t_phase);
  phase_seconds_[5] = layers_s;
  phase_seconds_[2] = pack_s;
  phase_seconds_[3] = std::max(0.0, consensus_s - layers_s - pack_s);

  // ---- 4. stitch ----
  std::vector<std::unique_ptr<biosoup::NucleicAcid>> dst;
  for (std::uint32_t i = 0; i < T; ++i) {
    const std::uint64_t w0 = first_window[i], w1 = first_window[i + 1];
    std::string polished(cons + cons_off[w0], cons + cons_off[w1]);
    std::uint32_t n_polished = 0;
    for (std::uint64_t w = w0; w < w1; ++w) n_polished += status[w] & 1;
    num_windows_ += w1 - w0;
    num_polished_windows_ += n_polished;
    const double ratio = w1 > w0 ? n_polished / static_cast<double>(w1 - w0) : 0;
    if (!drop_unpolished || ratio > 0) {
      std::string tags = " LN:i:" + std::to_string(polished.size());
      tags += " RC:i:" + std::to_string(coverage[i]);
      tags += " XC:f:" + std::to_string(ratio);
      dst.emplace_back(new biosoup::NucleicAcid(targets[i]->name + tags, polished));
    }
  }
  phase_seconds_[4] = Seconds(t_phase);
  return dst;
}

}  // namespace racon
