// Stage 2's fast route timed against the route it replaced: the same read set through
// stage 1, the pile annotation, containment and chimeric removal (GPU routes and the
// reference's host code), then either raven_b200::FindOverlapsAndRepetetiveRegions (one
// device call) or PreviousRoute (the former body of that function: rvn_minimize,
// rvn_filter and rvn_map per batch, Pile::AddKmers serially on the host, the identity
// filter through rvn_edit_distance_batch), alternating. Only stage 2 is timed. Prints
// one JSON line per run: route, seconds, filtered positions (previous route), and a
// digest of the end state (every overlap list and every pile's cereal JSON).
//   usage: stage2_time <reads.bin> <k> <w> <freq> <identity> <reps>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <fstream>
#include <functional>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "cereal/archives/json.hpp"
#include "raven/graph/construct.h"
#include "raven/graph/serialization/binary.h"
#include "raven/pile.h"
#include "raven_b200/construct_b200.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace raven {
void StoreGraphToFile(const Graph&) { throw std::logic_error("no checkpoints here"); }
}  // namespace raven

namespace {

std::uint64_t g_filtered = 0;  // filtered positions the previous route handed to AddKmers

void PreviousRoute(
    const std::shared_ptr<thread_pool::ThreadPool>& /*thread_pool*/,
    ram::MinimizerEngine& engine, double freq, std::uint8_t kmer_len, double identity,
    const std::vector<std::unique_ptr<raven::Pile>>& piles,
    std::vector<std::vector<biosoup::Overlap>>& overlaps,
    std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences) {
  biosoup::Timer timer;
  std::sort(sequences.begin(), sequences.end(),
            [&](const std::unique_ptr<biosoup::NucleicAcid>& lhs,
                const std::unique_ptr<biosoup::NucleicAcid>& rhs) -> bool {
              return piles[lhs->id]->is_invalid() < piles[rhs->id]->is_invalid() ||
                     (piles[lhs->id]->is_invalid() == piles[rhs->id]->is_invalid() &&
                      lhs->id < rhs->id);
            });
  // id -> position in the sorted vector (= position in the uploaded set)
  std::uint32_t max_id = 0;
  for (const auto& it : sequences) max_id = std::max(max_id, it->id);
  std::vector<std::uint32_t> sequences_map(static_cast<std::size_t>(max_id) + 1, 0);
  for (std::uint32_t i = 0; i < sequences.size(); ++i) sequences_map[sequences[i]->id] = i;

  std::uint32_t s = 0;  // (stays 0 when no read is invalid: construct.cc:343-349)
  for (std::uint32_t i = 0; i < sequences.size(); ++i) {
    if (piles[sequences[i]->id]->is_invalid()) {
      s = i;
      break;
    }
  }

  overlaps.resize(sequences.size() + 1);
  if (s > 0) engine.Upload(sequences.begin(), sequences.begin() + s);
  rvn_ctx* ctx = engine.context();
  auto check = [&](int rc) {
    if (rc == RVN_ERR_INVALID) throw std::invalid_argument(rvn_last_error(ctx));
    if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));
  };
  std::size_t bytes = 0;
  for (std::uint32_t i = 0, j = 0; i < s; ++i) {
    bytes += sequences[i]->inflated_len;
    if (i != s - 1 && bytes < (1U << 30)) continue;
    bytes = 0;
    timer.Start();
    std::vector<biosoup::Overlap> mapped;  // all Map results of the batch, query order
    {
      std::lock_guard<std::mutex> lock(engine.mutex());
      check(rvn_minimize(ctx, j, i + 1, 0));
      std::uint32_t occ = 0;
      check(rvn_filter(ctx, freq, &occ));
      check(rvn_map(ctx, 0, i + 1, 1, 1, 0, 1));
      const rvn_overlap* o = nullptr;
      const std::uint64_t *off = nullptr, *foff = nullptr;
      const std::uint32_t* f = nullptr;
      std::uint64_t n = 0;
      check(rvn_map_results(ctx, &o, &off, &n, &f, &foff));
      mapped.reserve(n);
      for (std::uint32_t k = 0; k < i + 1; ++k) {
        const std::vector<std::uint32_t> filtered(f + foff[k], f + foff[k + 1]);
        g_filtered += filtered.size();
        piles[sequences[k]->id]->AddKmers(filtered, kmer_len, sequences[k]);  // :382-383
        for (std::uint64_t e = off[k]; e < off[k + 1]; ++e) {
          mapped.emplace_back(o[e].lhs_id, o[e].lhs_begin, o[e].lhs_end, o[e].rhs_id,
                              o[e].rhs_begin, o[e].rhs_end, o[e].score, o[e].strand != 0);
        }
      }
    }
    if (identity != 0) {  // :385-424, batched
      std::vector<biosoup::Overlap> upd;
      for (auto& o : mapped) {
        if (raven::OverlapUpdate(o, piles)) upd.emplace_back(o);
      }
      const auto keep = raven_b200::detail::IdentityFilter(
          engine, upd, identity, [&](std::uint32_t id) { return sequences_map[id]; });
      mapped.clear();
      for (std::size_t x = 0; x < upd.size(); ++x) {
        if (keep[x]) mapped.emplace_back(upd[x]);
      }
    }
    std::cerr << "[raven::Graph::Construct] minimized + mapped valid sequences (GPU) " << j
              << " - " << i + 1 << " / " << s << " " << std::fixed << timer.Stop() << "s"
              << std::endl;
    for (auto& jt : mapped) {  // :430-455
      if (!raven::OverlapUpdate(jt, piles)) continue;
      const std::uint32_t type = raven::GetOverlapType(jt, piles);
      if (type == 0) {
        continue;
      } else if (type == 1) {
        piles[jt.lhs_id]->set_is_contained();
      } else if (type == 2) {
        piles[jt.rhs_id]->set_is_contained();
      } else {
        if (!overlaps.back().empty() && overlaps.back().back().lhs_id == jt.lhs_id &&
            overlaps.back().back().rhs_id == jt.rhs_id) {
          if (raven::GetOverlapLength(overlaps.back().back()) < raven::GetOverlapLength(jt)) {
            overlaps.back().back() = jt;
          }
        } else {
          overlaps.back().emplace_back(jt);
        }
      }
    }
    j = i + 1;
  }

  for (const auto& pile : piles) {  // :465-469
    if (pile->is_contained()) pile->set_is_invalid();
  }
  {
    std::uint32_t k = 0;
    for (std::uint32_t i = 0; i < overlaps.back().size(); ++i) {
      if (raven::OverlapUpdate(overlaps.back()[i], piles)) overlaps.back()[k++] = overlaps.back()[i];
    }
    overlaps.back().resize(k);
  }
  std::sort(sequences.begin(), sequences.end(),
            [&](const std::unique_ptr<biosoup::NucleicAcid>& lhs,
                const std::unique_ptr<biosoup::NucleicAcid>& rhs) -> bool {
              return lhs->id < rhs->id;
            });
}


template <typename T>
std::vector<T> ReadVec(std::ifstream& f) {
  std::uint64_t n = 0;
  f.read(reinterpret_cast<char*>(&n), 8);
  std::vector<T> v(n);
  f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
  return v;
}

std::uint64_t Fnv(const std::string& s, std::uint64_t h = 1469598103934665603ULL) {
  for (unsigned char c : s) h = (h ^ c) * 1099511628211ULL;
  return h;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 7) {
    std::cerr << "usage: stage2_time reads.bin k w freq identity reps\n";
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const auto words = ReadVec<std::uint64_t>(in);
  const auto woff = ReadVec<std::uint64_t>(in);
  const auto lens = ReadVec<std::uint32_t>(in);
  const std::uint32_t k = std::stoul(argv[2]), w = std::stoul(argv[3]);
  const double freq = std::stod(argv[4]), identity = std::stod(argv[5]);
  const int reps = std::stoi(argv[6]);
  auto pool = std::make_shared<thread_pool::ThreadPool>(8);
  ram::MinimizerEngine engine{pool, k, w};
  try {
    for (int run = 0; run < 2 * reps; ++run) {
      const bool fresh = run % 2 == 1;  // previous, new, previous, new, ...
      std::vector<std::unique_ptr<biosoup::NucleicAcid>> seqs;
      for (std::size_t i = 0; i < lens.size(); ++i) {
        auto s = std::make_unique<biosoup::NucleicAcid>();
        s->id = i;
        s->name = std::to_string(i);
        s->deflated_data.assign(words.begin() + woff[i], words.begin() + woff[i + 1]);
        s->inflated_len = lens[i];
        seqs.emplace_back(std::move(s));
      }
      std::vector<std::unique_ptr<raven::Pile>> piles;
      std::vector<std::vector<biosoup::Overlap>> overlaps(seqs.size());
      raven_b200::FindOverlapsAndCreatePiles(pool, engine, seqs, freq, piles, overlaps, 32, false);
      raven_b200::TrimAndAnnotatePiles(pool, piles, overlaps, engine);
      raven_b200::ResolveContainedReads(piles, overlaps, seqs, pool, identity, engine);
      raven::ResolveChimericSequences(pool, piles, overlaps, seqs);
      g_filtered = 0;
      const auto t0 = std::chrono::steady_clock::now();
      if (fresh) {
        raven_b200::FindOverlapsAndRepetetiveRegions(pool, engine, freq, k, identity, piles,
                                                     overlaps, seqs);
      } else {
        PreviousRoute(pool, engine, freq, k, identity, piles, overlaps, seqs);
      }
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      std::ostringstream st;
      for (const auto& list : overlaps) {
        for (const auto& o : list) {
          st << o.lhs_id << ' ' << o.lhs_begin << ' ' << o.lhs_end << ' ' << o.rhs_id << ' '
             << o.rhs_begin << ' ' << o.rhs_end << ' ' << o.score << ' ' << o.strand << ';';
        }
        st << '|';
      }
      {
        cereal::JSONOutputArchive ar(st);
        for (const auto& p : piles) ar(cereal::make_nvp(std::to_string(p->id()), *p));
      }
      std::uint64_t valid = 0;
      for (const auto& p : piles) valid += !p->is_invalid();
      std::cout << "{\"route\": \"" << (fresh ? "one_call" : "previous") << "\", \"seconds\": "
                << sec << ", \"filtered_positions\": " << g_filtered
                << ", \"final_overlaps\": " << overlaps.back().size()
                << ", \"valid_piles_after\": " << valid << ", \"digest\": \"" << std::hex
                << Fnv(st.str()) << std::dec << "\"}" << std::endl;
    }
  } catch (const std::exception& e) {
    std::cerr << "stage2_time: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}
