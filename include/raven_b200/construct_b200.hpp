// raven-b200: GPU replacement of raven::FindOverlapsAndCreatePiles
// (RavenLib/src/construct.cc:14-121) with the reference's exact signature
// (RavenLib/include/raven/graph/construct.h:22-29). One call = the whole stage
// on the device (sketch, index, filter, map/chain, piles, gather, truncation);
// the results are written back into RavenLib's own containers.
//
// Needs RavenLib's headers ("raven/pile.h") on the include path: it is meant to
// be compiled inside RavenLib (INTEGRATION.md), replacing the body of
// construct.cc:14-121 with a call to raven_b200::FindOverlapsAndCreatePiles.
#ifndef RAVEN_B200_CONSTRUCT_B200_HPP_
#define RAVEN_B200_CONSTRUCT_B200_HPP_

#include <algorithm>
#include <cstdint>
#include <iostream>
#include <future>
#include <memory>
#include <stdexcept>
#include <vector>

#include "biosoup/nucleic_acid.hpp"
#include "biosoup/overlap.hpp"
#include "biosoup/timer.hpp"
#include "cereal/access.hpp"
#include "ram/minimizer_engine.hpp"
#include "raven/graph/overlap_utils.h"
#include "raven/pile.h"
#include "raven_b200.h"
#include "raven_b200/load_sequences.hpp"  // raven_b200::LoadSequences
#include "raven_b200/overlap_clip.hpp"
#include "thread_pool/thread_pool.hpp"

namespace raven_b200 {

namespace detail {

// raven::Pile keeps its histogram private and only lets AddLayers touch it;
// the one door it leaves open is `friend cereal::access` + serialize(), which
// hands out references to every field. This "archive" uses it to move the
// device-computed histogram in.
struct PileDoor {
  const std::uint16_t* src;
  std::size_t n;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t&, std::uint32_t&, std::uint16_t&,
                  bool&, bool&, bool&, bool&, std::vector<std::uint16_t>& data,
                  Ts&...) {
    if (data.size() != n) {
      throw std::logic_error("[raven_b200] pile size mismatch");
    }
    data.assign(src, src + n);
  }
};

}  // namespace detail

inline void FindOverlapsAndCreatePiles(
    const std::shared_ptr<thread_pool::ThreadPool>& /*thread_pool*/,
    ram::MinimizerEngine& minimizer_engine,
    const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences,
    double freq, std::vector<std::unique_ptr<raven::Pile>>& piles,
    std::vector<std::vector<biosoup::Overlap>>& overlaps,
    std::size_t kMaxNumOverlaps = 32, bool useMinhash = false) {
  piles.reserve(sequences.size());
  for (const auto& it : sequences) {
    piles.emplace_back(new raven::Pile(it->id, it->inflated_len));
  }
  if (overlaps.size() < sequences.size()) overlaps.resize(sequences.size());

  biosoup::Timer timer;
  timer.Start();
  minimizer_engine.Upload(sequences);  // ids must equal positions (they do in raven)
  std::lock_guard<std::mutex> lock(minimizer_engine.mutex());
  rvn_ctx* ctx = minimizer_engine.context();
  int rc = rvn_find_overlaps_and_create_piles(ctx, freq, kMaxNumOverlaps,
                                              useMinhash, 0, 0);
  if (rc == RVN_ERR_INVALID) throw std::invalid_argument(rvn_last_error(ctx));
  if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));

  const rvn_overlap* o = nullptr;
  const std::uint64_t *ooff = nullptr, *poff = nullptr;
  const std::uint16_t* pile = nullptr;
  std::uint64_t n_mapped = 0;
  rc = rvn_stage1_results(ctx, &o, &ooff, &pile, &poff, &n_mapped);
  if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));

  for (std::size_t i = 0; i < sequences.size(); ++i) {
    auto& dst = overlaps[i];
    for (std::uint64_t e = ooff[i]; e < ooff[i + 1]; ++e) {
      dst.emplace_back(o[e].lhs_id, o[e].lhs_begin, o[e].lhs_end, o[e].rhs_id,
                       o[e].rhs_begin, o[e].rhs_end, o[e].score, o[e].strand != 0);
    }
    detail::PileDoor door{pile + poff[i], static_cast<std::size_t>(poff[i + 1] - poff[i])};
    auto visit = cereal::fields(door);
    cereal::access::member_serialize(visit, *piles[i]);
  }
  std::cerr << "[raven::Graph::Construct] minimized + mapped sequences (GPU) "
            << std::fixed << timer.Stop() << "s" << std::endl;
}

namespace detail {

// the result of Pile::FindValidRegion + FindMedian into a pile, the way
// UpdateValidRegion (pile.cc:144-157) and FindMedian (pile.cc:168-172) leave it
struct PileTrimDoor {
  std::uint32_t begin, end;
  std::uint16_t median;
  bool invalid;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t& b, std::uint32_t& e, std::uint16_t& m,
                  bool& is_invalid, bool&, bool&, bool&, std::vector<std::uint16_t>& data,
                  Ts&...) {
    if (invalid) {
      is_invalid = true;
      return;
    }
    for (std::uint32_t i = b; i < begin; ++i) data[i] = 0;
    for (std::uint32_t i = end; i < e; ++i) data[i] = 0;
    b = begin;
    e = end;
    m = median;
  }
};

}  // namespace detail

// raven::TrimAndAnnotatePiles (construct.cc:123-152) right after
// raven_b200::FindOverlapsAndCreatePiles: the valid regions and medians of ALL piles come
// from the histograms that call left on the device (rvn_stage1_pile_regions); the host
// pool applies them and runs the reference's own FindChimericRegions.
inline void TrimAndAnnotatePiles(
    const std::shared_ptr<thread_pool::ThreadPool>& thread_pool,
    const std::vector<std::unique_ptr<raven::Pile>>& piles,
    std::vector<std::vector<biosoup::Overlap>>& overlaps,
    ram::MinimizerEngine& minimizer_engine) {
  biosoup::Timer timer;
  timer.Start();
  const std::size_t n = piles.size();
  std::vector<std::uint32_t> begin(n), end(n);
  std::vector<std::uint16_t> median(n);
  std::vector<std::uint8_t> invalid(n);
  {
    std::lock_guard<std::mutex> lock(minimizer_engine.mutex());
    rvn_ctx* ctx = minimizer_engine.context();
    const int rc = rvn_stage1_pile_regions(ctx, 4, begin.data(), end.data(), median.data(),
                                           invalid.data());
    if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));
  }
  std::vector<std::future<void>> futures;
  const std::size_t chunk = std::max<std::size_t>(64, n / 1024 + 1);
  for (std::size_t i0 = 0; i0 < n; i0 += chunk) {
    futures.emplace_back(thread_pool->Submit(
        [&](std::size_t i0, std::size_t i1) {
          for (std::size_t i = i0; i < i1; ++i) {
            detail::PileTrimDoor door{begin[i], end[i], median[i], invalid[i] != 0};
            auto visit = cereal::fields(door);
            cereal::access::member_serialize(visit, *piles[i]);
            if (piles[i]->is_invalid()) {
              std::vector<biosoup::Overlap>().swap(overlaps[i]);
            } else {
              piles[i]->FindChimericRegions();
            }
          }
        },
        i0, std::min(n, i0 + chunk)));
  }
  for (auto& f : futures) f.wait();
  std::cerr << "[raven::Graph::Construct] annotated piles (GPU) " << std::fixed
            << timer.Stop() << "s" << std::endl;
}

namespace detail {

// keep[i] = 1 iff overlap i passes the identity filter; the reads are addressed
// through index_of(id) = position in the set uploaded to the engine
template <typename IndexOf>
std::vector<char> IdentityFilter(ram::MinimizerEngine& engine,
                                 const std::vector<biosoup::Overlap>& ovl, double identity,
                                 IndexOf index_of) {
  const std::size_t n = ovl.size();
  std::vector<char> keep(n, 0);
  if (n == 0) return keep;
  std::vector<std::uint32_t> lr(n), lb(n), ll(n), rr(n), rb(n), rl(n);
  std::vector<std::uint8_t> st(n);
  std::vector<std::int32_t> limit(n), dist(n);
  for (std::size_t i = 0; i < n; ++i) {
    const auto& o = ovl[i];
    lr[i] = index_of(o.lhs_id);
    lb[i] = o.lhs_begin;
    ll[i] = o.lhs_end - o.lhs_begin;
    rr[i] = index_of(o.rhs_id);
    rb[i] = o.rhs_begin;
    rl[i] = o.rhs_end - o.rhs_begin;
    st[i] = o.strand ? 1 : 0;
    limit[i] = rvn::IdentityBound(identity, std::max(ll[i], rl[i]));
    if (limit[i] < 0) limit[i] = 0;  // (decided below; the search stays bounded)
  }
  std::lock_guard<std::mutex> lock(engine.mutex());
  rvn_ctx* ctx = engine.context();
  const int rc = rvn_edit_distance_batch(ctx, n, lr.data(), lb.data(), ll.data(), rr.data(),
                                         rb.data(), rl.data(), st.data(), limit.data(),
                                         dist.data());
  if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));
  for (std::size_t i = 0; i < n; ++i) {
    if (dist[i] < 0) continue;  // beyond the bound: score < identity
    const double score =
        1. - static_cast<double>(dist[i]) / std::max<std::size_t>(ll[i], rl[i]);
    keep[i] = !(score < identity);
  }
  return keep;
}

}  // namespace detail

// raven::ResolveContainedReads (RavenLib/src/construct.cc:154-246) with the
// identity filter (edlibAlign per overlap, :165-210) as ONE batched device call.
// Same arguments plus the engine that still holds the read set of stage 1
// (ids == positions). With identity == 0 it is the reference's own function.
inline void ResolveContainedReads(
    const std::vector<std::unique_ptr<raven::Pile>>& piles,
    std::vector<std::vector<biosoup::Overlap>>& overlaps,
    const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences,
    const std::shared_ptr<thread_pool::ThreadPool>& thread_pool, double identity,
    ram::MinimizerEngine& engine) {
  if (identity != 0) {
    biosoup::Timer timer;
    timer.Start();
    engine.Upload(sequences);  // (a no-op for the device if stage 1 just ran: same set)
    std::vector<biosoup::Overlap> flat;
    std::vector<std::pair<std::uint32_t, std::uint32_t>> where;  // (list, slot)
    for (std::uint32_t i = 0; i < overlaps.size(); ++i) {
      for (std::uint32_t j = 0; j < overlaps[i].size(); ++j) {
        if (!raven::OverlapUpdate(overlaps[i][j], piles)) continue;  // :170-172
        flat.emplace_back(overlaps[i][j]);
        where.emplace_back(i, j);
      }
    }
    const auto keep =
        detail::IdentityFilter(engine, flat, identity, [](std::uint32_t id) { return id; });
    std::vector<std::vector<char>> mark(overlaps.size());
    for (std::uint32_t i = 0; i < overlaps.size(); ++i) mark[i].assign(overlaps[i].size(), 0);
    for (std::size_t x = 0; x < flat.size(); ++x) mark[where[x].first][where[x].second] = keep[x];
    for (std::uint32_t i = 0; i < overlaps.size(); ++i) {
      std::uint32_t k = 0;
      for (std::uint32_t j = 0; j < overlaps[i].size(); ++j) {
        if (mark[i][j]) overlaps[i][k++] = overlaps[i][j];
      }
      overlaps[i].resize(k);
    }
    std::cerr << "[raven::Graph::Construct] filtered overlaps (GPU) " << std::fixed
              << timer.Stop() << "s" << std::endl;
  }
  // the containment part is host logic on piles: the reference's own code
  raven::ResolveContainedReads(piles, overlaps, sequences, thread_pool, 0);
}

namespace detail {

// Pile::AddKmers' result moved into a pile through the same door as PileDoor: kmers_
// takes the device's bits, resized as the reference resizes it (pile.cc:67-72), so a
// touched pile whose k-mers all fail the complexity test keeps an all-zero kmers_.
struct KmerDoor {
  const std::uint32_t* bits;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t&, std::uint32_t&, std::uint16_t&, bool&, bool&,
                  bool&, bool&, std::vector<std::uint16_t>& data, std::vector<bool>& kmers,
                  Ts&...) {
    if (kmers.empty()) kmers.resize(data.size() + 1, false);
    for (std::size_t b = 0; b < data.size() + 1; ++b) {
      if (bits[b >> 5] >> (b & 31) & 1u) kmers[b] = true;
    }
  }
};

}  // namespace detail

// raven::FindOverlapsAndRepetetiveRegions (RavenLib/src/construct.cc:316-491)
// with the reference's exact signature: the map of every batch, Pile::AddKmers and the
// identity filter are ONE device call (rvn_find_overlaps_and_repetitive_regions) over
// the valid reads; the k-mer marks move into the piles, and the classification loop
// (OverlapUpdate / GetOverlapType / longest per pair, :430-455) is the reference's, on
// the host. The k-mers are the engine's k long: the reference's only caller passes that
// k as kmer_len (construct.cc:661-688).
inline void FindOverlapsAndRepetetiveRegions(
    const std::shared_ptr<thread_pool::ThreadPool>& /*thread_pool*/,
    ram::MinimizerEngine& engine, double freq, std::uint8_t /*kmer_len*/, double identity,
    const std::vector<std::unique_ptr<raven::Pile>>& piles,
    std::vector<std::vector<biosoup::Overlap>>& overlaps,
    std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences) {
  biosoup::Timer timer;
  timer.Start();
  std::sort(sequences.begin(), sequences.end(),
            [&](const std::unique_ptr<biosoup::NucleicAcid>& lhs,
                const std::unique_ptr<biosoup::NucleicAcid>& rhs) -> bool {
              return piles[lhs->id]->is_invalid() < piles[rhs->id]->is_invalid() ||
                     (piles[lhs->id]->is_invalid() == piles[rhs->id]->is_invalid() &&
                      lhs->id < rhs->id);
            });
  std::uint32_t s = 0;  // (stays 0 when no read is invalid: construct.cc:343-349)
  for (std::uint32_t i = 0; i < sequences.size(); ++i) {
    if (piles[sequences[i]->id]->is_invalid()) {
      s = i;
      break;
    }
  }
  overlaps.resize(sequences.size() + 1);
  if (s > 0) {
    engine.Upload(sequences.begin(), sequences.begin() + s);
    std::vector<std::uint32_t> begin(s), end(s);
    for (std::uint32_t i = 0; i < s; ++i) {
      begin[i] = piles[sequences[i]->id]->begin();
      end[i] = piles[sequences[i]->id]->end();
    }
    std::vector<biosoup::Overlap> mapped;  // final results of all batches, in loop order
    {
      std::lock_guard<std::mutex> lock(engine.mutex());
      rvn_ctx* ctx = engine.context();
      auto check = [&](int rc) {
        if (rc == RVN_ERR_INVALID) throw std::invalid_argument(rvn_last_error(ctx));
        if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));
      };
      check(rvn_find_overlaps_and_repetitive_regions(ctx, freq, identity, s, begin.data(),
                                                     end.data()));
      const rvn_overlap* o = nullptr;
      const std::uint64_t *ooff = nullptr, *koff = nullptr;
      const std::uint32_t* bits = nullptr;
      const std::uint8_t* touched = nullptr;
      std::uint64_t n_mapped = 0;
      check(rvn_stage2_results(ctx, &o, &ooff, &bits, &koff, &touched, &n_mapped));
      for (std::uint32_t i = 0; i < s; ++i) {  // :382-383
        if (!touched[i]) continue;
        detail::KmerDoor door{bits + koff[i]};
        auto visit = cereal::fields(door);
        cereal::access::member_serialize(visit, *piles[sequences[i]->id]);
      }
      mapped.reserve(ooff[s]);
      for (std::uint64_t e = 0; e < ooff[s]; ++e) {
        mapped.emplace_back(o[e].lhs_id, o[e].lhs_begin, o[e].lhs_end, o[e].rhs_id,
                            o[e].rhs_begin, o[e].rhs_end, o[e].score, o[e].strand != 0);
      }
    }
    std::cerr << "[raven::Graph::Construct] minimized + mapped valid sequences (GPU) " << s
              << " " << std::fixed << timer.Stop() << "s" << std::endl;
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

}  // namespace raven_b200

#endif  // RAVEN_B200_CONSTRUCT_B200_HPP_
