// ORACLE — TEST INFRASTRUCTURE ONLY.
// extern "C" surface of oracle/_ref/libraven_ref_stage2.so: the reference's own
// raven::FindOverlapsAndRepetetiveRegions (RavenLib/src/construct.cc and the sources it
// needs, compiled in place from /root/reference by oracle/Makefile) over fresh piles
// whose valid regions and invalid flags the caller gives, on the oracle restatement of
// ram (oracle/ram/) and the oracle's edlib port. tests/stage2_edges.py compares its CPU
// restatement and the device call (rvn_find_overlaps_and_repetitive_regions) with it.
// A library of its own, so that a prebuilt oracle/_ref/libraven_ref.so of an older tree
// can never stand in for it.
#include <atomic>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <vector>

#include "flat_api.hpp"
#include "ram/minimizer_engine.hpp"
#include "raven/graph/construct.h"
#include "raven/graph/serialization/binary.h"
#include "raven/pile.h"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace raven {
// construct.cc only reaches this with checkpoints = true, which stage 2 never passes
void StoreGraphToFile(const Graph&) {
  throw std::logic_error("checkpoints are not part of the pinned path");
}
}  // namespace raven

namespace {

// Pile keeps its fields private; the only door the reference leaves open is
// `friend cereal::access` + serialize(). These archives set and capture fields.
struct PileRegionSetter {  // a given valid region (in bins) and invalid flag
  std::uint32_t begin, end;
  bool invalid;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t& b, std::uint32_t& e, std::uint16_t&,
                  bool& inv, Ts&...) {
    b = begin;
    e = end;
    inv = invalid;
  }
};

struct PileStage2Probe {  // kmers_ and is_contained_
  std::vector<bool> kmers;
  bool contained = false;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t&, std::uint32_t&, std::uint16_t&, bool&,
                  bool& cont, bool&, bool&, std::vector<std::uint16_t>&,
                  std::vector<bool>& k, Ts&...) {
    kmers = k;
    contained = cont;
  }
};

}  // namespace

ORC_BAG_ACCESSORS(refs2)

// raven::FindOverlapsAndRepetetiveRegions (construct.cc:316-491) over fresh piles whose
// valid regions ([rbeg, rend) in bins) and invalid flags are given: the sorted valid ids
// and s (its first invalid position, 0 when every read is valid), the final
// overlaps.back(), and per pile kmers_ (flat, kmer_off), whether kmers_ was resized
// (touched) and is_contained_.
ORC_EXPORT orc_bag* ref_stage2(orc_reads* r, std::uint32_t k, std::uint32_t w, double freq,
                               double identity, std::uint32_t threads, const std::uint32_t* rbeg,
                               const std::uint32_t* rend, const std::uint8_t* invalid) {
  const std::uint32_t n = static_cast<std::uint32_t>(r->seqs.size());
  std::vector<std::unique_ptr<raven::Pile>> piles;
  for (std::uint32_t i = 0; i < n; ++i) {
    piles.emplace_back(new raven::Pile(r->seqs[i]->id, r->seqs[i]->inflated_len));
    PileRegionSetter set{rbeg[i], rend[i], invalid[i] != 0};
    auto put = cereal::fields(set);
    cereal::access::member_serialize(put, *piles.back());
  }
  // the call sorts the valid reads first, by id, and maps the first s of them
  std::vector<std::uint32_t> valid;
  for (std::uint32_t i = 0; i < n; ++i) {
    if (!invalid[i]) valid.push_back(i);
  }
  const std::uint32_t s = valid.size() < n ? static_cast<std::uint32_t>(valid.size()) : 0;
  valid.resize(s);

  auto pool = std::make_shared<thread_pool::ThreadPool>(threads ? threads : 1);
  ram::MinimizerEngine engine{pool, k, w};
  std::vector<std::vector<biosoup::Overlap>> overlaps(n);
  raven::FindOverlapsAndRepetetiveRegions(pool, engine, freq, static_cast<std::uint8_t>(k),
                                          identity, piles, overlaps, r->seqs);

  auto* bag = new orc_bag();
  std::vector<std::uint32_t> ovl;
  for (const auto& o : overlaps.back()) PushOverlap(ovl, o);
  std::vector<std::uint8_t> kmers, touched, contained;
  std::vector<std::uint64_t> kmer_off{0};
  for (const auto& p : piles) {
    PileStage2Probe probe;
    auto get = cereal::fields(probe);
    cereal::access::member_serialize(get, *p);
    kmers.insert(kmers.end(), probe.kmers.begin(), probe.kmers.end());
    kmer_off.emplace_back(kmers.size());
    touched.emplace_back(probe.kmers.empty() ? 0 : 1);
    contained.emplace_back(probe.contained ? 1 : 0);
  }
  std::vector<std::uint32_t> sv{s};
  bag->Put("valid", valid);
  bag->Put("s", sv);
  bag->Put("overlaps", ovl);
  bag->Put("kmers", kmers);
  bag->Put("kmer_off", kmer_off);
  bag->Put("touched", touched);
  bag->Put("contained", contained);
  return bag;
}
