// The reference's OWN overlap stages (RavenLib construct.cc, compiled in place)
// over the ram::MinimizerEngine facade, with the Map counters of each stage:
// raven::FindOverlapsAndCreatePiles, then raven::FindOverlapsAndRepetetiveRegions
// after the reference's pile annotation and read resolution. The same stage 2
// also runs through the batched replacements (raven_b200::*), from their own
// stage 1, so tests/test_gpu_facade_batch.py can compare the two end states.
// Built into oracle/_ref by oracle/facade_batch.mk.
//   usage: facade_batch_test <reads.bin> <out.bin> <k> <w> <freq> <minhash> <threads>
// Output: stage 1 (overlaps, offsets, piles, pile offsets, counters), stage 2
// over the facade (overlaps, offsets, pile fields, order, counters, valid reads
// mapped), stage 2 of the replacements (overlaps, offsets, pile fields, order).
#include <atomic>
#include <cstdint>
#include <fstream>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "raven/graph/construct.h"
#include "raven/graph/serialization/binary.h"
#include "raven/pile.h"
#include "raven_b200/construct_b200.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace raven {
void StoreGraphToFile(const Graph&) { throw std::logic_error("no checkpoints here"); }
}  // namespace raven

namespace {

using Region = std::pair<std::uint32_t, std::uint32_t>;
using Reads = std::vector<std::unique_ptr<biosoup::NucleicAcid>>;
using Piles = std::vector<std::unique_ptr<raven::Pile>>;
using Overlaps = std::vector<std::vector<biosoup::Overlap>>;

struct PileDump {
  std::vector<std::uint32_t>* out;
  void operator()(std::uint32_t& id, std::uint32_t& b, std::uint32_t& e, std::uint16_t& med,
                  bool& inv, bool& cont, bool& chim, bool& rep, std::vector<std::uint16_t>& data,
                  std::vector<bool>& kmers, std::vector<Region>& cr, std::vector<Region>& rr) {
    out->insert(out->end(), {id, b, e, med, inv, cont, chim, rep,
                             static_cast<std::uint32_t>(data.size())});
    for (auto v : data) out->push_back(v);
    out->push_back(static_cast<std::uint32_t>(kmers.size()));
    for (std::size_t i = 0; i < kmers.size(); ++i) {
      if (kmers[i]) out->push_back(static_cast<std::uint32_t>(i));
    }
    out->push_back(0xFFFFFFFFu);
    for (const auto& v : {cr, rr}) {
      out->push_back(static_cast<std::uint32_t>(v.size()));
      for (const auto& r : v) {
        out->push_back(r.first);
        out->push_back(r.second);
      }
    }
  }
};

struct PileData {
  std::vector<std::uint16_t> data;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t&, std::uint32_t&, std::uint16_t&,
                  bool&, bool&, bool&, bool&, std::vector<std::uint16_t>& d, Ts&...) {
    data = d;
  }
};

template <typename T>
std::vector<T> ReadVec(std::ifstream& f) {
  std::uint64_t n = 0;
  f.read(reinterpret_cast<char*>(&n), 8);
  std::vector<T> v(n);
  f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
  return v;
}

template <typename T>
void WriteVec(std::ofstream& f, const std::vector<T>& v) {
  std::uint64_t n = v.size();
  f.write(reinterpret_cast<const char*>(&n), 8);
  f.write(reinterpret_cast<const char*>(v.data()), n * sizeof(T));
}

void DumpOverlaps(std::ofstream& out, const Overlaps& overlaps) {
  std::vector<std::uint32_t> ovl;
  std::vector<std::uint64_t> off{0};
  for (const auto& list : overlaps) {
    for (const auto& o : list) {
      ovl.insert(ovl.end(), {o.lhs_id, o.lhs_begin, o.lhs_end, o.rhs_id, o.rhs_begin,
                             o.rhs_end, o.score, static_cast<std::uint32_t>(o.strand)});
    }
    off.push_back(ovl.size() / 8);
  }
  WriteVec(out, ovl);
  WriteVec(out, off);
}

void DumpStage2(std::ofstream& out, const Overlaps& overlaps, const Piles& piles,
                const Reads& seqs) {
  DumpOverlaps(out, overlaps);
  std::vector<std::uint32_t> pd, order;
  for (const auto& p : piles) {
    PileDump d{&pd};
    auto visit = cereal::fields(d);
    cereal::access::member_serialize(visit, *p);
  }
  for (const auto& s : seqs) order.push_back(s->id);
  WriteVec(out, pd);
  WriteVec(out, order);
}

void DumpCounters(std::ofstream& out, const ram::MinimizerEngine& engine) {
  const auto c = engine.map_counters();
  WriteVec(out, std::vector<std::uint64_t>{c.batch_maps, c.served, c.single_maps});
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 8) {
    std::cerr << "usage: facade_batch_test reads.bin out.bin k w freq minhash threads\n";
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const auto words = ReadVec<std::uint64_t>(in);
  const auto woff = ReadVec<std::uint64_t>(in);
  const auto lens = ReadVec<std::uint32_t>(in);
  const std::uint32_t k = std::stoul(argv[3]), w = std::stoul(argv[4]);
  const double freq = std::stod(argv[5]);
  const bool minhash = std::stoi(argv[6]) != 0;
  auto pool = std::make_shared<thread_pool::ThreadPool>(std::stoul(argv[7]));
  auto make_reads = [&]() {
    Reads seqs;
    for (std::size_t i = 0; i < lens.size(); ++i) {
      auto s = std::make_unique<biosoup::NucleicAcid>();
      s->id = i;
      s->name = std::to_string(i);
      s->deflated_data.assign(words.begin() + woff[i], words.begin() + woff[i + 1]);
      s->inflated_len = lens[i];
      s->is_reverse_complement = false;
      seqs.emplace_back(std::move(s));
    }
    return seqs;
  };
  std::ofstream out(argv[2], std::ios::binary);
  try {
    {  // the reference's functions over the facade
      Reads seqs = make_reads();
      ram::MinimizerEngine engine{pool, k, w};
      Piles piles;
      Overlaps overlaps(seqs.size());
      raven::FindOverlapsAndCreatePiles(pool, engine, seqs, freq, piles, overlaps, 32, minhash);
      DumpOverlaps(out, overlaps);
      std::vector<std::uint16_t> pile;
      std::vector<std::uint64_t> poff{0};
      for (const auto& p : piles) {
        PileData d;
        auto visit = cereal::fields(d);
        cereal::access::member_serialize(visit, *p);
        pile.insert(pile.end(), d.data.begin(), d.data.end());
        poff.push_back(pile.size());
      }
      WriteVec(out, pile);
      WriteVec(out, poff);
      DumpCounters(out, engine);

      raven::TrimAndAnnotatePiles(pool, piles, overlaps);
      raven::ResolveContainedReads(piles, overlaps, seqs, pool, 0);
      raven::ResolveChimericSequences(pool, piles, overlaps, seqs);
      std::uint64_t valid = 0;
      for (const auto& p : piles) valid += p->is_invalid() ? 0 : 1;
      raven::FindOverlapsAndRepetetiveRegions(pool, engine, freq, k, 0, piles, overlaps, seqs);
      DumpStage2(out, overlaps, piles, seqs);
      DumpCounters(out, engine);
      WriteVec(out, std::vector<std::uint64_t>{valid});
    }
    {  // the batched replacements
      Reads seqs = make_reads();
      ram::MinimizerEngine engine{pool, k, w};
      Piles piles;
      Overlaps overlaps(seqs.size());
      raven_b200::FindOverlapsAndCreatePiles(pool, engine, seqs, freq, piles, overlaps, 32,
                                             minhash);
      raven_b200::TrimAndAnnotatePiles(pool, piles, overlaps, engine);
      raven::ResolveContainedReads(piles, overlaps, seqs, pool, 0);
      raven::ResolveChimericSequences(pool, piles, overlaps, seqs);
      raven_b200::FindOverlapsAndRepetetiveRegions(pool, engine, freq, k, 0, piles, overlaps,
                                                   seqs);
      DumpStage2(out, overlaps, piles, seqs);
    }
  } catch (const std::exception& e) {
    std::cerr << "facade_batch_test: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}
