// Stage 2 as one device call against the reference: the reference's OWN
// raven::FindOverlapsAndRepetetiveRegions (RavenLib construct.cc compiled in place, per-read
// Map calls through the ram::MinimizerEngine facade, Pile::AddKmers and edlibAlign on the
// host) next to raven_b200::FindOverlapsAndRepetetiveRegions, which runs over
// rvn_find_overlaps_and_repetitive_regions. Both start from the same state (stage 1, the
// pile annotation, containment and chimeric removal). Written per run: the state stage 2
// starts from (sorted valid ids, s, each valid pile's region), then the end state: every
// overlap list and every pile as the reference's cereal JSON (tests/test_gpu_stage2.py).
//   usage: stage2_call_test <reads.bin> <out.bin> <k> <w> <freq> <identity> <all_valid>
// all_valid = 1 clears every pile's is_invalid before stage 2 (the s == 0 case).
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <fstream>
#include <iostream>
#include <memory>
#include <sstream>
#include <stdexcept>
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

struct ClearInvalid {
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t&, std::uint32_t&, std::uint16_t&, bool& inv,
                  Ts&...) {
    inv = false;
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

}  // namespace

int main(int argc, char** argv) {
  if (argc < 8) {
    std::cerr << "usage: stage2_call_test reads.bin out.bin k w freq identity all_valid\n";
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const auto words = ReadVec<std::uint64_t>(in);
  const auto woff = ReadVec<std::uint64_t>(in);
  const auto lens = ReadVec<std::uint32_t>(in);
  const std::uint32_t k = std::stoul(argv[3]), w = std::stoul(argv[4]);
  const double freq = std::stod(argv[5]), identity = std::stod(argv[6]);
  const bool all_valid = std::stoi(argv[7]) != 0;
  auto pool = std::make_shared<thread_pool::ThreadPool>(4);
  std::ofstream out(argv[2], std::ios::binary);
  try {
    for (int mode = 0; mode < 2; ++mode) {
      std::vector<std::unique_ptr<biosoup::NucleicAcid>> seqs;
      for (std::size_t i = 0; i < lens.size(); ++i) {
        auto s = std::make_unique<biosoup::NucleicAcid>();
        s->id = i;
        s->name = std::to_string(i);
        s->deflated_data.assign(words.begin() + woff[i], words.begin() + woff[i + 1]);
        s->inflated_len = lens[i];
        s->is_reverse_complement = false;
        seqs.emplace_back(std::move(s));
      }
      ram::MinimizerEngine engine{pool, k, w};
      std::vector<std::unique_ptr<raven::Pile>> piles;
      std::vector<std::vector<biosoup::Overlap>> overlaps(seqs.size());
      raven_b200::FindOverlapsAndCreatePiles(pool, engine, seqs, freq, piles, overlaps, 32, false);
      raven_b200::TrimAndAnnotatePiles(pool, piles, overlaps, engine);
      raven_b200::ResolveContainedReads(piles, overlaps, seqs, pool, identity, engine);
      raven::ResolveChimericSequences(pool, piles, overlaps, seqs);
      if (all_valid) {
        for (auto& p : piles) {
          ClearInvalid door;
          auto visit = cereal::fields(door);
          cereal::access::member_serialize(visit, *p);
        }
      }
      // the state stage 2 starts from: valid reads in the reference's sorted order
      std::vector<std::uint32_t> valid, region;
      std::uint32_t s = 0;
      {
        std::vector<std::uint32_t> order(seqs.size());
        for (std::uint32_t i = 0; i < seqs.size(); ++i) order[i] = seqs[i]->id;
        std::stable_sort(order.begin(), order.end(), [&](std::uint32_t a, std::uint32_t b) {
          return piles[a]->is_invalid() < piles[b]->is_invalid() ||
                 (piles[a]->is_invalid() == piles[b]->is_invalid() && a < b);
        });
        for (std::uint32_t i = 0; i < order.size(); ++i) {
          if (piles[order[i]]->is_invalid()) {
            s = i;
            break;
          }
        }
        for (std::uint32_t i = 0; i < s; ++i) {
          valid.push_back(order[i]);
          region.push_back(piles[order[i]]->begin());
          region.push_back(piles[order[i]]->end());
        }
      }
      if (mode == 0) {
        raven::FindOverlapsAndRepetetiveRegions(pool, engine, freq, k, identity, piles, overlaps,
                                                seqs);
      } else {
        raven_b200::FindOverlapsAndRepetetiveRegions(pool, engine, freq, k, identity, piles,
                                                     overlaps, seqs);
      }
      std::vector<std::uint32_t> ovl;
      std::vector<std::uint64_t> off{0};
      for (const auto& list : overlaps) {
        for (const auto& o : list) {
          ovl.insert(ovl.end(), {o.lhs_id, o.lhs_begin, o.lhs_end, o.rhs_id, o.rhs_begin,
                                 o.rhs_end, o.score, static_cast<std::uint32_t>(o.strand)});
        }
        off.push_back(ovl.size() / 8);
      }
      std::ostringstream js;
      {
        cereal::JSONOutputArchive ar(js);
        for (const auto& p : piles) ar(cereal::make_nvp(std::to_string(p->id()), *p));
      }
      const std::string j = js.str();
      WriteVec(out, valid);
      WriteVec(out, std::vector<std::uint32_t>{s});
      WriteVec(out, region);
      WriteVec(out, ovl);
      WriteVec(out, off);
      WriteVec(out, std::vector<char>(j.begin(), j.end()));
    }
  } catch (const std::exception& e) {
    std::cerr << "stage2_call_test: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}
