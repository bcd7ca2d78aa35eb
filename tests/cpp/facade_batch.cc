// Replays a schedule of ram::MinimizerEngine calls (the product's facade over
// libraven_b200.so, no reference sources) and dumps every Map result, so that
// tests/test_gpu_facade_batch.py can compare them with the CPU oracle replaying
// the same schedule (build() compiles it into tests/cpp/_build). Map calls
// between two other lines run concurrently on a pool, the way raven's stage 1
// issues them (construct.cc:59-64).
//   usage: facade_batch <reads.bin> <script.txt> <out.bin> <k> <w> <threads>
// Script lines:
//   minimize <first> <last> <minhash>
//   filter <frequency>
//   map <read> <avoid_equal> <avoid_symmetric> <minhash> <want_filtered>
//   map_rc <read> ...                 (the same on a reverse-complemented view)
//   mutate <read> <source>            (read takes the source's bases, keeps its id)
//   reset <read>                      (frees the read)
//   counters                          (dumps batch maps, served, single maps)
// Output, in script order: per map line its overlaps (8 u32 each) and filtered
// positions; per counters line three u64.
#include <atomic>
#include <cstdint>
#include <fstream>
#include <future>
#include <iostream>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "ram/minimizer_engine.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace {

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

struct Result {
  std::vector<std::uint32_t> overlaps, filtered;
};

}  // namespace

int main(int argc, char** argv) {
  if (argc < 7) {
    std::cerr << "usage: facade_batch reads.bin script.txt out.bin k w threads\n";
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const auto words = ReadVec<std::uint64_t>(in);
  const auto woff = ReadVec<std::uint64_t>(in);
  const auto lens = ReadVec<std::uint32_t>(in);
  const std::uint32_t k = std::stoul(argv[4]), w = std::stoul(argv[5]);
  auto pool = std::make_shared<thread_pool::ThreadPool>(std::stoul(argv[6]));

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

  std::ifstream script(argv[2]);
  std::ofstream out(argv[3], std::ios::binary);
  try {
    ram::MinimizerEngine engine{pool, k, w};
    std::vector<std::future<Result>> pending;
    auto drain = [&]() {
      for (auto& f : pending) {
        const Result r = f.get();
        WriteVec(out, r.overlaps);
        WriteVec(out, r.filtered);
      }
      pending.clear();
    };
    std::string line;
    while (std::getline(script, line)) {
      std::istringstream ls(line);
      std::string op;
      if (!(ls >> op)) continue;
      if (op == "map" || op == "map_rc") {
        std::uint32_t i = 0;
        int ae = 0, as = 0, mh = 0, wf = 0;
        ls >> i >> ae >> as >> mh >> wf;
        std::shared_ptr<std::unique_ptr<biosoup::NucleicAcid>> view;
        if (op == "map_rc") {
          view = std::make_shared<std::unique_ptr<biosoup::NucleicAcid>>(
              new biosoup::NucleicAcid(*seqs[i]));
          (*view)->ReverseAndComplement();
        }
        pending.emplace_back(pool->Submit(
            [&, view, i, ae, as, mh, wf]() -> Result {
              Result r;
              std::vector<std::uint32_t> filtered;
              const auto& seq = view ? *view : seqs[i];
              for (const auto& o : engine.Map(seq, ae, as, mh, wf ? &filtered : nullptr)) {
                r.overlaps.insert(r.overlaps.end(),
                                  {o.lhs_id, o.lhs_begin, o.lhs_end, o.rhs_id, o.rhs_begin,
                                   o.rhs_end, o.score, static_cast<std::uint32_t>(o.strand)});
              }
              r.filtered = filtered;
              return r;
            }));
        continue;
      }
      drain();
      if (op == "minimize") {
        std::uint32_t first = 0, last = 0;
        int mh = 0;
        ls >> first >> last >> mh;
        engine.Minimize(seqs.begin() + first, seqs.begin() + last, mh != 0);
      } else if (op == "filter") {
        double f = 0;
        ls >> f;
        engine.Filter(f);
      } else if (op == "mutate") {
        std::uint32_t i = 0, src = 0;
        ls >> i >> src;
        seqs[i]->deflated_data = seqs[src]->deflated_data;
        seqs[i]->inflated_len = seqs[src]->inflated_len;
      } else if (op == "reset") {
        std::uint32_t i = 0;
        ls >> i;
        seqs[i].reset();
      } else if (op == "counters") {
        const auto c = engine.map_counters();
        WriteVec(out, std::vector<std::uint64_t>{c.batch_maps, c.served, c.single_maps});
      } else {
        throw std::invalid_argument("unknown script line: " + line);
      }
    }
    drain();
  } catch (const std::exception& e) {
    std::cerr << "facade_batch: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}
