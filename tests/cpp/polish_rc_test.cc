// Product-only test driver: racon::Polisher::Polish over targets and reads whose
// biosoup::NucleicAcid has is_reverse_complement set - a state only C++ callers reach
// (the Python and flat entry points build plain objects). The product facade's output
// is compared with the oracle polisher's (oracle/liboracle.so, loaded at run time) on
// the same objects: the same names and the same polished bases.
// Usage: polish_rc_test <path of liboracle.so>; prints "polish_rc_test ok".
#include <dlfcn.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "../../oracle/flat_api.hpp"
#include "biosoup/nucleic_acid.hpp"
#include "racon/polisher.hpp"
#include "thread_pool/thread_pool.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace {

using Seqs = std::vector<std::unique_ptr<biosoup::NucleicAcid>>;

std::string Mutate(std::mt19937_64& rng, const std::string& s, double rate) {
  std::uniform_real_distribution<double> u(0, 1);
  std::string out;
  for (char c : s) {
    const double x = u(rng);
    if (x < rate / 3) continue;
    if (x < 2 * rate / 3) {
      out += "ACGT"[(std::string("ACGT").find(c) + 1 + rng() % 3) % 4];
    } else {
      out += c;
      if (x < rate) out += "ACGT"[rng() % 4];
    }
  }
  return out;
}

std::string ReverseComplement(const std::string& s) {
  std::string r(s.rbegin(), s.rend());
  for (char& c : r) c = "TGCA"[std::string("ACGT").find(c)];
  return r;
}

// one set of objects: the product's, or the oracle's built from the same words
struct Flat {
  std::vector<std::uint64_t> words, woff{0};
  std::vector<std::uint32_t> lens;
  std::vector<std::uint8_t> bq;
  std::vector<std::uint64_t> bq_off{0};
  std::vector<bool> rc;
};

Flat Flatten(const Seqs& v) {
  Flat f;
  for (const auto& s : v) {
    f.words.insert(f.words.end(), s->deflated_data.begin(), s->deflated_data.end());
    f.woff.push_back(f.words.size());
    f.lens.push_back(s->inflated_len);
    f.bq.insert(f.bq.end(), s->block_quality.begin(), s->block_quality.end());
    f.bq_off.push_back(f.bq.size());
    f.rc.push_back(s->is_reverse_complement);
  }
  return f;
}

template <typename F>
F Sym(void* lib, const char* name) {
  void* p = dlsym(lib, name);
  if (!p) {
    std::fprintf(stderr, "missing symbol %s\n", name);
    std::exit(2);
  }
  return reinterpret_cast<F>(p);
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 2) {
    std::fprintf(stderr, "usage: polish_rc_test <liboracle.so>\n");
    return 2;
  }
  std::mt19937_64 rng(29);
  std::string genome;
  for (int i = 0; i < 24000; ++i) genome += "ACGT"[rng() % 4];
  // two draft contigs; the second is stored reverse complemented with the flag set, so
  // its view reads along the genome
  Seqs targets, sequences;
  for (int t = 0; t < 2; ++t) {
    const std::string d = Mutate(rng, genome.substr(t * 12000, 12000), 0.01);
    targets.emplace_back(new biosoup::NucleicAcid("Utg" + std::to_string(t),
                                                  t ? ReverseComplement(d) : d));
    if (t) targets.back()->ReverseAndComplement();
  }
  // reads of both strands with qualities; every third one is flagged (its stored bases
  // are the reverse complement of what it reads), some have no qualities, and lengths
  // fall on and off the 32-base words and 64-base quality blocks
  for (int i = 0; i < 150; ++i) {
    std::uint32_t len = 1500 + rng() % 3000;
    if (i % 5 == 0) len += 64 - len % 64;  // whole quality blocks
    if (i % 5 == 1) len += 32 - len % 32;  // whole words
    const std::uint32_t b = rng() % (genome.size() - len);
    std::string r = Mutate(rng, genome.substr(b, len), 0.06);
    if (i % 2) r = ReverseComplement(r);
    const bool flag = i % 3 == 0;
    std::string qual;
    for (std::size_t x = 0; x < r.size(); ++x) qual += static_cast<char>('!' + 4 + rng() % 22);
    auto s = i % 7 == 3 ? std::make_unique<biosoup::NucleicAcid>("r" + std::to_string(i),
                                                                 flag ? ReverseComplement(r) : r)
                        : std::make_unique<biosoup::NucleicAcid>(
                              "r" + std::to_string(i), flag ? ReverseComplement(r) : r, qual);
    if (flag) s->ReverseAndComplement();
    sequences.emplace_back(std::move(s));
  }

  void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) {
    std::fprintf(stderr, "dlopen: %s\n", dlerror());
    return 2;
  }
  using Create = orc_reads* (*)(const std::uint64_t*, const std::uint64_t*, const std::uint32_t*,
                                std::uint32_t, const std::uint8_t*, const std::uint64_t*);
  using PolishFn = orc_bag* (*)(orc_reads*, orc_reads*, double, double, std::uint32_t, int, int,
                                int, int, std::uint32_t);
  using BagLen = std::int64_t (*)(orc_bag*, const char*);
  using BagPtr = const void* (*)(orc_bag*, const char*);
  auto create = Sym<Create>(lib, "orc_reads_create");
  auto polish = Sym<PolishFn>(lib, "orc_polish");
  auto bag_len = Sym<BagLen>(lib, "orc_bag_len");
  auto bag_ptr = Sym<BagPtr>(lib, "orc_bag_ptr");
  auto bag_free = Sym<void (*)(orc_bag*)>(lib, "orc_bag_free");
  auto reads_free = Sym<void (*)(orc_reads*)>(lib, "orc_reads_free");
  // the oracle's objects: the same words, qualities, flags and names
  auto oracle_reads = [&](const Seqs& v) {
    const Flat f = Flatten(v);
    orc_reads* r = create(f.words.data(), f.woff.data(), f.lens.data(),
                          static_cast<std::uint32_t>(v.size()), f.bq.data(), f.bq_off.data());
    for (std::size_t i = 0; i < v.size(); ++i) {
      r->seqs[i]->is_reverse_complement = f.rc[i];
      r->seqs[i]->name = v[i]->name;
    }
    return r;
  };

  // the flagged reads alone: they must reach both targets by themselves
  Seqs flagged;
  for (const auto& s : sequences) {
    if (s->is_reverse_complement) flagged.emplace_back(new biosoup::NucleicAcid(*s));
  }
  struct Case {
    double q;
    const Seqs* reads;
  };
  int failures = 0;
  for (const Case& cs : {Case{0.0, &sequences}, Case{10.0, &sequences}, Case{0.0, &flagged}}) {
    const double q = cs.q;
    auto pool = std::make_shared<thread_pool::ThreadPool>(4);
    auto got = racon::Polisher::Create(pool, q, 0.3, 500, true, 3, -5, -4)
                   ->Polish(targets, *cs.reads, false);
    orc_reads* ot = oracle_reads(targets);
    orc_reads* os = oracle_reads(*cs.reads);
    orc_bag* bag = polish(ot, os, q, 0.3, 500, 1, 3, -5, -4, 4);
    const auto* seq = static_cast<const char*>(bag_ptr(bag, "sequences"));
    const auto* off = static_cast<const std::uint64_t*>(bag_ptr(bag, "seq_off"));
    const std::string names(static_cast<const char*>(bag_ptr(bag, "names")),
                            static_cast<std::size_t>(bag_len(bag, "names")));
    const std::size_t n_want = static_cast<std::size_t>(bag_len(bag, "seq_off")) / 8 - 1;
    std::string got_names;
    for (const auto& p : got) got_names += p->name + "\n";
    bool ok = got.size() == n_want && got_names == names;
    for (std::size_t i = 0; ok && i < n_want; ++i) {
      ok = got[i]->InflateData() == std::string(seq + off[i], seq + off[i + 1]);
      // the flagged reads aligned and polished both targets, the flagged one included
      const std::string& name = got[i]->name;
      const double polished = std::stod(name.substr(name.find(" XC:f:") + 6));
      if (ok && (polished < 0.5 || got[i]->InflateData() == targets[i]->InflateData())) {
        std::printf("target %zu is not polished: %s\n", i, name.c_str());
        ok = false;
      }
    }
    std::printf("q=%.1f, %zu reads: %zu polished targets, %s\n", q, cs.reads->size(), got.size(),
                ok ? "equal" : "DIFFERENT");
    failures += !ok || n_want != targets.size();
    bag_free(bag);
    reads_free(ot);
    reads_free(os);
  }
  if (failures) return 1;
  std::printf("polish_rc_test ok\n");
  return 0;
}
