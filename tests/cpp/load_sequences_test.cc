// GPU check of raven_b200::LoadSequences against raven's input loop over the drop-in
// bioparser (RavenExe/src/main.cc:258-299 with raven::CreateParser, RavenLib/src/io.cc:7-41),
// field by field, ids included.
//   usage: load_sequences_test <path>...   -> "ok <reads>" (exit 0) or the first difference
#include <atomic>
#include <iostream>
#include <string>
#include <vector>

#include "bioparser/fasta_parser.hpp"
#include "bioparser/fastq_parser.hpp"
#include "biosoup/nucleic_acid.hpp"
#include "raven_b200/load_sequences.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace {

bool IsSuffix(const std::string& s, const std::string& suff) {
  return s.size() >= suff.size() && s.compare(s.size() - suff.size(), suff.size(), suff) == 0;
}

std::vector<std::unique_ptr<biosoup::NucleicAcid>> Reference(const std::vector<std::string>& paths) {
  using P = bioparser::Parser<biosoup::NucleicAcid>;
  std::vector<std::unique_ptr<biosoup::NucleicAcid>> sequences;
  for (const auto& path : paths) {
    std::unique_ptr<P> p;
    if (IsSuffix(path, ".fasta") || IsSuffix(path, ".fa") || IsSuffix(path, ".fasta.gz") ||
        IsSuffix(path, ".fa.gz")) {
      p = P::Create<bioparser::FastaParser>(path);
    } else {
      p = P::Create<bioparser::FastqParser>(path);
    }
    auto chunk = p->Parse(-1);
    for (auto& it : chunk) sequences.emplace_back(std::move(it));
  }
  return sequences;
}

}  // namespace

int main(int argc, char** argv) {
  const std::vector<std::string> paths(argv + 1, argv + argc);
  biosoup::NucleicAcid::num_objects = 0;
  const auto want = Reference(paths);
  biosoup::NucleicAcid::num_objects = 0;
  const auto got = raven_b200::LoadSequences(paths);
  if (got.size() != want.size()) {
    std::cout << "reads " << got.size() << " != " << want.size() << "\n";
    return 1;
  }
  for (std::size_t i = 0; i < got.size(); ++i) {
    const auto& a = *got[i];
    const auto& b = *want[i];
    if (a.id != b.id || a.name != b.name || a.deflated_data != b.deflated_data ||
        a.block_quality != b.block_quality || a.inflated_len != b.inflated_len ||
        a.is_reverse_complement != b.is_reverse_complement) {
      std::cout << "read " << i << " differs (" << b.name << ")\n";
      return 1;
    }
  }
  if (biosoup::NucleicAcid::num_objects != want.size()) {
    std::cout << "num_objects " << biosoup::NucleicAcid::num_objects << "\n";
    return 1;
  }
  std::cout << "ok " << got.size() << "\n";
  return 0;
}
