// The drop-in parser's route for profiles/fastx_load.py: raven's input loop over one FASTQ(.gz)
// file (bioparser::FastqParser + biosoup::NucleicAcid). Prints "<reads> <bases>".
#include <atomic>
#include <iostream>

#include "bioparser/fastq_parser.hpp"
#include "biosoup/nucleic_acid.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  auto p = bioparser::Parser<biosoup::NucleicAcid>::Create<bioparser::FastqParser>(argv[1]);
  const auto reads = p->Parse(-1);
  unsigned long long bases = 0;
  for (const auto& it : reads) bases += it->inflated_len;
  std::cout << reads.size() << " " << bases << "\n";
  return 0;
}
