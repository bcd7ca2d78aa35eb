// Host build of raven_b200/csrc/chain.cuh for tests/test_chain_host.py.
#include <vector>

#include "../raven_b200/csrc/chain.cuh"

// ChainPairSerial over the m hits of one pair; params = k, bandwidth, chain, matches,
// gap. Writes up to cap overlaps and returns how many there are.
extern "C" __attribute__((visibility("default"))) std::uint64_t rvn_test_chain_pair(
    const std::uint64_t* group, const std::uint64_t* positions, std::uint32_t m,
    std::uint32_t lhs_id, const std::uint32_t* params, rvn_overlap* out, std::uint64_t cap) {
  std::vector<std::uint64_t> P(positions, positions + m);
  std::vector<std::uint32_t> D(m);
  for (std::uint32_t i = 0; i < m; ++i) D[i] = static_cast<std::uint32_t>(group[i]);
  const rvn::Column c{P.data(), D.data(), 1};
  const rvn::ChainParams cp{params[0], params[1], params[2], params[3], params[4]};
  std::uint64_t n = 0;
  rvn::ChainPairSerial(c, m, m ? static_cast<std::uint32_t>(group[0] >> 32) : 0, lhs_id, cp,
                       [&](const rvn_overlap& o) {
                         if (n < cap) out[n] = o;
                         ++n;
                       });
  return n;
}
