// The one __host__ __device__ definition of stage 2's clip and identity bound
// (include/raven_b200/overlap_clip.hpp) on the host, against the reference's own
// raven::OverlapUpdate (RavenLib overlap_utils.cc, compiled in place) and against the
// bound the host identity filter used before it moved into that header, on seeded random
// overlaps and regions with their edges. Prints "ok <cases>" or the first mismatch.
//   usage: overlap_clip_test <seed> <cases>
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <iostream>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "biosoup/overlap.hpp"
#include "raven/graph/overlap_utils.h"
#include "raven/pile.h"
#include "raven_b200/overlap_clip.hpp"

std::atomic<std::uint32_t> biosoup::NucleicAcid::num_objects{0};

namespace {

struct SetRegion {  // begin_ / end_ are in bins of 16 bases (pile.h:37-39)
  std::uint32_t b, e;
  bool invalid;
  template <typename... Ts>
  void operator()(std::uint32_t&, std::uint32_t& begin, std::uint32_t& end, std::uint16_t&,
                  bool& is_invalid, Ts&...) {
    begin = b;
    end = e;
    is_invalid = invalid;
  }
};

// the identity filter's bound as construct_b200.hpp computed it before
std::int32_t OldBound(double identity, std::size_t longest) {
  if (longest == 0) return -1;
  auto keeps = [&](std::int64_t ed) {
    const double score = 1. - static_cast<double>(ed) / longest;
    return !(score < identity);
  };
  std::int64_t e = static_cast<std::int64_t>((1. - identity) * static_cast<double>(longest)) + 2;
  e = std::min<std::int64_t>(std::max<std::int64_t>(e, 0), static_cast<std::int64_t>(longest));
  while (e >= 0 && !keeps(e)) --e;
  while (e >= 0 && e < static_cast<std::int64_t>(longest) && keeps(e + 1)) ++e;
  return static_cast<std::int32_t>(e);
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 3) {
    std::cerr << "usage: overlap_clip_test seed cases\n";
    return 2;
  }
  std::mt19937_64 rng(std::stoull(argv[1]));
  const std::uint64_t cases = std::stoull(argv[2]);
  auto uni = [&](std::uint64_t lo, std::uint64_t hi) {  // [lo, hi]
    return std::uniform_int_distribution<std::uint64_t>(lo, hi)(rng);
  };
  std::vector<std::unique_ptr<raven::Pile>> piles;
  piles.emplace_back(new raven::Pile(0, 1));
  piles.emplace_back(new raven::Pile(1, 1));
  std::uint64_t clipped = 0, dropped = 0;
  for (std::uint64_t t = 0; t < cases; ++t) {
    // regions: anything from empty to the whole read, often right at an overlap's end
    std::uint32_t len[2], rb[2], re[2];
    bool inv[2];
    for (int p = 0; p < 2; ++p) {
      len[p] = static_cast<std::uint32_t>(uni(0, 4) == 0 ? uni(0, 300) : uni(84, 40000));
      const std::uint32_t bins = len[p] >> 4;
      rb[p] = static_cast<std::uint32_t>(uni(0, 3) == 0 ? 0 : uni(0, bins));
      re[p] = static_cast<std::uint32_t>(uni(0, 3) == 0 ? bins : uni(rb[p], bins));
      inv[p] = uni(0, 15) == 0;
      SetRegion door{rb[p], re[p], inv[p]};
      auto visit = cereal::fields(door);
      cereal::access::member_serialize(visit, *piles[p]);
    }
    auto pos = [&](int p) -> std::uint32_t {
      switch (uni(0, 5)) {  // the region's edges and the bases next to them
        case 0: return (rb[p] << 4) + static_cast<std::uint32_t>(uni(0, 2)) - 1;
        case 1: return (re[p] << 4) + static_cast<std::uint32_t>(uni(0, 2)) - 1;
        case 2: return (rb[p] << 4) + 84 + static_cast<std::uint32_t>(uni(0, 2)) - 1;
        default: return static_cast<std::uint32_t>(uni(0, len[p]));
      }
    };
    std::uint32_t a = pos(0), b = pos(0), c = pos(1), d = pos(1);
    if (a > b) std::swap(a, b);
    if (c > d) std::swap(c, d);
    if (uni(0, 7) == 0) std::swap(a, b);  // begin >= end as well
    biosoup::Overlap o(0, a, b, 1, c, d, 7, uni(0, 1) != 0);
    biosoup::Overlap want = o;
    const bool want_ok = raven::OverlapUpdate(want, piles);
    std::uint32_t lb = a, le = b, xb = c, xe = d;
    const bool got_ok = rvn::OverlapClip(lb, le, xb, xe, o.strand,
                                         rvn::PileRegion{rb[0] << 4, re[0] << 4, inv[0]},
                                         rvn::PileRegion{rb[1] << 4, re[1] << 4, inv[1]});
    if (got_ok != want_ok || lb != want.lhs_begin || le != want.lhs_end ||
        xb != want.rhs_begin || xe != want.rhs_end) {
      std::cout << "MISMATCH clip case " << t << ": (" << a << "," << b << "," << c << ","
                << d << "," << o.strand << ") regions (" << (rb[0] << 4) << "," << (re[0] << 4)
                << "," << inv[0] << ") (" << (rb[1] << 4) << "," << (re[1] << 4) << ","
                << inv[1] << ") reference " << want_ok << " got " << got_ok << "\n";
      return 1;
    }
    (want_ok ? clipped : dropped)++;
    // the bound: identity on a grid, at its ends and at random; lengths small and large
    const double grid[] = {0.0, 0.5, 0.8, 0.9, 0.95, 0.99, 0.999, 1.0};
    const double identity = uni(0, 1) ? grid[uni(0, 7)]
                                      : std::uniform_real_distribution<double>(0, 1)(rng);
    const std::uint64_t longest = uni(0, 3) == 0 ? uni(0, 200) : uni(0, 200000);
    const std::int32_t got = rvn::IdentityBound(identity, longest);
    const std::int32_t old = OldBound(identity, longest);
    auto keeps = [&](std::int64_t ed) {
      return !(1. - static_cast<double>(ed) / static_cast<double>(longest) < identity);
    };
    const bool exact = longest == 0 ? got == -1
                                    : ((got < 0 || keeps(got)) &&
                                       (got >= static_cast<std::int64_t>(longest) ||
                                        !keeps(static_cast<std::int64_t>(got) + 1)));
    if (got != old || !exact) {
      std::cout << "MISMATCH bound case " << t << ": identity " << identity << " longest "
                << longest << " got " << got << " before " << old << "\n";
      return 1;
    }
  }
  std::cout << "ok " << cases << " clipped " << clipped << " dropped " << dropped << "\n";
  return 0;
}
