// raven_b200 — the identity filter's arithmetic of raven::FindOverlapsAndRepetetiveRegions
// (RavenLib/src/construct.cc:385-424), one definition for the host and the device: the
// stage-2 kernels of editdist.cu and the host IdentityFilter of construct_b200.hpp both
// include it. Plain C++ without a CUDA compiler (tests/cpp/overlap_clip_test.cc checks it
// against the reference's overlap_utils.cc on the host).
#ifndef RAVEN_B200_OVERLAP_CLIP_HPP_
#define RAVEN_B200_OVERLAP_CLIP_HPP_

#include <cstdint>

#ifndef RVN_HD
#if defined(__CUDACC__)
#define RVN_HD __host__ __device__ __forceinline__
#else
#define RVN_HD inline
#endif
#endif

namespace rvn {

// Largest edit distance the identity filter still keeps for substrings whose longer one
// has `longest` bases: the reference drops an overlap iff
// 1. - double(ed) / longest < identity. Both operations are monotone in ed, so the
// decision is "ed <= bound" - computed here with the SAME double arithmetic, which makes
// a bounded distance search exact. -1: nothing passes.
RVN_HD std::int32_t IdentityBound(double identity, std::uint64_t longest) {
  if (longest == 0) return -1;
  const std::int64_t n = static_cast<std::int64_t>(longest);
  auto keeps = [&](std::int64_t ed) {
    const double score = 1. - static_cast<double>(ed) / static_cast<double>(longest);
    return !(score < identity);
  };
  std::int64_t e = static_cast<std::int64_t>((1. - identity) * static_cast<double>(longest)) + 2;
  e = e < 0 ? 0 : (e > n ? n : e);
  while (e >= 0 && !keeps(e)) --e;
  while (e >= 0 && e < n && keeps(e + 1)) ++e;
  return static_cast<std::int32_t>(e);
}

// The valid region [begin, end) of a pile in bases (raven::Pile::begin() / end()) and
// its is_invalid() flag.
struct PileRegion {
  std::uint32_t begin, end;
  bool invalid;
};

// raven::OverlapUpdate (RavenLib/src/overlap_utils.cc:14-60) on the overlap's fields:
// clips both sides to the piles' valid regions (lhs: its own pile, rhs: the rhs pile;
// the other side's cut mirrored through the strand) and returns false, leaving the
// fields untouched, when either side leaves its region or keeps fewer than 84 bases.
RVN_HD bool OverlapClip(std::uint32_t& o_lhs_begin, std::uint32_t& o_lhs_end,
                        std::uint32_t& o_rhs_begin, std::uint32_t& o_rhs_end, bool strand,
                        PileRegion l, PileRegion r) {
  if (l.invalid || r.invalid) return false;
  if (o_lhs_begin >= l.end || o_lhs_end <= l.begin || o_rhs_begin >= r.end ||
      o_rhs_end <= r.begin) {
    return false;
  }
  const std::uint32_t rb_cut = o_rhs_begin < r.begin ? r.begin - o_rhs_begin : 0;
  const std::uint32_t re_cut = o_rhs_end > r.end ? o_rhs_end - r.end : 0;
  const std::uint32_t lb_cut = o_lhs_begin < l.begin ? l.begin - o_lhs_begin : 0;
  const std::uint32_t le_cut = o_lhs_end > l.end ? o_lhs_end - l.end : 0;
  // (unsigned arithmetic wraps as the reference's does)
  std::uint32_t lhs_begin = o_lhs_begin + (strand ? rb_cut : re_cut);
  std::uint32_t lhs_end = o_lhs_end - (strand ? re_cut : rb_cut);
  std::uint32_t rhs_begin = o_rhs_begin + (strand ? lb_cut : le_cut);
  std::uint32_t rhs_end = o_rhs_end - (strand ? le_cut : lb_cut);
  if (lhs_begin >= l.end || lhs_end <= l.begin || rhs_begin >= r.end || rhs_end <= r.begin) {
    return false;
  }
  lhs_begin = lhs_begin > l.begin ? lhs_begin : l.begin;
  lhs_end = lhs_end < l.end ? lhs_end : l.end;
  rhs_begin = rhs_begin > r.begin ? rhs_begin : r.begin;
  rhs_end = rhs_end < r.end ? rhs_end : r.end;
  if (lhs_begin >= lhs_end || lhs_end - lhs_begin < 84 || rhs_begin >= rhs_end ||
      rhs_end - rhs_begin < 84) {
    return false;
  }
  o_lhs_begin = lhs_begin;
  o_lhs_end = lhs_end;
  o_rhs_begin = rhs_begin;
  o_rhs_end = rhs_end;
  return true;
}

}  // namespace rvn

#endif  // RAVEN_B200_OVERLAP_CLIP_HPP_
