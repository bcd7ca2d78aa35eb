// ORACLE — TEST INFRASTRUCTURE ONLY.
// Global (NW, unit cost) alignment PATH, the role of
// edlibAlign(..., {k=-1, EDLIB_MODE_NW, EDLIB_TASK_PATH}) inside racon
// (SURVEY.md App. A.4 step 3), by plain banded dynamic programming. Among the
// equally optimal paths upstream edlib (un-vendored; version not stated in the
// tree) returns ONE, fixed by two rules of its edlib.cpp that are restated here:
//   * obtainAlignmentTraceback: walking back from the end, a cell first tries the
//     cell above ('I', query base only), then the cell to the left ('D', target
//     base only), then the diagonal;
//   * obtainAlignment: that traceback only serves problems whose alignment data
//     ((2*8+4) * ceil(|q|/64) * |t| + 8 * |t| bytes) stays below 1 MiB; larger ones
//     are split Hirschberg-style at target column |t|/2 through the SMALLEST
//     query row on an optimal path (rows 1..|q|-1 first, then 0, then |q|).
// PINNED: with these rules the reference's own end-to-end golden value is
// reproduced exactly (RavenTest.Assemble == 1137, raven_test.cpp:66;
// tests/test_oracle.py::test_end_to_end_pin_against_reference_golden). Without the
// split the six fixed preference orders give 1131..1166 (ORC_NW_NO_HIRSCHBERG,
// ORC_NW_PREF experiment knobs).
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

#include "racon/polisher.hpp"

namespace racon {

namespace {

constexpr std::int32_t kInf = 1 << 29;

// D[r][L] for r = 0..n over the band |r - c| <= k: edit distance between q[0, r)
// and t[0, L); entries outside the band are kInf. Every entry <= k is exact.
std::vector<std::int32_t> DistanceColumn(const char* q, std::int64_t n, const char* t,
                                         std::int64_t L, std::int64_t k) {
  std::vector<std::int32_t> col(n + 1, kInf), nxt(n + 1, kInf);
  for (std::int64_t r = 0; r <= std::min(n, k); ++r) col[r] = static_cast<std::int32_t>(r);
  for (std::int64_t c = 1; c <= L; ++c) {
    const std::int64_t lo = std::max<std::int64_t>(0, c - k), hi = std::min(n, c + k);
    if (lo > 0) nxt[lo - 1] = kInf;
    for (std::int64_t r = lo; r <= hi; ++r) {
      std::int32_t best = col[r] + 1;  // left
      if (r > 0) {
        best = std::min(best, nxt[r - 1] + 1);                          // up
        best = std::min(best, col[r - 1] + (q[r - 1] != t[c - 1]));     // diagonal
      }
      nxt[r] = std::min(best, kInf);
    }
    if (hi < n) nxt[hi + 1] = kInf;
    // rows that left the band at the top must not be read again
    if (lo >= 1 && lo - 1 <= n) col[lo - 1] = kInf;
    col.swap(nxt);
  }
  // cells outside the final band hold stale values: blank them
  for (std::int64_t r = 0; r <= n; ++r) {
    if (r < L - k || r > L + k) col[r] = kInf;
  }
  return col;
}

// edlib's obtainAlignmentTraceback on the full matrix of (q, t): from (n, m) walk
// back preferring up (query base alone, 'I'), then left (target base alone, 'D'),
// then the diagonal. `pref` = experiment knob (ORC_NW_PREF).
void Traceback(const char* q, std::int64_t n, const char* t, std::int64_t m,
               std::int64_t k, const int* pref, std::string* out) {
  // band of diagonals j - i in [lo, hi], clipped to the matrix; row i keeps
  // columns [max(0, i + lo), min(m, i + hi)] (at most m + 1 of them, so a long
  // query against a short target does not pay for the whole diagonal range)
  const std::int64_t lo = std::max(-n, -k + std::min<std::int64_t>(0, m - n) - 1);
  const std::int64_t hi = std::min(m, k + std::max<std::int64_t>(0, m - n) + 1);
  const std::int64_t width = std::min(hi - lo + 1, m + 1);
  std::vector<std::int32_t> H(static_cast<std::size_t>(n + 1) * width, kInf);
  auto slot = [&](std::int64_t i, std::int64_t j) -> std::size_t {
    return static_cast<std::size_t>(i) * width + (j - std::max<std::int64_t>(0, i + lo));
  };
  auto at = [&](std::int64_t i, std::int64_t j) -> std::int32_t& { return H[slot(i, j)]; };
  auto get = [&](std::int64_t i, std::int64_t j) -> std::int32_t {
    if (i < 0 || j < 0 || j > m || j - i < lo || j - i > hi) return kInf;
    return H[slot(i, j)];
  };
  for (std::int64_t i = 0; i <= n; ++i) {
    const std::int64_t jb = std::max<std::int64_t>(0, i + lo), je = std::min(m, i + hi);
    for (std::int64_t j = jb; j <= je; ++j) {
      std::int32_t v;
      if (i == 0) {
        v = static_cast<std::int32_t>(j);
      } else if (j == 0) {
        v = static_cast<std::int32_t>(i);
      } else {
        v = std::min(get(i - 1, j - 1) + (q[i - 1] != t[j - 1]),
                     std::min(get(i - 1, j) + 1, get(i, j - 1) + 1));
      }
      at(i, j) = std::min(v, kInf);
    }
  }
  std::string rev;
  std::int64_t i = n, j = m;
  while (i > 0 || j > 0) {
    const std::int32_t cur = get(i, j);
    int move = 0;
    for (int z = 0; z < 3 && !move; ++z) {
      const int which = pref[z];
      if (which == 2 && i > 0 && get(i - 1, j) + 1 == cur) move = 2;
      if (which == 3 && j > 0 && get(i, j - 1) + 1 == cur) move = 3;
      if (which == 1 && i > 0 && j > 0 &&
          get(i - 1, j - 1) + (q[i - 1] != t[j - 1]) == cur) move = 1;
    }
    if (move == 2) { rev += 'I'; --i; }
    else if (move == 3) { rev += 'D'; --j; }
    else { rev += 'M'; --i; --j; }
  }
  out->append(rev.rbegin(), rev.rend());
}

// edlib's obtainAlignment: plain traceback when its alignment data would stay
// below 1 MB, else Hirschberg's split at the middle target column - the path
// passes row r of that column for the SMALLEST r in [1, n-1] with
// forward[r] + backward[r] == best, then r = 0, then r = n (edlib.cpp,
// obtainAlignmentHirschberg: loop over the in-band rows first, the two boundary
// cells afterwards) - and both halves recursively.
void ObtainAlignment(const char* q, std::int64_t n, const char* t, std::int64_t m,
                     std::int64_t best, bool hirschberg, const int* pref,
                     std::string* out) {
  if (n == 0) { out->append(m, 'D'); return; }
  if (m == 0) { out->append(n, 'I'); return; }
  const std::int64_t blocks = (n + 63) / 64;
  const long long data_size = (2ll * 8 + 4) * blocks * m + 2ll * 4 * m;
  if (!hirschberg || data_size < 1024 * 1024) {
    Traceback(q, n, t, m, best, pref, out);
    return;
  }
  const std::int64_t L = m / 2, R = m - L;
  const std::vector<std::int32_t> fw = DistanceColumn(q, n, t, L, best);
  std::string rq(q, q + n), rt(t, t + m);
  std::reverse(rq.begin(), rq.end());
  std::reverse(rt.begin(), rt.end());
  const std::vector<std::int32_t> bwr = DistanceColumn(rq.data(), n, rt.data(), R, best);
  auto bw = [&](std::int64_t r) { return bwr[n - r]; };  // q[r, n) vs t[L, m)
  std::int64_t split = -1;
  for (std::int64_t r = 1; r <= n - 1; ++r) {
    if (fw[r] + bw(r) == best) { split = r; break; }
  }
  if (split < 0 && fw[0] + bw(0) == best) split = 0;
  if (split < 0 && fw[n] + bw(n) == best) split = n;
  if (split < 0) { Traceback(q, n, t, m, best, pref, out); return; }  // (cannot happen)
  ObtainAlignment(q, split, t, L, fw[split], hirschberg, pref, out);
  ObtainAlignment(q + split, n - split, t + L, R, bw(split), hirschberg, pref, out);
}

}  // namespace

// global edit distance by the same banded programme (band doubling)
std::int64_t GlobalDistance(const std::string& q, const std::string& t) {
  const std::int64_t n = q.size(), m = t.size();
  if (n == 0 || m == 0) return n + m;
  for (std::int64_t k = std::max<std::int64_t>(64, std::llabs(n - m) + 1);; k *= 2) {
    const std::int32_t d = DistanceColumn(q.data(), n, t.data(), m, k)[n];
    if (d <= k) return d;
  }
}

std::string GlobalAlignmentPath(const std::string& q, const std::string& t) {
  const std::int64_t n = q.size(), m = t.size();
  if (n == 0) return std::string(m, 'D');
  if (m == 0) return std::string(n, 'I');
  // tie preference of the traceback (experiment knob: ORC_NW_PREF=231 = up, left,
  // diagonal = edlib); ORC_NW_NO_HIRSCHBERG=1 disables the split
  int pref[3] = {2, 3, 1};
  if (const char* e = std::getenv("ORC_NW_PREF")) {
    for (int z = 0; z < 3 && e[z]; ++z) pref[z] = e[z] - '0';
  }
  const bool hirschberg = std::getenv("ORC_NW_NO_HIRSCHBERG") == nullptr;
  // the distance first (band doubling), like edlib
  std::int64_t best = -1;
  for (std::int64_t k = std::max<std::int64_t>(64, std::llabs(n - m) + 1);; k *= 2) {
    const std::int32_t d = DistanceColumn(q.data(), n, t.data(), m, k)[n];
    if (d <= k) { best = d; break; }
  }
  std::string path;
  path.reserve(n + m);
  ObtainAlignment(q.data(), n, t.data(), m, best, hirschberg, pref, &path);
  return path;
}

// racon Overlap::find_breaking_points (cigar walk): for every window boundary
// of the target (multiples of w, and the overlap end) the first and the
// one-past-last aligned (target, query) pair inside that window
std::vector<std::pair<std::uint32_t, std::uint32_t>> BreakingPoints(
    const std::string& path, std::uint32_t q_begin, std::uint32_t t_begin,
    std::uint32_t t_end, std::uint32_t w) {
  std::vector<std::int64_t> window_ends;
  for (std::uint32_t i = 0; i < t_end; i += w) {
    if (i > t_begin) window_ends.emplace_back(static_cast<std::int64_t>(i) - 1);
  }
  window_ends.emplace_back(static_cast<std::int64_t>(t_end) - 1);

  std::vector<std::pair<std::uint32_t, std::uint32_t>> dst;
  std::size_t wi = 0;
  bool found_first = false;
  std::pair<std::uint32_t, std::uint32_t> first{0, 0}, last{0, 0};
  std::int64_t q_ptr = static_cast<std::int64_t>(q_begin) - 1;
  std::int64_t t_ptr = static_cast<std::int64_t>(t_begin) - 1;
  auto close_window = [&]() {
    if (wi < window_ends.size() && t_ptr == window_ends[wi]) {
      if (found_first) {
        dst.emplace_back(first);
        dst.emplace_back(last);
      }
      found_first = false;
      ++wi;
    }
  };
  for (char op : path) {
    if (op == 'M') {
      ++q_ptr;
      ++t_ptr;
      if (!found_first) {
        found_first = true;
        first = {static_cast<std::uint32_t>(t_ptr), static_cast<std::uint32_t>(q_ptr)};
      }
      last = {static_cast<std::uint32_t>(t_ptr + 1), static_cast<std::uint32_t>(q_ptr + 1)};
      close_window();
    } else if (op == 'I') {
      ++q_ptr;
    } else {  // 'D'
      ++t_ptr;
      close_window();
    }
  }
  return dst;
}

}  // namespace racon
