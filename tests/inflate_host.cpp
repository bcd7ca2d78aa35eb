// Host build of raven_b200/csrc/inflate.cuh for tests/test_inflate_host.py.
#include <algorithm>
#include <vector>

#include "../raven_b200/csrc/inflate.cuh"

#define RVN_TEST_API extern "C" __attribute__((visibility("default")))

// Inflate of the raw deflate stream in[0, n) into out[0, cap): the output length, or -1.
RVN_TEST_API std::int64_t rvn_test_inflate(const std::uint8_t* in, std::uint64_t n,
                                           std::uint8_t* out, std::uint32_t cap) {
  rvn::InfTables t;
  return rvn::Inflate(in, n, out, cap, t);
}

// CRC-32 of data[0, n) as FxInflateKernel computes it: `slices` raw registers, each shifted
// past the bytes after its slice and XOR-ed, then the initial inversion shifted past all.
RVN_TEST_API std::uint32_t rvn_test_crc32(const std::uint8_t* data, std::uint32_t n,
                                          std::uint32_t slices) {
  std::vector<std::uint32_t> tab(256);
  for (std::uint32_t i = 0; i < 256; ++i) tab[i] = rvn::InfCrcTableEntry(i);
  const std::uint32_t slice = (n + slices - 1) / slices;
  std::uint32_t acc = 0;
  for (std::uint32_t s = 0; s < slices; ++s) {
    const std::uint32_t b = std::min(n, s * slice), e = std::min(n, b + slice);
    std::uint32_t r = 0;
    for (std::uint32_t i = b; i < e; ++i) r = tab[(r ^ data[i]) & 255] ^ (r >> 8);
    acc ^= rvn::InfCrcShift(r, n - e);
  }
  return ~(acc ^ rvn::InfCrcShift(0xFFFFFFFFu, n));
}
