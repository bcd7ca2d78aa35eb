// raven_b200 — RFC 1951 inflate of one BGZF member, and CRC-32 by slices: the one copy, called
// by FxInflateKernel (fastx.cu) and compiled for the host as well (tests/test_inflate_host.py
// runs it against zlib's raw inflate).
//
// It accepts the streams zlib's raw inflate accepts and rejects the ones it rejects:
// over-subscribed codes; incomplete codes, except a literal/length or distance code that is a
// single code of length 1 (or, for distances, no code at all); a missing end-of-block code;
// more than 286 length or 30 distance codes; a repeat code 16 with nothing to repeat and
// repeats past the code lengths; length symbols 286/287 and distance symbols 30/31 (only the
// fixed code can name them); block type 3; a stored block whose NLEN is not ~LEN; a distance
// before the start of the output. A member adds two rules of its own: the stream ends exactly
// at the end of its input, and the output never passes the member's ISIZE.
#pragma once

#include <cstdint>

#ifndef RVN_HD
#if defined(__CUDACC__)
#define RVN_HD __host__ __device__ __forceinline__
#else
#define RVN_HD inline
#endif
#endif

namespace rvn {

constexpr int kInfLitRoot = 10;   // literal/length codes up to 10 bits decode in one lookup
constexpr int kInfDistRoot = 8;   // distance codes up to 8 bits likewise
constexpr int kInfCodeRoot = 7;   // the code-length code (at most 7 bits): always one lookup
constexpr uint32_t kInfMaxOutput = 65536;  // a BGZF member's largest ISIZE

// The decode tables of one block. A root table entry is symbol << 4 | length; 0 names a code
// longer than the root (or none), which the canonical walk over count / sym decodes.
struct InfTables {
  uint16_t lit_table[1 << kInfLitRoot];
  uint16_t dist_table[1 << kInfDistRoot];
  uint16_t lit_count[16], lit_sym[288];
  uint16_t dist_count[16], dist_sym[32];
  uint8_t lens[320];  // the block's code lengths: literal/length, then distance
};

// LSB-first bit reader over in[0, n); bytes past n read as zero and Overrun() tells
struct InfBits {
  const uint8_t* in;
  uint64_t n, pos;
  uint64_t buf;
  int cnt;
  RVN_HD void Refill() {
    while (cnt <= 56) {
      buf |= static_cast<uint64_t>(pos < n ? in[pos] : 0u) << cnt;
      ++pos;
      cnt += 8;
    }
  }
  RVN_HD uint32_t Take(int k) {  // k <= cnt
    const uint32_t v = static_cast<uint32_t>(buf & ((1ULL << k) - 1));
    buf >>= k;
    cnt -= k;
    return v;
  }
  RVN_HD uint64_t Consumed() const { return pos * 8 - static_cast<uint64_t>(cnt); }
  RVN_HD bool Overrun() const { return Consumed() > n * 8; }
};

RVN_HD uint32_t InfReverse(uint32_t code, int len) {
#if defined(__CUDA_ARCH__)
  return __brev(code) >> (32 - len);
#else
  uint32_t r = 0;
  for (int i = 0; i < len; ++i) r |= ((code >> i) & 1u) << (len - 1 - i);
  return r;
#endif
}

// Canonical code of lens[0, n) into count / sym and the root table. `lengths`: the code-length
// code, which must be complete; otherwise zlib's rule for literal/length and distance codes.
RVN_HD bool InfBuild(const uint8_t* lens, int n, uint16_t* count, uint16_t* sym, uint16_t* table,
                     int root, bool lengths) {
  for (int l = 0; l < 16; ++l) count[l] = 0;
  for (int s = 0; s < n; ++s) ++count[lens[s]];
  count[0] = 0;
  int left = 1, max = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - count[l];
    if (left < 0) return false;  // over-subscribed
    if (count[l]) max = l;
  }
  for (int i = 0; i < (1 << root); ++i) table[i] = 0;
  if (max == 0) return !lengths;  // no codes: any symbol read from it is an error
  if (left > 0 && (lengths || max != 1)) return false;  // incomplete
  uint32_t code = 0;
  int j = 0;
  for (int l = 1; l < 16; ++l) {
    if (count[l]) {
      for (int s = 0; s < n; ++s) {
        if (lens[s] != l) continue;
        sym[j++] = static_cast<uint16_t>(s);
        if (l <= root) {
          const uint16_t e = static_cast<uint16_t>(s << 4 | l);
          for (uint32_t k = InfReverse(code, l); k < (1u << root); k += 1u << l) table[k] = e;
        }
        ++code;
      }
    }
    code <<= 1;
  }
  return true;
}

// one symbol (the buffer holds at least 15 bits); -1: no symbol has this code
RVN_HD int InfDecode(InfBits& b, const uint16_t* count, const uint16_t* sym,
                     const uint16_t* table, int root) {
  const uint32_t e = table[b.buf & ((1u << root) - 1)];
  if (e & 15) {
    b.Take(e & 15);
    return static_cast<int>(e >> 4);
  }
  int code = 0, first = 0, index = 0;
  uint64_t bits = b.buf;
  for (int l = 1; l < 16; ++l) {
    code |= static_cast<int>(bits & 1);
    bits >>= 1;
    const int c = count[l];
    if (code - c < first) {
      b.Take(l);
      return sym[index + (code - first)];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

// the order of the code-length code's lengths (RFC 1951 3.2.7), five bits each
RVN_HD int InfLengthOrder(int i) {
  constexpr uint64_t lo = 16ULL | 17ULL << 5 | 18ULL << 10 | 0ULL << 15 | 8ULL << 20 |
                          7ULL << 25 | 9ULL << 30 | 6ULL << 35 | 10ULL << 40 | 5ULL << 45;
  constexpr uint64_t hi = 11ULL | 4ULL << 5 | 12ULL << 10 | 3ULL << 15 | 13ULL << 20 |
                          2ULL << 25 | 14ULL << 30 | 1ULL << 35 | 15ULL << 40;
  return static_cast<int>(((i < 10 ? lo >> (5 * i) : hi >> (5 * (i - 10)))) & 31);
}

// Inflates the raw deflate stream in[0, n) into out[0, cap). Returns the output length, or -1
// when the stream is invalid, needs more than cap bytes of output or does not end at n.
RVN_HD int64_t Inflate(const uint8_t* in, uint64_t n, uint8_t* out, uint32_t cap, InfTables& t) {
  InfBits b{in, n, 0, 0, 0};
  uint32_t o = 0;
  for (;;) {
    b.Refill();
    if (b.Overrun()) return -1;
    const uint32_t last = b.Take(1), type = b.Take(2);
    if (type == 0) {  // stored
      b.Take(b.cnt & 7);
      const uint32_t len = b.Take(16), nlen = b.Take(16);
      if (len != (~nlen & 0xFFFFu) || len > cap - o) return -1;
      for (uint32_t i = 0; i < len; ++i) {
        if (b.cnt < 8) b.Refill();
        out[o++] = static_cast<uint8_t>(b.Take(8));
      }
      if (b.Overrun()) return -1;
    } else if (type == 3) {
      return -1;
    } else {
      int nlen, ndist;
      if (type == 1) {  // fixed
        nlen = 288;
        ndist = 32;
        for (int s = 0; s < 288; ++s) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        for (int s = 0; s < 32; ++s) t.lens[288 + s] = 5;
      } else {  // dynamic
        nlen = static_cast<int>(b.Take(5)) + 257;
        ndist = static_cast<int>(b.Take(5)) + 1;
        const int ncode = static_cast<int>(b.Take(4)) + 4;
        if (nlen > 286 || ndist > 30) return -1;
        uint8_t* cl = t.lens + 300;  // (19 lengths, free until the code lengths are read)
        for (int i = 0; i < 19; ++i) cl[i] = 0;
        b.Refill();
        for (int i = 0; i < ncode; ++i) cl[InfLengthOrder(i)] = static_cast<uint8_t>(b.Take(3));
        if (!InfBuild(cl, 19, t.lit_count, t.lit_sym, t.lit_table, kInfCodeRoot, true)) return -1;
        for (int have = 0; have < nlen + ndist;) {
          b.Refill();
          const int s = InfDecode(b, t.lit_count, t.lit_sym, t.lit_table, kInfCodeRoot);
          if (s < 0) return -1;
          if (s < 16) {
            t.lens[have++] = static_cast<uint8_t>(s);
            continue;
          }
          int rep;
          uint8_t v = 0;
          if (s == 16) {
            if (have == 0) return -1;
            v = t.lens[have - 1];
            rep = 3 + static_cast<int>(b.Take(2));
          } else if (s == 17) {
            rep = 3 + static_cast<int>(b.Take(3));
          } else {
            rep = 11 + static_cast<int>(b.Take(7));
          }
          if (have + rep > nlen + ndist) return -1;
          while (rep--) t.lens[have++] = v;
        }
        if (b.Overrun() || t.lens[256] == 0) return -1;
      }
      if (!InfBuild(t.lens, nlen, t.lit_count, t.lit_sym, t.lit_table, kInfLitRoot, false) ||
          !InfBuild(t.lens + nlen, ndist, t.dist_count, t.dist_sym, t.dist_table, kInfDistRoot,
                    false)) {
        return -1;
      }
      for (;;) {
        // one refill covers a length (15 + 5 bits) and its distance (15 + 13)
        if (b.cnt < 48) {
          b.Refill();
          if (b.Overrun()) return -1;
        }
        const int s = InfDecode(b, t.lit_count, t.lit_sym, t.lit_table, kInfLitRoot);
        if (s < 256) {
          if (s < 0 || o == cap) return -1;
          out[o++] = static_cast<uint8_t>(s);
          continue;
        }
        if (s == 256) break;
        const int i = s - 257;
        if (i >= 29) return -1;
        uint32_t len;
        if (i < 8) {
          len = 3 + i;
        } else if (i == 28) {
          len = 258;
        } else {
          const int e = (i >> 2) - 1;
          len = ((4u + (i & 3)) << e) + 3 + b.Take(e);
        }
        const int d = InfDecode(b, t.dist_count, t.dist_sym, t.dist_table, kInfDistRoot);
        if (d < 0 || d >= 30) return -1;
        uint32_t dist;
        if (d < 4) {
          dist = 1 + d;
        } else {
          const int e = (d >> 1) - 1;
          dist = ((2u + (d & 1)) << e) + 1 + b.Take(e);
        }
        if (dist > o || len > cap - o) return -1;
        for (uint32_t k = 0; k < len; ++k, ++o) out[o] = out[o - dist];
      }
    }
    if (last) break;
  }
  if (b.Overrun() || (b.Consumed() + 7) / 8 != n) return -1;
  return o;
}

// CRC-32 (the gzip trailer's), reflected, as a register without the initial and final
// inversion: crc32(D) = ~(InfCrcShift(~0, |D|) ^ InfCrcRaw(D)), and the raw register of a
// concatenation is the XOR of each part's register shifted past the bytes after it.
constexpr uint32_t kInfCrcPoly = 0xEDB88320u;

RVN_HD uint32_t InfCrcTableEntry(uint32_t i) {
  for (int k = 0; k < 8; ++k) i = i & 1 ? (i >> 1) ^ kInfCrcPoly : i >> 1;
  return i;
}

// a * b modulo the CRC polynomial, in the reflected representation (x^0 is bit 31)
RVN_HD uint32_t InfCrcMul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = b & 1 ? (b >> 1) ^ kInfCrcPoly : b >> 1;
  }
  return p;
}

// the raw register r moved past n zero bytes: r * x^(8n)
RVN_HD uint32_t InfCrcShift(uint32_t r, uint64_t n) {
  uint32_t x = 1u << 23;  // x^8
  for (; n; n >>= 1) {
    if (n & 1) r = InfCrcMul(x, r);
    x = InfCrcMul(x, x);
  }
  return r;
}

}  // namespace rvn
