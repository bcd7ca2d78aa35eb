// raven_b200 — rvn_reads_upload_files: FASTA / FASTQ files, plain or gzip, parsed and packed on
// the device into the context's read set.
//
// The files are read with zlib's gzread, as the drop-in bioparser reads them, on a thread of
// their own into two pinned slots, so that the next piece is read (or inflated) while the one
// before is copied and parsed. A chunk of text on the device is the tail of the chunk before
// (its first incomplete record) followed by new pieces. Per chunk:
//   lines     FxCountKernel / FxLineKernel: newline and non-space masks of 16-byte loads, scanned
//             per 4 KiB tile: every line's end and the non-space bytes before it (a line's
//             stripped length is a difference of two of those counts)
//   records   FASTA: the lines that begin with '>'. FASTQ: the drop-in's state machine
//             (fastq_parser.hpp) as a chain over lines: FxFastqNextKernel gives every line the
//             line after the record that would begin there (or an error, or "incomplete"), and
//             pointer doubling (FxChainKernel) marks the chain from the chunk's first line
//   measure   FxRecordKernel: per record its byte ranges, length and name
//   pack      FxPackKernel, a warp per record: the bases at their rank among the record's
//             non-space bytes, gathered in shared memory and written as whole words, the block
//             qualities likewise, the name
// Errors carry the message the reference's input loop prints (RavenExe/src/main.cc:258-299)
// for the first failing record in file order.
//
// A file whose first member is a whole BGZF member (the blocked gzip of the SAM specification,
// as bgzip and samtools write it) is read raw instead: the reader walks the member headers,
// whose BC subfields give each member's compressed size, and FxInflateKernel inflates the
// members side by side, a warp each, straight into the chunk text (inflate.cuh). At a member
// boundary, bytes that do not begin with 1f 8b end the file, as zlib ignores them; a gzip
// member that is not a whole BGZF member (another header, a truncated member, an ISIZE above
// 64 KiB) hands the rest of the file to zlib, opened at that member. Every other file is read
// with gzread as above.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>

#pragma nv_diag_suppress 68  // (the header's default arguments of -1 for uint32_t)
#include "../../include/biosoup/nucleic_acid.hpp"
#pragma nv_diag_default 68
#include "engine.cuh"
#include "inflate.cuh"

namespace rvn {

namespace {

constexpr int kFxThreads = 256;
constexpr int kFxWarps = kFxThreads / 32;
constexpr uint64_t kFxTile = kFxThreads * 16ULL;  // text bytes per CTA of the line index
constexpr uint64_t kFxPad = 16;                   // slack behind the text for 16-byte loads
constexpr uint64_t kFxDefaultChunk = 256ULL << 20;
constexpr int kFxHalves = 40;  // per warp: 16-base halves of the words being packed
constexpr unsigned long long kFxNoError = ~0ULL;

// biosoup::NucleotideCode of every byte (255: not a nucleotide)
__constant__ uint8_t c_fx_code[256];

// the 16 text bytes at p (16-aligned) below n, as masks: newlines, and bytes a line keeps after
// the drop-in's StripSpaces (not ' ', '\t', '\r', '\n')
__device__ __forceinline__ void FxMasks(const uint8_t* text, uint64_t p, uint64_t lo, uint64_t hi,
                                        uint32_t w[4], uint32_t* nl, uint32_t* keep) {
  *nl = *keep = 0;
  w[0] = w[1] = w[2] = w[3] = 0;
  if (p >= hi) return;
  const uint4 v = *reinterpret_cast<const uint4*>(text + p);
  w[0] = v.x;
  w[1] = v.y;
  w[2] = v.z;
  w[3] = v.w;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const uint32_t b = (w[j >> 2] >> (8 * (j & 3))) & 0xFFu;
    const bool in = p + j >= lo && p + j < hi;
    *nl |= static_cast<uint32_t>(in && b == '\n') << j;
    *keep |= static_cast<uint32_t>(in && b != '\n' && b != ' ' && b != '\t' && b != '\r') << j;
  }
}

__device__ __forceinline__ uint32_t FxByte(const uint32_t w[4], int j) {
  return (w[j >> 2] >> (8 * (j & 3))) & 0xFFu;
}

// newlines << 16 | kept bytes of a tile (each at most 4096)
__global__ void __launch_bounds__(kFxThreads)
FxCountKernel(const uint8_t* __restrict__ text, uint64_t n, uint32_t* __restrict__ tile_nl,
              uint32_t* __restrict__ tile_keep) {
  __shared__ uint32_t sm[33];
  const uint64_t p = blockIdx.x * kFxTile + threadIdx.x * 16ULL;
  uint32_t w[4], nl, keep;
  FxMasks(text, p, 0, n, w, &nl, &keep);
  uint32_t total;
  BlockExclusiveSum<uint32_t, kFxThreads>((__popc(nl) << 16) | __popc(keep), sm, &total);
  if (threadIdx.x == 0) {
    tile_nl[blockIdx.x] = total >> 16;
    tile_keep[blockIdx.x] = total & 0xFFFFu;
  }
}

// line k ends at line_end[k] (its newline) with keep_at[k] kept bytes before that
__global__ void __launch_bounds__(kFxThreads)
FxLineKernel(const uint8_t* __restrict__ text, uint64_t n, const uint64_t* __restrict__ nl_off,
             const uint64_t* __restrict__ keep_off, uint64_t* __restrict__ line_end,
             uint64_t* __restrict__ keep_at) {
  __shared__ uint32_t sm[33];
  const uint64_t p = blockIdx.x * kFxTile + threadIdx.x * 16ULL;
  uint32_t w[4], nl, keep;
  FxMasks(text, p, 0, n, w, &nl, &keep);
  uint32_t total;
  const uint32_t ex =
      BlockExclusiveSum<uint32_t, kFxThreads>((__popc(nl) << 16) | __popc(keep), sm, &total);
  uint64_t k = nl_off[blockIdx.x] + (ex >> 16);
  const uint64_t k0 = keep_off[blockIdx.x] + (ex & 0xFFFFu);
  while (nl) {
    const int j = __ffs(nl) - 1;
    nl &= nl - 1;
    line_end[k] = p + j;
    keep_at[k] = k0 + __popc(keep & ((1u << j) - 1));
    ++k;
  }
}

// the last line of the last chunk may lack its newline: it ends at n
__global__ void FxFinishLinesKernel(const uint8_t* text, uint64_t n, int final_chunk,
                                    const uint64_t* n_nl, const uint64_t* keep_total,
                                    uint64_t* line_end, uint64_t* keep_at, uint64_t* n_lines) {
  uint64_t k = *n_nl;
  if (final_chunk && n > 0 && text[n - 1] != '\n') {
    line_end[k] = n;
    keep_at[k] = *keep_total;
    ++k;
  }
  *n_lines = k;
}

struct FxLines {
  const uint8_t* text;
  uint64_t n;
  const uint64_t* end;
  const uint64_t* keep;
  uint64_t count;
  __device__ __forceinline__ uint64_t Start(uint64_t k) const {
    return k ? min(end[k - 1] + 1, n) : 0;
  }
  __device__ __forceinline__ uint64_t Keep0(uint64_t k) const { return k ? keep[k - 1] : 0; }
  // length without the trailing '\r' (the drop-in's ReadLine)
  __device__ __forceinline__ uint64_t Length(uint64_t k) const {
    const uint64_t s = Start(k), e = end[k];
    return e - s - (e > s && text[e - 1] == '\r' ? 1 : 0);
  }
  __device__ __forceinline__ uint32_t First(uint64_t k) const {
    const uint64_t s = Start(k);
    return s < end[k] ? text[s] : 0u;
  }
};

__global__ void FxFastaFlagKernel(FxLines L, uint32_t* __restrict__ flag) {
  for (uint64_t k = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; k < L.count;
       k += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    flag[k] = L.First(k) == '>';
  }
}

__global__ void FxScatterKernel(const uint32_t* __restrict__ flag, const uint64_t* __restrict__ off,
                                uint64_t count, uint32_t* __restrict__ rec_line) {
  for (uint64_t k = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; k < count;
       k += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    if (flag[k]) rec_line[off[k]] = static_cast<uint32_t>(k);
  }
}

// FASTA: a line before the first header that is not empty (fasta_parser.hpp: !in_record)
__global__ void FxFastaLeadKernel(FxLines L, const uint64_t* n_hdr, const uint32_t* rec_line,
                                  unsigned long long* err_key) {
  const uint64_t lead = *n_hdr ? rec_line[0] : L.count;
  for (uint64_t k = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; k < lead;
       k += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    if (L.Length(k) > 0) atomicMin(err_key, 0ULL);
  }
}

// FASTA cut: out[0] complete records, out[1] the first byte of the tail
__global__ void FxFastaCutKernel(FxLines L, int final_chunk, const uint64_t* n_hdr,
                                 const uint32_t* rec_line, uint64_t* out) {
  const uint64_t h = *n_hdr;
  if (final_chunk) {
    out[0] = h;
    out[1] = L.n;
  } else {
    out[0] = h ? h - 1 : 0;
    out[1] = h ? L.Start(rec_line[h - 1]) : L.Start(L.count);
  }
}

// FASTQ: where the record that would begin at line v ends. Nodes are the lines, then END
// (= count: past the last line), ERR (a record the drop-in rejects) and INC (a record the
// chunk does not hold whole); the three are their own successors. plus[v] / qual_last[v]: the
// record's '+' line and last quality line.
__global__ void FxFastqNextKernel(FxLines L, int final_chunk, uint32_t* __restrict__ next,
                                  uint32_t* __restrict__ plus, uint32_t* __restrict__ qual_last) {
  const uint64_t END = L.count, ERR = L.count + 1, INC = L.count + 2;
  for (uint64_t v = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; v < L.count + 3;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    uint64_t to;
    if (v >= END) {
      to = v;
    } else if (L.Length(v) == 0) {
      to = v + 1;  // blank lines before a header are skipped
    } else if (L.First(v) != '@') {
      to = ERR;
    } else {
      uint64_t p = v + 1;
      while (p < L.count && L.First(p) != '+') ++p;
      if (p == L.count) {
        to = final_chunk ? ERR : INC;
      } else {
        const uint64_t seq = L.Keep0(p) - L.keep[v];
        const uint64_t target = L.keep[p] + seq;
        // the first line at which the stripped quality reaches the sequence's length
        uint64_t lo = p + 1, hi = L.count;
        while (lo < hi) {
          const uint64_t mid = (lo + hi) >> 1;
          if (L.keep[mid] >= target) hi = mid; else lo = mid + 1;
        }
        if (seq == 0) {
          to = ERR;
        } else if (lo == L.count) {
          to = final_chunk ? ERR : INC;
        } else if (L.keep[lo] != target) {
          to = ERR;  // more quality than sequence
        } else {
          to = lo + 1;
          plus[v] = static_cast<uint32_t>(p);
          qual_last[v] = static_cast<uint32_t>(lo);
        }
      }
    }
    next[v] = static_cast<uint32_t>(to);
  }
}

// one round of pointer doubling: a marked node marks its 2^round-th successor (the chain
// from node 0 is marked up to 2^(round+1) steps), and jump_out = jump_in o jump_in
__global__ void FxChainKernel(const uint32_t* __restrict__ jump_in, uint32_t* __restrict__ jump_out,
                              uint8_t* mark, uint64_t nodes) {
  for (uint64_t v = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; v < nodes;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t j = jump_in[v];
    if (mark[v]) mark[j] = 1;
    jump_out[v] = jump_in[j];
  }
}

// FASTQ records: the marked lines that begin a whole record; stop: the marked line whose
// record is rejected or incomplete
__global__ void FxFastqFlagKernel(FxLines L, const uint32_t* __restrict__ next,
                                  const uint8_t* __restrict__ mark, uint32_t* __restrict__ flag,
                                  unsigned long long* stop) {
  for (uint64_t v = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; v < L.count;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const bool on = mark[v] != 0;
    flag[v] = on && next[v] <= L.count && L.Length(v) > 0;
    if (on && next[v] > L.count) atomicMin(stop, static_cast<unsigned long long>(v));
  }
}

// FASTQ cut: out[0] records, out[1] the first byte of the tail, out[2] 1 if the chain ended
// in a rejected record
__global__ void FxFastqCutKernel(FxLines L, const uint64_t* n_rec, const uint8_t* mark,
                                 const unsigned long long* stop, uint64_t* out) {
  out[0] = *n_rec;
  out[1] = mark[L.count + 2] ? L.Start(*stop) : L.Start(L.count);
  out[2] = mark[L.count + 1] ? 1 : 0;
}

struct FxRec {
  uint64_t seq_b, seq_e, qual_b, qual_e, name_pos;
  uint32_t len, name_len;
};

// per record: byte ranges, length, name (the header up to its first ' ' or '\t'); a record
// without a name or bases is rejected, one of 2^31 bases or more is over the limit
__global__ void FxRecordKernel(FxLines L, int fastq, const uint32_t* __restrict__ rec_line,
                               uint64_t n_rec, uint64_t n_hdr, const uint32_t* __restrict__ plus,
                               const uint32_t* __restrict__ qual_last, FxRec* __restrict__ rec,
                               uint32_t* __restrict__ n_words, uint32_t* __restrict__ n_bq,
                               uint32_t* __restrict__ n_name, unsigned long long* err_key,
                               unsigned long long* over_limit) {
  for (uint64_t r = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; r < n_rec;
       r += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t h = rec_line[r];
    FxRec x;
    uint64_t len;
    x.seq_b = L.end[h] + 1;
    if (fastq) {
      const uint32_t p = plus[h], q = qual_last[h];
      x.seq_e = L.Start(p);
      x.qual_b = L.end[p] + 1;
      x.qual_e = min(L.end[q] + 1, L.n);
      len = L.Keep0(p) - L.keep[h];
    } else {
      const uint64_t hn = r + 1 < n_hdr ? rec_line[r + 1] : L.count;
      x.seq_e = L.Start(hn);
      x.qual_b = x.qual_e = 0;
      len = L.Keep0(hn) - L.keep[h];
    }
    x.seq_b = min(x.seq_b, x.seq_e);
    const uint64_t s = L.Start(h) + 1, e = L.Start(h) + L.Length(h);
    uint64_t t = s;
    while (t < e && L.text[t] != ' ' && L.text[t] != '\t') ++t;
    x.name_pos = s;
    x.name_len = static_cast<uint32_t>(t - s);
    if (x.name_len == 0 || len == 0) atomicMin(err_key, 2ULL * (r + 1));
    if (len >= (1ULL << 31)) {
      atomicMax(over_limit, 1ULL);
      len = 0;  // (not packed: the call fails)
    }
    x.len = static_cast<uint32_t>(len);
    rec[r] = x;
    n_words[r] = static_cast<uint32_t>((len + 31) >> 5);
    n_bq[r] = fastq ? static_cast<uint32_t>((len + 63) >> 6) : 0;
    n_name[r] = x.name_len;
  }
}

// warp-wide exclusive sum; *total: the warp's sum
__device__ __forceinline__ uint32_t FxWarpExclusive(uint32_t v, uint32_t* total) {
  const int lane = threadIdx.x & 31;
  uint32_t incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  *total = __shfl_sync(0xffffffffu, incl, 31);
  return incl - v;
}

// A warp per record. Each lane takes 16 bytes of the record's sequence (then quality) lines
// per step; a byte's rank among the record's kept bytes is the warp's count before it. Codes
// are OR-ed into 16-base halves in shared memory (at most two per lane and step) and whole
// words leave as coalesced stores; the last, partial word moves to the front. Qualities: the
// sums of 64-character blocks in shared memory, each whole block's mean stored as a byte.
__global__ void __launch_bounds__(kFxThreads)
FxPackKernel(const uint8_t* __restrict__ text, const FxRec* __restrict__ rec, uint64_t n_rec,
             const uint64_t* __restrict__ woff, const uint64_t* __restrict__ bq_off,
             const uint64_t* __restrict__ name_off, uint64_t* __restrict__ words,
             uint8_t* __restrict__ bq, char* __restrict__ names, unsigned long long* err_key) {
  __shared__ uint8_t code[256];
  __shared__ uint32_t stage[kFxWarps][kFxHalves];
  for (int i = threadIdx.x; i < 256; i += kFxThreads) code[i] = c_fx_code[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  uint32_t* buf = stage[threadIdx.x >> 5];
  for (uint64_t r = blockIdx.x * static_cast<uint64_t>(kFxWarps) + (threadIdx.x >> 5); r < n_rec;
       r += static_cast<uint64_t>(gridDim.x) * kFxWarps) {
    const FxRec x = rec[r];
    for (uint32_t i = lane; i < x.name_len; i += 32) {
      names[name_off[r] + i] = static_cast<char>(text[x.name_pos + i]);
    }
    if (x.len == 0) continue;
    // bases
    for (int i = lane; i < kFxHalves; i += 32) buf[i] = 0;
    __syncwarp();
    uint64_t* out = words + woff[r];
    uint32_t carry = 0;
    bool bad = false;
    for (uint64_t pos = x.seq_b & ~15ULL; pos < x.seq_e; pos += 512) {
      const uint64_t p = pos + lane * 16ULL;
      uint32_t w[4], nl, keep;
      FxMasks(text, p, x.seq_b, x.seq_e, w, &nl, &keep);
      uint32_t total;
      const uint32_t rank = carry + FxWarpExclusive(__popc(keep), &total);
      uint32_t v = 0;
      int k = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (keep >> j & 1) {
          const uint32_t c = code[FxByte(w, j)];
          bad |= c > 3;
          v |= (c & 3) << (2 * k);
          ++k;
        }
      }
      if (k) {
        const uint64_t t = static_cast<uint64_t>(v) << (2 * (rank & 15));
        atomicOr(&buf[rank >> 4], static_cast<uint32_t>(t));
        if (t >> 32) atomicOr(&buf[(rank >> 4) + 1], static_cast<uint32_t>(t >> 32));
      }
      __syncwarp();
      const uint32_t filled = carry + total, whole = filled >> 5;
      for (uint32_t i = lane; i < whole; i += 32) {
        out[i] = buf[2 * i] | static_cast<uint64_t>(buf[2 * i + 1]) << 32;
      }
      const uint32_t keep0 = buf[2 * whole], keep1 = buf[2 * whole + 1];
      __syncwarp();
      for (int i = lane; i < kFxHalves; i += 32) buf[i] = i == 0 ? keep0 : i == 1 ? keep1 : 0;
      __syncwarp();
      out += whole;
      carry = filled & 31;
    }
    if (carry && lane == 0) out[0] = buf[0] | static_cast<uint64_t>(buf[1]) << 32;
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(err_key, 2ULL * (r + 1) + 1);
    __syncwarp();
    if (x.qual_e <= x.qual_b) continue;
    // block qualities: NucleicAcid's sum of (char - '!') as uint32 over 64 characters, over
    // the block's length, truncated to a byte (nucleic_acid.hpp)
    for (int i = lane; i < kFxHalves; i += 32) buf[i] = 0;
    __syncwarp();
    uint8_t* qo = bq + bq_off[r];
    carry = 0;
    for (uint64_t pos = x.qual_b & ~15ULL; pos < x.qual_e; pos += 512) {
      const uint64_t p = pos + lane * 16ULL;
      uint32_t w[4], nl, keep;
      FxMasks(text, p, x.qual_b, x.qual_e, w, &nl, &keep);
      uint32_t total;
      const uint32_t rank = carry + FxWarpExclusive(__popc(keep), &total);
      const uint32_t split = ((rank >> 6) + 1) * 64 - rank;  // this lane's chars in rank's block
      uint32_t s0 = 0, s1 = 0;
      uint32_t k = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (keep >> j & 1) {
          const uint32_t q = static_cast<uint32_t>(static_cast<int>(
                                 static_cast<int8_t>(FxByte(w, j))) - '!');
          if (k < split) s0 += q; else s1 += q;
          ++k;
        }
      }
      if (k) {
        atomicAdd(&buf[rank >> 6], s0);
        if (k > split) atomicAdd(&buf[(rank >> 6) + 1], s1);
      }
      __syncwarp();
      const uint32_t filled = carry + total, whole = filled >> 6;
      for (uint32_t i = lane; i < whole; i += 32) qo[i] = static_cast<uint8_t>(buf[i] / 64);
      const uint32_t keep0 = buf[whole];
      __syncwarp();
      for (int i = lane; i < kFxHalves; i += 32) buf[i] = i == 0 ? keep0 : 0;
      __syncwarp();
      qo += whole;
      carry = filled & 63;
    }
    if (carry && lane == 0) qo[0] = static_cast<uint8_t>(buf[0] / carry);
    __syncwarp();
  }
}

constexpr int kFxInfWarps = 8;  // members per CTA of FxInflateKernel

// one BGZF member of a piece: its deflate data in the piece's compressed bytes, its text in
// the piece's text, and its trailer
struct FxMember {
  uint64_t in_off, out_off;
  uint32_t in_len, isize, crc, pad;
};

// A warp per member. Lane 0 inflates it (inflate.cuh, tables in shared memory) into the text;
// then each lane takes the CRC-32 of a 32nd of the output, and the registers are shifted past
// the bytes after their slices and XOR-ed. A member that fails, or whose CRC or ISIZE differ
// from its trailer, records its index in *bad. (The bound of 4 CTAs per SM keeps ptxas from
// spilling; shared memory allows 7.)
__global__ void __launch_bounds__(kFxInfWarps * 32, 4)
FxInflateKernel(const uint8_t* __restrict__ comp, const FxMember* __restrict__ mem,
                uint32_t n_mem, uint8_t* text, unsigned* bad) {
  __shared__ InfTables tabs[kFxInfWarps];
  __shared__ uint32_t crc_tab[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) crc_tab[i] = InfCrcTableEntry(i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t m = blockIdx.x * kFxInfWarps + warp; m < n_mem; m += gridDim.x * kFxInfWarps) {
    const FxMember x = mem[m];
    uint8_t* out = text + x.out_off;
    int got = 0;  // (an output length of at most 2^16, or -1)
    if (lane == 0) {
      got = static_cast<int>(Inflate(comp + x.in_off, x.in_len, out, x.isize, tabs[warp]));
    }
    const bool whole = __shfl_sync(0xffffffffu, got, 0) == static_cast<int>(x.isize);
    __syncwarp();
    const uint32_t n = whole ? x.isize : 0;
    const uint32_t slice = (n + 31) / 32;
    const uint32_t b = min(n, lane * slice), e = min(n, b + slice);
    uint32_t r = 0;
    for (uint32_t i = b; i < e; ++i) r = crc_tab[(r ^ out[i]) & 255] ^ (r >> 8);
    r = InfCrcShift(r, n - e);
#pragma unroll
    for (int d = 16; d; d >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, d);
    if (lane == 0 && (!whole || ~(r ^ InfCrcShift(0xFFFFFFFFu, n)) != x.crc)) {
      atomicMin(bad, m);
    }
  }
}

unsigned Grid(uint64_t n, const Ctx& c) {
  return static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>((n + 255) / 256,
                                                                          c.sms * 16ULL)));
}

bool IsSuffix(const std::string& s, const char* suff) {
  const size_t n = std::strlen(suff);
  return s.size() >= n && s.compare(s.size() - n, n, suff) == 0;
}

const char* kFastaInvalid = "[bioparser::FastaParser] error: invalid file format";
const char* kFastqInvalid = "[bioparser::FastqParser] error: invalid file format";
const char* kNotNucleotide = "[biosoup::NucleicAcid::NucleicAcid] error: not a nucleotide";

constexpr uint32_t kBgzfMaxMember = 65536;  // BSIZE + 1 of a BGZF member is at most 2^16

// A file read raw, for its BGZF members: a window of preads, and Member() that finds the whole
// member at an offset from its header alone.
class BgzfFile {
 public:
  explicit BgzfFile(const std::string& path) : fd_(open(path.c_str(), O_RDONLY)) {
    struct stat st;
    if (fd_ >= 0 && fstat(fd_, &st) == 0) size_ = static_cast<uint64_t>(st.st_size);
  }
  ~BgzfFile() {
    if (fd_ >= 0) close(fd_);
  }
  BgzfFile(const BgzfFile&) = delete;
  BgzfFile& operator=(const BgzfFile&) = delete;
  bool ok() const { return fd_ >= 0; }
  uint64_t size() const { return size_; }
  // bytes [pos, pos + n) of the file (n <= kBgzfMaxMember), or null when fewer can be read
  const uint8_t* At(uint64_t pos, uint64_t n) {
    if (pos >= lo_ && pos + n <= hi_) return win_.data() + (pos - lo_);
    // the window grows from 64 KiB to 4 MiB, so a first look at a file that is not BGZF
    // reads little
    fill_ = std::min<uint64_t>(fill_ * 2, 4ULL << 20);
    const uint64_t want = pos < size_ ? std::min(std::max(n, fill_), size_ - pos) : 0;
    if (win_.size() < want) win_.resize(want);
    uint64_t got = 0;
    while (got < want) {
      const ssize_t r = pread(fd_, win_.data() + got, want - got, static_cast<off_t>(pos + got));
      if (r <= 0) break;
      got += static_cast<uint64_t>(r);
    }
    lo_ = pos;
    hi_ = pos + got;
    return got >= n ? win_.data() : nullptr;
  }
  // The length of the whole BGZF member at pos (its deflate data relative to pos, ISIZE and
  // CRC in *m), or 0 when the bytes there are not one: the header 1f 8b 08 with FLG = FEXTRA
  // alone and a BC subfield of length 2 among well-formed subfields, BSIZE + 1 bytes inside
  // the file, and an ISIZE of at most 64 KiB.
  uint32_t Member(uint64_t pos, FxMember* m) {
    const uint64_t left = pos < size_ ? size_ - pos : 0;
    const uint64_t span = std::min<uint64_t>(left, kBgzfMaxMember);
    if (span < 18) return 0;
    const uint8_t* h = At(pos, span);
    if (!h || h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || h[3] != 4) return 0;
    const uint32_t xend = 12 + (h[10] | h[11] << 8);
    if (xend + 8 > span) return 0;
    uint32_t total = 0, q = 12;
    while (q + 4 <= xend) {
      const uint32_t slen = h[q + 2] | h[q + 3] << 8;
      if (q + 4 + slen > xend) return 0;
      if (h[q] == 'B' && h[q + 1] == 'C' && slen == 2 && total == 0) {
        total = (h[q + 4] | h[q + 5] << 8) + 1;
      }
      q += 4 + slen;
    }
    if (q != xend || total < xend + 8 || total > span) return 0;
    const uint8_t* t = h + total - 8;
    m->crc = t[0] | t[1] << 8 | t[2] << 16 | static_cast<uint32_t>(t[3]) << 24;
    m->isize = t[4] | t[5] << 8 | t[6] << 16 | static_cast<uint32_t>(t[7]) << 24;
    if (m->isize > kInfMaxOutput) return 0;
    m->in_off = xend;
    m->in_len = total - xend - 8;
    m->out_off = 0;
    m->pad = 0;
    return total;
  }

 private:
  int fd_;
  uint64_t size_ = 0;
  std::vector<uint8_t> win_;
  uint64_t lo_ = 0, hi_ = 0, fill_ = 32 << 10;
};

// One file, read ahead into two pinned slots on a thread of its own: as text with gzread, or,
// while bgzf is set, as whole BGZF members (a piece then holds compressed bytes and the
// member table, and ends once its members' ISIZEs reach the piece size). Take(i) waits for
// slot i (the pieces alternate between the slots), Release(i) hands it back.
class FxReader {
 public:
  FxReader(gzFile f, std::unique_ptr<BgzfFile> bgzf, const std::string& path,
           PinBuf<uint8_t>* slots, uint64_t piece)
      : f_(f), bgzf_(std::move(bgzf)), path_(path), slots_(slots), piece_(piece) {
    thread_ = std::thread([this] { Run(); });
  }
  ~FxReader() {
    {
      std::lock_guard<std::mutex> l(m_);
      stop_ = true;
    }
    cv_.notify_all();
    thread_.join();
    if (f_) gzclose(f_);
  }
  struct Piece {
    uint64_t len;      // text bytes (once inflated)
    uint64_t raw;      // compressed bytes in the slot (0: the slot holds the text)
    uint32_t members;  // BGZF members in the slot
    bool last;
    bool failed;
  };
  Piece Take(int i) {
    std::unique_lock<std::mutex> l(m_);
    cv_.wait(l, [&] { return full_[i]; });
    return piece_of_[i];
  }
  // the member table of the piece in slot i, until Release(i)
  const std::vector<FxMember>& Members(int i) const { return members_[i]; }
  void Release(int i) {
    {
      std::lock_guard<std::mutex> l(m_);
      full_[i] = false;
    }
    cv_.notify_all();
  }

 private:
  void Run() {
    for (int i = 0;; i ^= 1) {
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return stop_ || !full_[i]; });
        if (stop_) return;
      }
      Piece p{0, 0, 0, false, false};
      if (bgzf_) ReadMembers(i, &p);
      if (!bgzf_ && !p.last && p.members == 0) ReadText(i, &p);
      {
        std::lock_guard<std::mutex> l(m_);
        piece_of_[i] = p;
        full_[i] = true;
      }
      cv_.notify_all();
      if (p.last) return;
    }
  }
  void ReadText(int i, Piece* p) {
    uint8_t* dst = slots_[i].get();
    while (p->len < piece_) {
      const unsigned want = static_cast<unsigned>(std::min<uint64_t>(piece_ - p->len, 1u << 30));
      const int got = gzread(f_, dst + p->len, want);
      if (got < 0) {
        p->failed = p->last = true;
        return;
      }
      if (got == 0) {
        p->last = true;
        return;
      }
      p->len += static_cast<uint64_t>(got);
    }
  }
  // whole members at pos_, until the piece's text reaches piece_ or its slot is full
  void ReadMembers(int i, Piece* p) {
    std::vector<FxMember>& mem = members_[i];
    mem.clear();
    uint8_t* dst = slots_[i].get();
    while (p->len < piece_) {
      const uint64_t left = bgzf_->size() - pos_;
      const uint8_t* h = left ? bgzf_->At(pos_, std::min<uint64_t>(left, 2)) : nullptr;
      if (left && !h) {
        p->failed = p->last = true;
        return;
      }
      // the end of the file, or bytes after the last member that zlib ignores
      if (left < 2 || h[0] != 0x1f || h[1] != 0x8b) {
        p->last = true;
        return;
      }
      FxMember m;
      const uint32_t total = bgzf_->Member(pos_, &m);
      if (total == 0) {
        HandToZlib(p);
        return;
      }
      if (p->raw + total > slots_[i].cap) return;
      std::memcpy(dst + p->raw, bgzf_->At(pos_, total), total);
      m.in_off += p->raw;
      m.out_off = p->len;
      mem.push_back(m);
      p->raw += total;
      p->len += m.isize;
      ++p->members;
      pos_ += total;
    }
  }
  // zlib reads the rest of the file from the gzip member at pos_, with the multi-member
  // rules the whole-file route has
  void HandToZlib(Piece* p) {
    const int fd = open(path_.c_str(), O_RDONLY);
    if (fd >= 0 && lseek(fd, static_cast<off_t>(pos_), SEEK_SET) == static_cast<off_t>(pos_)) {
      f_ = gzdopen(fd, "rb");
    }
    if (!f_) {
      if (fd >= 0) close(fd);
      p->failed = p->last = true;
      return;
    }
    gzbuffer(f_, 1 << 20);
    bgzf_.reset();
  }
  gzFile f_;
  std::unique_ptr<BgzfFile> bgzf_;
  uint64_t pos_ = 0;
  std::string path_;
  PinBuf<uint8_t>* slots_;
  uint64_t piece_;
  std::vector<FxMember> members_[2];
  std::mutex m_;
  std::condition_variable cv_;
  bool full_[2] = {false, false};
  bool stop_ = false;
  Piece piece_of_[2];
  std::thread thread_;
};

// the parsed set while it is being built: its words are in c.d_words
struct FxSet {
  uint64_t words = 0;
  std::vector<uint32_t> lens;
  std::vector<uint8_t> bq;
  std::vector<uint64_t> bq_off{0};
  std::string names;
  std::vector<uint64_t> name_off{0};
};

// device scratch of one call
struct FxScratch {
  DevBuf<uint8_t> text[2];
  DevBuf<uint32_t> tile_nl, tile_keep, flag, rec_line, next, jump[2], plus, qual_last, n_words,
      n_bq, n_name;
  DevBuf<uint64_t> nl_off, keep_off, line_end, keep_at, flag_off, woff, bq_off, name_off, scalars;
  DevBuf<uint8_t> mark, bq;
  DevBuf<char> names;
  DevBuf<FxRec> rec;
  DevBuf<uint8_t> comp;
  DevBuf<FxMember> members;
  DevBuf<unsigned> bad;
  float read_ms = 0;
};

// room for `need` words in c.d_words (the words before `keep` stay)
void GrowWords(Ctx& c, uint64_t need, uint64_t keep) {
  if (need <= c.d_words.cap) return;
  size_t free_b = 0, total_b = 0;
  RVN_CUDA(cudaMemGetInfo(&free_b, &total_b));
  // the new buffer (with DevBuf's slack of 1/16) is allocated beside the old one
  const uint64_t room = free_b / sizeof(uint64_t) * 15 / 16;
  if (need + 64 > room) {
    throw LimitError("the packed bases of the parsed reads (" +
                     std::to_string(need * sizeof(uint64_t)) + " bytes) do not fit the device (" +
                     std::to_string(free_b) + " bytes free)");
  }
  c.d_words.reserve_keep(std::max(need, std::min(2 * c.d_words.cap, room - 64)), keep, c.stream);
}

// Parses the chunk text[0, n) (final: the file ends with it) and appends its complete records
// to the set. Returns the first byte of the tail (the first record the chunk does not hold
// whole; n when there is none).
uint64_t ParseChunk(Ctx& c, FxScratch& s, const uint8_t* text, uint64_t n, bool final_chunk,
                    bool fastq, FxSet& set, const std::string& path) {
  if (n == 0) return 0;
  TimerBegin(c, "fastx_parse");
  const uint64_t tiles = (n + kFxTile - 1) / kFxTile;
  uint32_t* tnl = s.tile_nl.reserve(tiles);
  uint32_t* tkeep = s.tile_keep.reserve(tiles);
  uint64_t* nl_off = s.nl_off.reserve(tiles + 1);
  uint64_t* keep_off = s.keep_off.reserve(tiles + 1);
  uint64_t* sc = s.scalars.reserve(8);
  auto* err_key = reinterpret_cast<unsigned long long*>(sc + 4);
  auto* over = reinterpret_cast<unsigned long long*>(sc + 5);
  auto* stop = reinterpret_cast<unsigned long long*>(sc + 6);
  RVN_CUDA(cudaMemsetAsync(sc + 4, 0xFF, 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(sc + 5, 0, 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(sc + 6, 0xFF, 8, c.stream));
  FxCountKernel<<<static_cast<unsigned>(tiles), kFxThreads, 0, c.stream>>>(text, n, tnl, tkeep);
  RVN_LAUNCH_CHECK();
  ++c.launches;
  ExclusiveScanU32(c, tnl, nl_off, tiles);
  ExclusiveScanU32(c, tkeep, keep_off, tiles);
  const uint64_t n_nl = ReadU64(c, nl_off + tiles);
  uint64_t* line_end = s.line_end.reserve(n_nl + 1);
  uint64_t* keep_at = s.keep_at.reserve(n_nl + 1);
  FxLineKernel<<<static_cast<unsigned>(tiles), kFxThreads, 0, c.stream>>>(text, n, nl_off, keep_off,
                                                                         line_end, keep_at);
  FxFinishLinesKernel<<<1, 1, 0, c.stream>>>(text, n, final_chunk ? 1 : 0, nl_off + tiles,
                                             keep_off + tiles, line_end, keep_at, sc);
  RVN_LAUNCH_CHECK();
  c.launches += 2;
  const uint64_t count = ReadU64(c, sc);
  if (count + 3 >= 0xFFFFFFFFULL) throw LimitError("a chunk of 2^32 lines or more");
  const FxLines L{text, n, line_end, keep_at, count};
  uint32_t* flag = s.flag.reserve(count + 1);
  uint64_t* flag_off = s.flag_off.reserve(count + 1);
  uint32_t* rec_line = s.rec_line.reserve(count + 1);
  uint32_t* plus = nullptr;
  uint32_t* qual_last = nullptr;
  const unsigned g = Grid(count + 3, c);
  uint64_t cut[3] = {0, n, 0};
  uint64_t n_hdr = 0;
  if (!fastq) {
    FxFastaFlagKernel<<<g, 256, 0, c.stream>>>(L, flag);
    RVN_LAUNCH_CHECK();
    ExclusiveScanU32(c, flag, flag_off, count);
    FxScatterKernel<<<g, 256, 0, c.stream>>>(flag, flag_off, count, rec_line);
    FxFastaLeadKernel<<<g, 256, 0, c.stream>>>(L, flag_off + count, rec_line, err_key);
    FxFastaCutKernel<<<1, 1, 0, c.stream>>>(L, final_chunk ? 1 : 0, flag_off + count, rec_line, sc);
    RVN_LAUNCH_CHECK();
    c.launches += 4;
    cut[0] = ReadU64(c, sc, sc + 1, &cut[1]);
    n_hdr = ReadU64(c, flag_off + count);
  } else {
    const uint64_t nodes = count + 3;
    uint32_t* next = s.next.reserve(nodes);
    uint32_t* ja = s.jump[0].reserve(nodes);
    uint32_t* jb = s.jump[1].reserve(nodes);
    plus = s.plus.reserve(count + 1);
    qual_last = s.qual_last.reserve(count + 1);
    uint8_t* mark = s.mark.reserve(nodes);
    FxFastqNextKernel<<<g, 256, 0, c.stream>>>(L, final_chunk ? 1 : 0, next, plus, qual_last);
    RVN_CUDA(cudaMemsetAsync(mark, 0, nodes, c.stream));
    RVN_CUDA(cudaMemsetAsync(mark, 1, 1, c.stream));
    RVN_LAUNCH_CHECK();
    ++c.launches;
    // 2^rounds >= nodes: every node of the chain from line 0 is marked
    const uint32_t* jin = next;
    for (uint64_t reach = 1; reach < nodes; reach <<= 1) {
      FxChainKernel<<<g, 256, 0, c.stream>>>(jin, ja, mark, nodes);
      RVN_LAUNCH_CHECK();
      ++c.launches;
      jin = ja;
      std::swap(ja, jb);
    }
    FxFastqFlagKernel<<<g, 256, 0, c.stream>>>(L, next, mark, flag, stop);
    RVN_LAUNCH_CHECK();
    ExclusiveScanU32(c, flag, flag_off, count);
    FxScatterKernel<<<g, 256, 0, c.stream>>>(flag, flag_off, count, rec_line);
    FxFastqCutKernel<<<1, 1, 0, c.stream>>>(L, flag_off + count, mark, stop, sc);
    RVN_LAUNCH_CHECK();
    c.launches += 3;
    cut[0] = ReadU64(c, sc, sc + 1, &cut[1]);
    cut[2] = ReadU64(c, sc + 2);
    n_hdr = cut[0];
  }
  const uint64_t n_rec = cut[0];
  if (set.lens.size() + n_rec >= 0xFFFFFFFFULL) throw LimitError("too many reads");
  FxRec* rec = s.rec.reserve(n_rec + 1);
  uint32_t* nw = s.n_words.reserve(n_rec + 1);
  uint32_t* nb = s.n_bq.reserve(n_rec + 1);
  uint32_t* nn = s.n_name.reserve(n_rec + 1);
  uint64_t* woff = s.woff.reserve(n_rec + 1);
  uint64_t* bq_off = s.bq_off.reserve(n_rec + 1);
  uint64_t* name_off = s.name_off.reserve(n_rec + 1);
  uint64_t totals[3] = {0, 0, 0};
  if (n_rec) {
    FxRecordKernel<<<Grid(n_rec, c), 256, 0, c.stream>>>(L, fastq ? 1 : 0, rec_line, n_rec, n_hdr,
                                                         plus, qual_last, rec, nw, nb, nn,
                                                         err_key, over);
    RVN_LAUNCH_CHECK();
    ++c.launches;
    ExclusiveScanU32(c, nw, woff, n_rec);
    ExclusiveScanU32(c, nb, bq_off, n_rec);
    ExclusiveScanU32(c, nn, name_off, n_rec);
    totals[0] = ReadU64(c, woff + n_rec, bq_off + n_rec, &totals[1]);
    totals[2] = ReadU64(c, name_off + n_rec);
    GrowWords(c, set.words + totals[0] + 2, set.words);
    uint8_t* bq = s.bq.reserve(totals[1] + 1);
    char* names = s.names.reserve(totals[2] + 1);
    const unsigned pg = static_cast<unsigned>(
        std::min<uint64_t>((n_rec + kFxWarps - 1) / kFxWarps, c.sms * 8ULL));
    FxPackKernel<<<pg, kFxThreads, 0, c.stream>>>(text, rec, n_rec, woff, bq_off, name_off,
                                                   c.d_words.get() + set.words, bq, names,
                                                   err_key);
    RVN_LAUNCH_CHECK();
    ++c.launches;
  }
  TimerEnd(c);
  uint64_t over_limit = 0;
  const uint64_t key = ReadU64(c, sc + 4, sc + 5, &over_limit);
  const std::string where = " (" + path + ")";
  if (key != kFxNoError) {
    throw InvalidArgument(std::string(key & 1 ? kNotNucleotide
                                              : fastq ? kFastqInvalid : kFastaInvalid) + where);
  }
  if (cut[2]) throw InvalidArgument(kFastqInvalid + where);
  if (over_limit) throw LimitError("read of 2^31 or more bases" + where);
  if (n_rec) {
    const size_t r0 = set.lens.size(), b0 = set.bq.size(), c0 = set.names.size();
    std::vector<FxRec> h_rec(n_rec);
    std::vector<uint64_t> h_noff(n_rec + 1);
    set.lens.resize(r0 + n_rec);
    set.bq.resize(b0 + totals[1]);
    set.names.resize(c0 + totals[2]);
    RVN_CUDA(cudaMemcpyAsync(h_rec.data(), rec, n_rec * sizeof(FxRec), cudaMemcpyDeviceToHost,
                             c.stream));
    RVN_CUDA(cudaMemcpyAsync(h_noff.data(), name_off, (n_rec + 1) * 8, cudaMemcpyDeviceToHost,
                             c.stream));
    if (totals[1]) {
      RVN_CUDA(cudaMemcpyAsync(set.bq.data() + b0, s.bq.get(), totals[1], cudaMemcpyDeviceToHost,
                               c.stream));
    }
    if (totals[2]) {
      RVN_CUDA(cudaMemcpyAsync(&set.names[c0], s.names.get(), totals[2], cudaMemcpyDeviceToHost,
                               c.stream));
    }
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    for (uint64_t r = 0; r < n_rec; ++r) {
      const uint32_t len = h_rec[r].len;
      set.lens[r0 + r] = len;
      set.bq_off.push_back(set.bq_off.back() + (fastq ? (len + 63ULL) >> 6 : 0));
      set.name_off.push_back(c0 + h_noff[r + 1]);
    }
    set.words += totals[0];
  }
  return cut[1];
}

// one file's records, chunk by chunk, appended to the set
void ParseFile(Ctx& c, FxScratch& s, PinBuf<uint8_t>* slots, uint64_t chunk,
               const std::string& path, bool fastq, FxSet& set) {
  const std::string unreadable =
      "[bioparser::Parser::Parse] error: unable to read file (" + path + ")";
  auto raw = std::make_unique<BgzfFile>(path);
  FxMember first;
  gzFile f = nullptr;
  if (raw->ok() && raw->Member(0, &first)) {
    slots[0].reserve(kBgzfMaxMember);  // a slot holds at least one member
    slots[1].reserve(kBgzfMaxMember);
  } else {
    raw.reset();
    f = gzopen(path.c_str(), "rb");
    if (f == nullptr) {
      throw InvalidArgument("[bioparser::Parser::Create] error: unable to open file " + path);
    }
    gzbuffer(f, 1 << 20);
  }
  FxReader reader(f, std::move(raw), path, slots, chunk);
  int cur = 0;
  uint64_t len = 0, fresh = 0, want = chunk;
  for (int slot = 0;; slot ^= 1) {
    const auto t0 = std::chrono::steady_clock::now();
    const FxReader::Piece p = reader.Take(slot);
    s.read_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0)
                     .count();
    if (p.failed) throw InvalidArgument(unreadable);
    uint8_t* text = s.text[cur].reserve_keep(len + p.len + kFxPad, len, c.stream);
    unsigned bad = ~0u;
    if (p.members) {
      TimerBegin(c, "fastx_copy");
      uint8_t* comp = s.comp.reserve(p.raw);
      FxMember* mem = s.members.reserve(p.members);
      RVN_CUDA(cudaMemcpyAsync(comp, slots[slot].get(), p.raw, cudaMemcpyHostToDevice, c.stream));
      RVN_CUDA(cudaMemcpyAsync(mem, reader.Members(slot).data(), p.members * sizeof(FxMember),
                               cudaMemcpyHostToDevice, c.stream));
      TimerEnd(c);
      unsigned* d_bad = s.bad.reserve(1);
      RVN_CUDA(cudaMemsetAsync(d_bad, 0xFF, sizeof(unsigned), c.stream));
      TimerBegin(c, "fastx_inflate");
      FxInflateKernel<<<CeilDiv(p.members, kFxInfWarps), kFxInfWarps * 32, 0, c.stream>>>(
          comp, mem, p.members, text + len, d_bad);
      RVN_LAUNCH_CHECK();
      TimerEnd(c);
      ++c.launches;
      RVN_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof(unsigned), cudaMemcpyDeviceToHost, c.stream));
    } else if (p.len) {
      TimerBegin(c, "fastx_copy");
      RVN_CUDA(cudaMemcpyAsync(text + len, slots[slot].get(), p.len, cudaMemcpyHostToDevice,
                               c.stream));
      TimerEnd(c);
    }
    RVN_CUDA(cudaStreamSynchronize(c.stream));
    reader.Release(slot);
    if (bad != ~0u) throw InvalidArgument(unreadable);
    len += p.len;
    fresh += p.len;
    if (!p.last && fresh < want) continue;
    const uint64_t tail = ParseChunk(c, s, text, len, p.last, fastq, set, path);
    if (p.last) return;
    // a chunk without a whole record: the next one is at least twice as long
    want = tail > 0 ? chunk : std::max(chunk, len);
    const uint64_t keep = len - tail;
    uint8_t* other = s.text[cur ^ 1].reserve(keep + chunk + kFxPad);
    if (keep) {
      RVN_CUDA(cudaMemcpyAsync(other, text + tail, keep, cudaMemcpyDeviceToDevice, c.stream));
    }
    cur ^= 1;
    len = keep;
    fresh = 0;
  }
}

}  // namespace

void UploadFiles(Ctx& c, const char* const* paths, uint32_t n_paths) {
  // the current set goes first: its device words are where the parsed set's words go
  UploadReads(c, nullptr, nullptr, nullptr, nullptr, 0, 0, 0xFFFFFFFFu, /*whole_set=*/true);
  c.reads_unset = true;
  uint8_t table[256];
  for (int b = 0; b < 256; ++b) table[b] = biosoup::NucleotideCode(static_cast<char>(b));
  RVN_CUDA(cudaMemcpyToSymbolAsync(c_fx_code, table, sizeof(table), 0, cudaMemcpyHostToDevice,
                                   c.stream));
  const uint64_t chunk = c.fastx_chunk_bytes ? c.fastx_chunk_bytes : kFxDefaultChunk;
  std::vector<std::string> files(n_paths);
  uint64_t piece = 1;  // the slots need not outgrow the largest plain file
  for (uint32_t i = 0; i < n_paths; ++i) {
    if (!paths[i]) throw InvalidArgument("null path");
    files[i] = paths[i];
    struct stat st;
    if (IsSuffix(files[i], ".gz") || stat(paths[i], &st) != 0) {
      piece = chunk;
    } else {
      piece = std::max<uint64_t>(piece, std::min<uint64_t>(chunk, st.st_size + 1ULL));
    }
  }
  FxSet set;
  FxScratch s;
  PinBuf<uint8_t> slots[2];
  for (uint32_t i = 0; i < n_paths; ++i) {
    // raven::CreateParser (RavenLib/src/io.cc:7-41)
    const std::string& path = files[i];
    bool fastq;
    if (IsSuffix(path, ".fasta") || IsSuffix(path, ".fa") || IsSuffix(path, ".fasta.gz") ||
        IsSuffix(path, ".fa.gz")) {
      fastq = false;
    } else if (IsSuffix(path, ".fastq") || IsSuffix(path, ".fq") || IsSuffix(path, ".fastq.gz") ||
               IsSuffix(path, ".fq.gz")) {
      fastq = true;
    } else {
      throw InvalidArgument("[raven::CreateParser] error: file " + path +
                            " has unsupported format extension (valid extensions: .fasta, "
                            ".fasta.gz, .fa, .fa.gz, .fastq, .fastq.gz, .fq, .fq.gz)");
    }
    if (!slots[0].get()) {
      slots[0].reserve(piece);
      slots[1].reserve(piece);
    }
    ParseFile(c, s, slots, piece, path, fastq, set);
  }
  c.timer.names.push_back("fastx_read");
  c.timer.ms.push_back(s.read_ms);
  c.timer.pending.emplace_back(nullptr, nullptr);
  const uint32_t n = static_cast<uint32_t>(set.lens.size());
  std::vector<uint64_t> woff(n + 1ULL, 0);
  for (uint32_t i = 0; i < n; ++i) woff[i + 1] = woff[i] + ((set.lens[i] + 31ULL) >> 5);
  GrowWords(c, set.words + 2, set.words);
  AdoptParsedReads(c, woff.data(), set.lens.data(), n);
  c.fx_bq.swap(set.bq);
  c.fx_bq_off.swap(set.bq_off);
  c.fx_names.swap(set.names);
  c.fx_name_off.swap(set.name_off);
  c.fx_valid = true;
  c.reads_unset = false;
}

void ParsedReads(Ctx& c, uint64_t* words, uint64_t* word_off, uint32_t* lens,
                 uint8_t* block_quality, uint64_t* bq_off, char* names, uint64_t* name_off) {
  if (!c.fx_valid) throw StateError("the read set was not made by rvn_reads_upload_files");
  const uint32_t n = c.n_reads;
  if (words && c.n_words) {
    if (c.bases.on_host) {
      std::memcpy(words, c.bases.h_words.get(), c.n_words * sizeof(uint64_t));
    } else {
      RVN_CUDA(cudaMemcpyAsync(words, c.d_words.get(), c.n_words * sizeof(uint64_t),
                               cudaMemcpyDeviceToHost, c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));
    }
  }
  if (word_off) std::copy(c.h_woff.begin(), c.h_woff.begin() + n + 1, word_off);
  if (lens) std::copy(c.h_len.begin(), c.h_len.begin() + n, lens);
  if (block_quality) std::copy(c.fx_bq.begin(), c.fx_bq.end(), block_quality);
  if (bq_off) std::copy(c.fx_bq_off.begin(), c.fx_bq_off.end(), bq_off);
  if (names) std::copy(c.fx_names.begin(), c.fx_names.end(), names);
  if (name_off) std::copy(c.fx_name_off.begin(), c.fx_name_off.end(), name_off);
}

}  // namespace rvn
