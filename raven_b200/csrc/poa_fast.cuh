// raven_b200 — POA fast path (included by poa.cu): layers of at most 575 bases.
//
// Same semantics as PoaKernel (poa.cu), re-laid for the hardware:
//   * every lane owns kS = 18 CONTIGUOUS DP columns and keeps the previous row
//     in registers: a node whose (only) predecessor is the row just computed -
//     the common case along the backbone - needs no memory read at all;
//   * the horizontal gap recurrence runs sequentially inside a lane and is
//     closed across lanes by ONE warp max-scan per row (of lane-end value -
//     lane * kS * g), instead of one scan per 32 columns;
//   * the traceback direction of every cell (spoa's preference: diagonal over
//     predecessors in in-edge order, vertical, horizontal) is decided while the
//     row is in registers and stored as one byte, so the traceback reads one
//     byte per step instead of re-deriving it from up to three matrix cells;
//   * hot per-node state (topological marks, ranks) lives in shared memory,
//     nodes and edges are packed into 8-byte records.
#pragma once

namespace rvn {
namespace {

constexpr int kS = 18;                 // DP columns per lane
constexpr uint32_t kFastCols = 32 * kS;  // 576 = longest layer + 1
constexpr uint32_t kDirStride = 32 * 20; // bytes per direction row (20 per lane)

constexpr uint8_t kFMarks = 3, kFIgnored = 4, kFInSub = 8, kFSink = 16;
constexpr uint8_t kDirDiag = 0x00, kDirVert = 0x40, kDirHorz = 0x80;

struct FastLayout {
  size_t nodeA, nodeB, edgeA, edgeW, stack, order, aln_node, aln_pos, pred, score, H,
      DIR, bytes;
};

__host__ __device__ inline FastLayout MakeFastLayout(const PoaShape& s) {
  FastLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    size_t at = o;
    o += (bytes + 15) & ~size_t(15);
    return at;
  };
  L.nodeA = take(8ULL * s.ncap);
  L.nodeB = take(8ULL * s.ncap);
  L.edgeA = take(8ULL * s.ecap);
  L.edgeW = take(4ULL * s.ecap);
  L.stack = take(2ULL * 4 * s.ncap);
  L.order = take(2ULL * (kPoaMaxLayers + 1));
  L.aln_node = take(2ULL * (s.ncap + s.lmax + 2));
  L.aln_pos = take(2ULL * (s.ncap + s.lmax + 2));
  L.pred = take(4ULL * s.ncap);
  L.score = take(8ULL * s.ncap);
  L.H = take(2ULL * s.rows * kFastCols);
  L.DIR = take(1ULL * s.rows * kDirStride);
  L.bytes = o;
  return L;
}

struct FastGraph {
  uint2* nodeA;  // x: in_head | in_tail << 16   y: out_head | code << 16 | n_aligned << 24
  uint2* nodeB;  // x: aligned0 | aligned1 << 16  y: aligned2 | cov << 16
  uint2* edgeA;  // x: tail | head << 16          y: next_in | next_out << 16
  int32_t* edgeW;
  uint16_t *stack, *order;
  int16_t *aln_node, *aln_pos;
  int32_t* pred;
  long long* score;
  int16_t* H;
  uint8_t* DIR;
  uint8_t* flags;  // shared memory
  uint16_t *r2n, *n2r;  // shared memory
  uint32_t n_nodes, n_edges, ncap, ecap, stack_cap;
  bool overflow;
};

__device__ __forceinline__ uint32_t NInHead(uint2 a) { return a.x & 0xFFFF; }
__device__ __forceinline__ uint32_t NInTail(uint2 a) { return a.x >> 16; }
__device__ __forceinline__ uint32_t NOutHead(uint2 a) { return a.y & 0xFFFF; }
__device__ __forceinline__ uint32_t NCode(uint2 a) { return (a.y >> 16) & 0xFF; }
__device__ __forceinline__ uint32_t NAligned(uint2 a) { return a.y >> 24; }
__device__ __forceinline__ uint32_t NAlignedAt(uint2 b, uint32_t i) {
  return i == 0 ? (b.x & 0xFFFF) : i == 1 ? (b.x >> 16) : (b.y & 0xFFFF);
}
__device__ __forceinline__ uint32_t ETail(uint2 e) { return e.x & 0xFFFF; }
__device__ __forceinline__ uint32_t EHead(uint2 e) { return e.x >> 16; }
__device__ __forceinline__ uint32_t ENextIn(uint2 e) { return e.y & 0xFFFF; }
__device__ __forceinline__ uint32_t ENextOut(uint2 e) { return e.y >> 16; }

__device__ uint32_t FAddNode(FastGraph& g, uint32_t code) {
  if (g.n_nodes >= g.ncap) {
    g.overflow = true;
    return 0;
  }
  const uint32_t v = g.n_nodes++;
  g.nodeA[v] = make_uint2(0xFFFFFFFFu, 0xFFFFu | (code << 16));
  g.nodeB[v] = make_uint2(0, 0);
  g.flags[v] = 0;
  return v;
}

__device__ void FAddEdge(FastGraph& g, uint32_t tail, uint32_t head, int32_t w) {
  uint32_t last_out = kNone;
  for (uint32_t e = NOutHead(g.nodeA[tail]); e != kNone;) {
    const uint2 ea = g.edgeA[e];
    if (EHead(ea) == head) {
      g.edgeW[e] += w;
      return;
    }
    last_out = e;
    e = ENextOut(ea);
  }
  if (g.n_edges >= g.ecap) {
    g.overflow = true;
    return;
  }
  const uint32_t e = g.n_edges++;
  g.edgeA[e] = make_uint2(tail | (head << 16), 0xFFFFFFFFu);
  g.edgeW[e] = w;
  if (last_out == kNone) {
    uint2 a = g.nodeA[tail];
    a.y = (a.y & 0xFFFF0000u) | e;
    g.nodeA[tail] = a;
  } else {
    uint2 ea = g.edgeA[last_out];
    ea.y = (ea.y & 0xFFFFu) | (e << 16);
    g.edgeA[last_out] = ea;
  }
  uint2 h = g.nodeA[head];
  if (NInHead(h) == kNone) {
    h.x = e | (e << 16);
  } else {
    const uint32_t it = NInTail(h);
    uint2 ea = g.edgeA[it];
    ea.y = (ea.y & 0xFFFF0000u) | e;
    g.edgeA[it] = ea;
    h.x = (h.x & 0xFFFFu) | (e << 16);
  }
  g.nodeA[head] = h;
}

__device__ __forceinline__ void FAddCov(FastGraph& g, uint32_t v) {
  uint2 b = g.nodeB[v];
  b.y += 1u << 16;
  g.nodeB[v] = b;
}
__device__ __forceinline__ uint32_t FCov(const FastGraph& g, uint32_t v) {
  return g.nodeB[v].y >> 16;
}

__device__ uint32_t FAddChain(FastGraph& g, const SeqView& s, uint32_t begin,
                              uint32_t end) {
  if (begin == end) return kNone;
  uint32_t first = kNone, prev = kNone;
  for (uint32_t i = begin; i < end && !g.overflow; ++i) {
    const uint32_t cur = FAddNode(g, CodeOf(s.bases[i]));
    if (prev != kNone) FAddEdge(g, prev, cur, s.weight(i - 1) + s.weight(i));
    if (first == kNone) first = cur;
    prev = cur;
  }
  return first;
}

__device__ void FLinkAligned(FastGraph& g, uint32_t a, uint32_t b) {
  // append b to a's aligned list
  uint2 na = g.nodeA[a];
  uint2 nb = g.nodeB[a];
  const uint32_t k = NAligned(na);
  if (k == 0) nb.x = (nb.x & 0xFFFF0000u) | b;
  else if (k == 1) nb.x = (nb.x & 0xFFFFu) | (b << 16);
  else nb.y = (nb.y & 0xFFFF0000u) | b;
  na.y += 1u << 24;
  g.nodeA[a] = na;
  g.nodeB[a] = nb;
}

// spoa Graph::TopologicalSort restricted to nodes flagged kFInSub (lane 0)
__device__ uint32_t FTopoSort(FastGraph& g) {
  const uint32_t n = g.n_nodes;
  uint32_t rank = 0, sp = 0;
  for (uint32_t root = 0; root < n; ++root) {
    if (!(g.flags[root] & kFInSub) || (g.flags[root] & kFMarks)) continue;
    g.stack[sp++] = static_cast<uint16_t>(root);
    while (sp > 0) {
      const uint32_t cur = g.stack[sp - 1];
      bool valid = true;
      if ((g.flags[cur] & kFMarks) != 2) {
        const uint2 a = g.nodeA[cur];
        for (uint32_t e = NInHead(a); e != kNone;) {
          const uint2 ea = g.edgeA[e];
          const uint32_t t = ETail(ea);
          const uint8_t ft = g.flags[t];
          if ((ft & kFInSub) && (ft & kFMarks) != 2) {
            if (sp >= g.stack_cap) {
              g.overflow = true;
              return 0;
            }
            g.stack[sp++] = static_cast<uint16_t>(t);
            valid = false;
          }
          e = ENextIn(ea);
        }
        const uint32_t na = NAligned(a);
        uint2 b = make_uint2(0, 0);
        if (na) b = g.nodeB[cur];
        if (!(g.flags[cur] & kFIgnored)) {
          for (uint32_t i = 0; i < na; ++i) {
            const uint32_t t = NAlignedAt(b, i);
            const uint8_t ft = g.flags[t];
            if ((ft & kFInSub) && (ft & kFMarks) != 2) {
              if (sp >= g.stack_cap) {
                g.overflow = true;
                return 0;
              }
              g.stack[sp++] = static_cast<uint16_t>(t);
              g.flags[t] = ft | kFIgnored;
              valid = false;
            }
          }
        }
        if (valid) {
          g.flags[cur] = (g.flags[cur] & ~kFMarks) | 2;
          if (!(g.flags[cur] & kFIgnored)) {
            g.n2r[cur] = static_cast<uint16_t>(rank);
            g.r2n[rank++] = static_cast<uint16_t>(cur);
            for (uint32_t i = 0; i < na; ++i) {
              const uint32_t t = NAlignedAt(b, i);
              if (g.flags[t] & kFInSub) {
                g.n2r[t] = static_cast<uint16_t>(rank);
                g.r2n[rank++] = static_cast<uint16_t>(t);
              }
            }
          }
        } else {
          g.flags[cur] = (g.flags[cur] & ~kFMarks) | 1;
        }
      }
      if (valid) --sp;
    }
  }
  return rank;
}

__device__ void FMarkSubgraph(FastGraph& g, uint32_t from, uint32_t min_id) {
  uint32_t sp = 0;
  g.stack[sp++] = static_cast<uint16_t>(from);
  while (sp > 0) {
    const uint32_t cur = g.stack[--sp];
    if ((g.flags[cur] & kFInSub) || cur < min_id) continue;
    const uint2 a = g.nodeA[cur];
    for (uint32_t e = NInHead(a); e != kNone;) {
      const uint2 ea = g.edgeA[e];
      if (sp >= g.stack_cap) {
        g.overflow = true;
        return;
      }
      g.stack[sp++] = static_cast<uint16_t>(ETail(ea));
      e = ENextIn(ea);
    }
    const uint32_t na = NAligned(a);
    if (na) {
      const uint2 b = g.nodeB[cur];
      for (uint32_t i = 0; i < na; ++i) {
        if (sp >= g.stack_cap) {
          g.overflow = true;
          return;
        }
        g.stack[sp++] = static_cast<uint16_t>(NAlignedAt(b, i));
      }
    }
    g.flags[cur] |= kFInSub;
  }
}

__device__ void FAddAlignment(FastGraph& g, const SeqView& s, uint32_t aln_len) {
  int32_t first_pos = -1, last_pos = -1;
  for (uint32_t i = 0; i < aln_len; ++i) {
    if (g.aln_pos[i] != -1) {
      if (first_pos < 0) first_pos = g.aln_pos[i];
      last_pos = g.aln_pos[i];
    }
  }
  const uint32_t before = g.n_nodes;
  uint32_t begin = FAddChain(g, s, 0, first_pos);
  uint32_t prev = before == g.n_nodes ? kNone : g.n_nodes - 1;
  const uint32_t last = FAddChain(g, s, last_pos + 1, s.len);
  const bool counts = s.len >= 2;
  if (counts) {
    for (uint32_t v = before; v < g.n_nodes; ++v) FAddCov(g, v);
  }
  for (uint32_t i = 0; i < aln_len && !g.overflow; ++i) {
    const int32_t pos = g.aln_pos[i];
    if (pos == -1) continue;
    const uint32_t code = CodeOf(s.bases[pos]);
    uint32_t cur = kNone;
    if (g.aln_node[i] == -1) {
      cur = FAddNode(g, code);
    } else {
      const uint32_t jt = static_cast<uint16_t>(g.aln_node[i]);
      const uint2 ja = g.nodeA[jt];
      if (NCode(ja) == code) {
        cur = jt;
      } else {
        const uint32_t na = NAligned(ja);
        const uint2 jb = g.nodeB[jt];
        for (uint32_t a = 0; a < na; ++a) {
          const uint32_t kt = NAlignedAt(jb, a);
          if (NCode(g.nodeA[kt]) == code) {
            cur = kt;
            break;
          }
        }
        if (cur == kNone) {
          cur = FAddNode(g, code);
          if (g.overflow) break;
          for (uint32_t a = 0; a < na; ++a) {
            const uint32_t kt = NAlignedAt(jb, a);
            FLinkAligned(g, kt, cur);
            FLinkAligned(g, cur, kt);
          }
          FLinkAligned(g, jt, cur);
          FLinkAligned(g, cur, jt);
        }
      }
    }
    if (g.overflow) break;
    if (counts) FAddCov(g, cur);
    if (begin == kNone) begin = cur;
    if (prev != kNone) FAddEdge(g, prev, cur, s.weight(pos - 1) + s.weight(pos));
    prev = cur;
  }
  if (last != kNone && !g.overflow) {
    FAddEdge(g, prev, last, s.weight(last_pos) + s.weight(last_pos + 1));
  }
}

// load / store one lane's kS cells of a row (18 int16 = 9 words)
__device__ __forceinline__ void LoadRow(const int16_t* row, uint32_t lane, int (&v)[kS]) {
  const uint32_t* p = reinterpret_cast<const uint32_t*>(row + lane * kS);
#pragma unroll
  for (int k = 0; k < kS / 2; ++k) {
    const uint32_t x = p[k];
    v[2 * k] = static_cast<int16_t>(x & 0xFFFF);
    v[2 * k + 1] = static_cast<int16_t>(x >> 16);
  }
}
__device__ __forceinline__ void StoreRow(int16_t* row, uint32_t lane, const int (&v)[kS]) {
  uint32_t* p = reinterpret_cast<uint32_t*>(row + lane * kS);
#pragma unroll
  for (int k = 0; k < kS / 2; ++k) {
    p[k] = (static_cast<uint32_t>(v[2 * k]) & 0xFFFF) |
           (static_cast<uint32_t>(v[2 * k + 1]) << 16);
  }
}

constexpr int kNegInf = -1000000;

// one warp per CTA; the register cap decides how many windows an SM holds at
// once (the kernel is bound by the latency of lane 0's graph surgery, so more
// resident windows = more throughput until the DP spills)
#ifndef RVN_POA_BLOCKS
#define RVN_POA_BLOCKS 16
#endif
__global__ void __launch_bounds__(32, RVN_POA_BLOCKS)
PoaKernelFast(uint32_t n_windows, const uint32_t* __restrict__ win_list,
              const uint32_t* __restrict__ win_first,
              const uint64_t* __restrict__ seq_off, const uint8_t* __restrict__ bases,
              const uint8_t* __restrict__ quals, const uint32_t* __restrict__ seq_begin,
              const uint32_t* __restrict__ seq_end, int m, int n, int gap, int trim,
              int tgs, PoaShape shape, uint8_t* __restrict__ scratch,
              size_t scratch_stride, uint8_t* __restrict__ cons,
              const uint64_t* __restrict__ cons_off, uint32_t* __restrict__ cons_len,
              uint32_t* __restrict__ cov_out, uint8_t* __restrict__ status,
              unsigned long long* __restrict__ cells) {
  extern __shared__ __align__(16) unsigned char smem[];
  if (blockIdx.x >= n_windows) return;
  const uint32_t lane = threadIdx.x;
  const uint32_t w = win_list ? win_list[blockIdx.x] : blockIdx.x;
  const uint32_t s0 = win_first[w], s1 = win_first[w + 1];
  const uint32_t nseq = KeptSequences(seq_off, seq_begin, seq_end, s0, s1, lane);
  const uint32_t L0 = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
  uint8_t* out = cons + cons_off[w];
  uint32_t* cov_dst = cov_out ? cov_out + cons_off[w] : nullptr;

  if (nseq < 3) {
    for (uint32_t i = lane; i < L0; i += 32) {
      out[i] = bases[seq_off[s0] + i];
      if (cov_dst) cov_dst[i] = 0;
    }
    if (lane == 0) {
      cons_len[w] = L0;
      status[w] = 0;
    }
    return;
  }
  {
    bool bad_letter = false;
    for (uint64_t i = seq_off[s0] + lane; i < seq_off[s1]; i += 32) {
      if (CodeOf(bases[i]) < 0) bad_letter = true;
    }
    if (__any_sync(0xffffffffu, bad_letter)) {
      if (lane == 0) {
        cons_len[w] = 0;
        status[w] = kPoaStatusInvalid;
      }
      return;
    }
  }

  uint8_t* base = scratch + scratch_stride * blockIdx.x;
  const FastLayout L = MakeFastLayout(shape);
  __shared__ FastGraph g;
  __shared__ uint32_t sh_rows, sh_fail;
  if (lane == 0) {
    g.nodeA = reinterpret_cast<uint2*>(base + L.nodeA);
    g.nodeB = reinterpret_cast<uint2*>(base + L.nodeB);
    g.edgeA = reinterpret_cast<uint2*>(base + L.edgeA);
    g.edgeW = reinterpret_cast<int32_t*>(base + L.edgeW);
    g.stack = reinterpret_cast<uint16_t*>(base + L.stack);
    g.order = reinterpret_cast<uint16_t*>(base + L.order);
    g.aln_node = reinterpret_cast<int16_t*>(base + L.aln_node);
    g.aln_pos = reinterpret_cast<int16_t*>(base + L.aln_pos);
    g.pred = reinterpret_cast<int32_t*>(base + L.pred);
    g.score = reinterpret_cast<long long*>(base + L.score);
    g.H = reinterpret_cast<int16_t*>(base + L.H);
    g.DIR = base + L.DIR;
    g.flags = smem;
    g.r2n = reinterpret_cast<uint16_t*>(smem + ((shape.ncap + 15) & ~15u));
    g.n2r = g.r2n + shape.ncap;
    g.n_nodes = g.n_edges = 0;
    g.ncap = shape.ncap;
    g.ecap = shape.ecap;
    g.stack_cap = 4 * shape.ncap;
    g.overflow = false;
    sh_fail = OrderLayers(g.order, seq_off, seq_begin, seq_end, s0, s1, L0, kFastCols - 1);
    if (!sh_fail) {
      SeqView bb{bases + seq_off[s0], quals ? quals + seq_off[s0] : nullptr, L0, 0};
      FAddChain(g, bb, 0, L0);
      if (L0 >= 2) {
        for (uint32_t v = 0; v < g.n_nodes; ++v) FAddCov(g, v);
      }
    }
  }
  __syncwarp();

  const uint32_t offset = static_cast<uint32_t>(0.01 * L0);
  unsigned long long my_cells = 0;

  for (uint32_t li = 0; li + 1 < nseq; ++li) {
    if (sh_fail || g.overflow) break;
    const uint32_t s = s0 + g.order[li];
    const SeqView sv{bases + seq_off[s], quals ? quals + seq_off[s] : nullptr,
                     static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]), 1};
    const uint32_t len = sv.len;
    const uint32_t lb = seq_begin[s], le = seq_end[s];
    const bool full = lb < offset && le > L0 - offset;

    // ---- the (sub)graph this layer aligns to, in topological order ----
    const uint32_t nn = g.n_nodes;
    for (uint32_t v = lane; v < nn; v += 32) g.flags[v] = full ? kFInSub : 0;
    __syncwarp();
    if (lane == 0) {
      if (!full) FMarkSubgraph(g, le, lb);
      const uint32_t rows = g.overflow ? 0 : FTopoSort(g);
      const int amax = max(max(abs(m), abs(n)), abs(gap));
      if (static_cast<long long>(amax) * (rows + len + 2) > 32000) g.overflow = true;
      sh_rows = rows;
    }
    __syncwarp();
    const uint32_t rows = sh_rows;
    if (g.overflow) break;
    my_cells += static_cast<unsigned long long>(rows + 1) * (len + 1);
    // sinks: no out-edge inside the (sub)graph
    for (uint32_t r = lane; r < rows; r += 32) {
      const uint32_t v = g.r2n[r];
      bool sink = true;
      for (uint32_t e = NOutHead(g.nodeA[v]); e != kNone;) {
        const uint2 ea = g.edgeA[e];
        if (g.flags[EHead(ea)] & kFInSub) {
          sink = false;
          break;
        }
        e = ENextOut(ea);
      }
      if (sink) g.flags[v] |= kFSink;
    }
    __syncwarp();

    // ---- DP: lane owns columns [lane*kS, lane*kS + kS) ----
    int16_t* H = g.H;
    uint8_t* DIR = g.DIR;
    const uint32_t j0 = lane * kS;
    int scode[kS];  // code of the sequence letter consumed by column j (j >= 1)
#pragma unroll
    for (int k = 0; k < kS; ++k) {
      const uint32_t j = j0 + k;
      scode[k] = (j >= 1 && j <= len) ? CodeOf(sv.bases[j - 1]) : 9;
    }
    int R[kS];  // the row computed last (row 0 to start with)
#pragma unroll
    for (int k = 0; k < kS; ++k) R[k] = static_cast<int>(j0 + k) * gap;
    StoreRow(H, lane, R);
    uint32_t r_row = 0;  // matrix row held in R
    int best_score = -2147483647, best_row = -1;

    for (uint32_t r = 0; r < rows; ++r) {
      const uint32_t v = g.r2n[r];
      const uint2 va = g.nodeA[v];
      const int vcode = static_cast<int>(NCode(va));
      int M[kS];
#pragma unroll
      for (int k = 0; k < kS; ++k) M[k] = kNegInf;
      int col0 = kNegInf;
      // predecessors inside the (sub)graph, in in-edge order; a node without
      // any uses the virtual start row 0
      auto next_pred = [&](uint32_t& e, bool& any, uint32_t& prow) -> bool {
        while (e != kNone) {
          const uint2 ea = g.edgeA[e];
          e = ENextIn(ea);
          const uint32_t t = ETail(ea);
          if (g.flags[t] & kFInSub) {
            prow = g.n2r[t] + 1u;
            any = true;
            return true;
          }
        }
        if (!any) {
          any = true;
          prow = 0;
          return true;
        }
        return false;
      };
      {
        uint32_t e = NInHead(va), prow = 0;
        bool any = false;
        while (next_pred(e, any, prow)) {
          int V[kS];
          if (prow == r_row) {
#pragma unroll
            for (int k = 0; k < kS; ++k) V[k] = R[k];
          } else {
            LoadRow(H + static_cast<size_t>(prow) * kFastCols, lane, V);
          }
          int left = __shfl_up_sync(0xffffffffu, V[kS - 1], 1);
          if (lane == 0) left = kNegInf;
#pragma unroll
          for (int k = 0; k < kS; ++k) {
            const int match = scode[k] == vcode ? m : n;
            const int d = (k == 0 ? left : V[k - 1]) + match;
            const int u = V[k] + gap;
            M[k] = max(M[k], max(d, u));
          }
          if (lane == 0) col0 = max(col0, V[0]);
        }
      }
      // column 0 of this row
      col0 = __shfl_sync(0xffffffffu, col0, 0) + gap;
      // horizontal recurrence: local pass, one warp scan, apply
      int Hc[kS];
      {
        int run = kNegInf;
#pragma unroll
        for (int k = 0; k < kS; ++k) {
          if (lane == 0 && k == 0) {
            run = col0;
          } else {
            run = max(M[k], run + gap);
          }
          Hc[k] = run;
        }
        // carry into lane l = max over lanes t < l of (end_t + (l-1-t)*kS*g)
        int b = run - static_cast<int>(lane) * kS * gap;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int o = __shfl_up_sync(0xffffffffu, b, d);
          if (static_cast<int>(lane) >= d) b = max(b, o);
        }
        int cin = __shfl_up_sync(0xffffffffu, b, 1);
        cin = lane == 0 ? kNegInf : cin + static_cast<int>(lane - 1) * kS * gap;
        // cin = value of the cell left of this lane's first column
#pragma unroll
        for (int k = 0; k < kS; ++k) {
          Hc[k] = max(Hc[k], cin + (k + 1) * gap);
        }
      }
      // directions: diagonal over predecessors in order, vertical, horizontal
      uint8_t D[kS];
#pragma unroll
      for (int k = 0; k < kS; ++k) D[k] = kDirHorz;
      {
        uint32_t done_diag = 0;  // bit k set once a diagonal predecessor is found
        uint8_t VD[kS];          // first vertical candidate, used if no diagonal
#pragma unroll
        for (int k = 0; k < kS; ++k) VD[k] = 0xFF;
        uint32_t e = NInHead(va), prow = 0, ord = 0;
        bool any = false;
        while (next_pred(e, any, prow)) {
          int V[kS];
          if (prow == r_row) {
#pragma unroll
            for (int k = 0; k < kS; ++k) V[k] = R[k];
          } else {
            LoadRow(H + static_cast<size_t>(prow) * kFastCols, lane, V);
          }
          int left = __shfl_up_sync(0xffffffffu, V[kS - 1], 1);
          if (lane == 0) left = kNegInf;
          const uint8_t o8 = static_cast<uint8_t>(ord < 63 ? ord : 63);
#pragma unroll
          for (int k = 0; k < kS; ++k) {
            const bool is_col0 = lane == 0 && k == 0;
            const int match = scode[k] == vcode ? m : n;
            const int d = (k == 0 ? left : V[k - 1]) + match;
            if (!is_col0 && !((done_diag >> k) & 1) && d == Hc[k]) {
              D[k] = kDirDiag | o8;
              done_diag |= 1u << k;
            }
            if (VD[k] == 0xFF && V[k] + gap == Hc[k]) VD[k] = kDirVert | o8;
          }
          ++ord;
        }
#pragma unroll
        for (int k = 0; k < kS; ++k) {
          if (!((done_diag >> k) & 1) && VD[k] != 0xFF) D[k] = VD[k];
        }
      }
      // store the row and its directions
      int16_t* row = H + static_cast<size_t>(r + 1) * kFastCols;
      StoreRow(row, lane, Hc);
      {
        uint32_t* dp = reinterpret_cast<uint32_t*>(DIR + static_cast<size_t>(r + 1) * kDirStride + lane * 20);
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          uint32_t x = 0;
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const int k = q * 4 + b;
            if (k < kS) x |= static_cast<uint32_t>(D[k]) << (8 * b);
          }
          dp[q] = x;
        }
      }
#pragma unroll
      for (int k = 0; k < kS; ++k) R[k] = Hc[k];
      r_row = r + 1;
      // sinks compete with their value in the last column
      {
        const uint32_t lj = len / kS, lk = len % kS;
        int sc = 0;
#pragma unroll
        for (int k = 0; k < kS; ++k) {
          if (static_cast<uint32_t>(k) == lk) sc = Hc[k];
        }
        sc = __shfl_sync(0xffffffffu, sc, lj);
        if ((g.flags[v] & kFSink) && best_score < sc) {
          best_score = sc;
          best_row = static_cast<int>(r + 1);
        }
      }
    }
    __syncwarp();

    // ---- (lane 0) traceback from the stored directions + merge ----
    if (lane == 0) {
      uint32_t alen = 0;
      uint32_t i = best_row < 0 ? 0 : static_cast<uint32_t>(best_row), j = len;
      if (best_row < 0) j = 0;
      const uint32_t acap = shape.ncap + shape.lmax + 2;
      while (!(i == 0 && j == 0)) {
        uint32_t pi = i, pj = j;
        if (i == 0) {
          pj = j - 1;  // row 0: horizontal only
        } else {
          const uint8_t d = DIR[static_cast<size_t>(i) * kDirStride + (j / kS) * 20 + (j % kS)];
          if (d & kDirHorz) {
            pj = j - 1;
          } else {
            // the predecessor with that ordinal among the in-edges inside the graph
            const uint32_t want = d & 0x3F;
            const uint32_t v = g.r2n[i - 1];
            uint32_t ord = 0, prow = 0;
            bool found = false;
            const bool diag = !(d & kDirVert);
            const int h = H[static_cast<size_t>(i) * kFastCols + j];
            const int match = diag ? ((CodeOf(sv.bases[j - 1]) ==
                                       static_cast<int>(NCode(g.nodeA[v]))) ? m : n) : 0;
            for (uint32_t e = NInHead(g.nodeA[v]); e != kNone;) {
              const uint2 ea = g.edgeA[e];
              e = ENextIn(ea);
              const uint32_t t = ETail(ea);
              if (!(g.flags[t] & kFInSub)) continue;
              if (want < 63 ? ord == want
                            : (ord >= 63 &&
                               (diag ? h == H[static_cast<size_t>(g.n2r[t] + 1) * kFastCols + j - 1] + match
                                     : h == H[static_cast<size_t>(g.n2r[t] + 1) * kFastCols + j] + gap))) {
                prow = g.n2r[t] + 1u;
                found = true;
                break;
              }
              ++ord;
            }
            if (!found) prow = 0;  // virtual start row
            pi = prow;
            if (diag) pj = j - 1;
          }
        }
        if (alen >= acap) {
          g.overflow = true;
          break;
        }
        g.aln_node[alen] = i == pi ? -1 : static_cast<int16_t>(g.r2n[i - 1]);
        g.aln_pos[alen] = j == pj ? -1 : static_cast<int16_t>(j - 1);
        ++alen;
        i = pi;
        j = pj;
      }
      for (uint32_t a = 0; a < alen / 2; ++a) {
        const int16_t tn = g.aln_node[a], tp = g.aln_pos[a];
        g.aln_node[a] = g.aln_node[alen - 1 - a];
        g.aln_pos[a] = g.aln_pos[alen - 1 - a];
        g.aln_node[alen - 1 - a] = tn;
        g.aln_pos[alen - 1 - a] = tp;
      }
      if (!g.overflow) {
        if (alen == 0) {
          const uint32_t before = g.n_nodes;
          FAddChain(g, sv, 0, sv.len);
          if (sv.len >= 2) {
            for (uint32_t v = before; v < g.n_nodes; ++v) FAddCov(g, v);
          }
        } else {
          FAddAlignment(g, sv, alen);
        }
      }
    }
    __syncwarp();
  }

  // ---- consensus (lane 0) ----
  {
    const uint32_t nn = g.n_nodes;
    for (uint32_t v = lane; v < nn; v += 32) g.flags[v] = kFInSub;
    __syncwarp();
  }
  if (lane == 0) {
    uint32_t st = 0, clen = 0;
    if (sh_fail) {
      st = sh_fail;
    } else if (g.overflow) {
      st = kPoaStatusCapacity;
    } else {
      const uint32_t rows = FTopoSort(g);
      if (g.overflow) {
        st = kPoaStatusCapacity;
      } else {
        for (uint32_t v = 0; v < g.n_nodes; ++v) {
          g.pred[v] = -1;
          g.score[v] = -1;
        }
        int32_t mx = -1;
        for (uint32_t r = 0; r < rows; ++r) {
          const uint32_t v = g.r2n[r];
          for (uint32_t e = NInHead(g.nodeA[v]); e != kNone;) {
            const uint2 ea = g.edgeA[e];
            const uint32_t t = ETail(ea);
            const long long wgt = g.edgeW[e];
            if (g.score[v] < wgt ||
                (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
              g.score[v] = wgt;
              g.pred[v] = static_cast<int32_t>(t);
            }
            e = ENextIn(ea);
          }
          if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
          if (mx < 0 || g.score[mx] < g.score[v]) mx = static_cast<int32_t>(v);
        }
        while (NOutHead(g.nodeA[mx]) != kNone) {
          const uint32_t rank = g.n2r[mx];
          for (uint32_t e = NOutHead(g.nodeA[mx]); e != kNone;) {
            const uint2 ea = g.edgeA[e];
            const uint32_t hd = EHead(ea);
            for (uint32_t f = NInHead(g.nodeA[hd]); f != kNone;) {
              const uint2 fa = g.edgeA[f];
              if (ETail(fa) != static_cast<uint32_t>(mx)) g.score[ETail(fa)] = -1;
              f = ENextIn(fa);
            }
            e = ENextOut(ea);
          }
          int32_t nmx = -1;
          for (uint32_t r = rank + 1; r < rows; ++r) {
            const uint32_t v = g.r2n[r];
            g.score[v] = -1;
            g.pred[v] = -1;
            for (uint32_t e = NInHead(g.nodeA[v]); e != kNone;) {
              const uint2 ea = g.edgeA[e];
              const uint32_t t = ETail(ea);
              const long long wgt = g.edgeW[e];
              e = ENextIn(ea);
              if (g.score[t] == -1) continue;
              if (g.score[v] < wgt ||
                  (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
                g.score[v] = wgt;
                g.pred[v] = static_cast<int32_t>(t);
              }
            }
            if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
            if (nmx < 0 || g.score[nmx] < g.score[v]) nmx = static_cast<int32_t>(v);
          }
          mx = nmx;
        }
        uint32_t plen = 0;
        int32_t v = mx;
        while (g.pred[v] != -1) {
          g.r2n[plen++] = static_cast<uint16_t>(v);
          v = g.pred[v];
        }
        g.r2n[plen++] = static_cast<uint16_t>(v);
        auto coverage = [&](uint32_t idx) -> uint32_t {
          const uint32_t nd = g.r2n[plen - 1 - idx];
          uint32_t cvg = FCov(g, nd);
          const uint32_t na = NAligned(g.nodeA[nd]);
          if (na) {
            const uint2 b = g.nodeB[nd];
            for (uint32_t a = 0; a < na; ++a) cvg += FCov(g, NAlignedAt(b, a));
          }
          return cvg;
        };
        uint32_t cb = 0, ce = plen;
        st = kPoaStatusOk;
        if (tgs && trim) {
          const uint32_t avg = (nseq - 1) / 2;
          int32_t b = 0, e2 = static_cast<int32_t>(plen) - 1;
          for (; b < static_cast<int32_t>(plen); ++b) {
            if (coverage(b) >= avg) break;
          }
          for (; e2 >= 0; --e2) {
            if (coverage(e2) >= avg) break;
          }
          if (b >= e2) {
            st |= kPoaStatusChimeric;
          } else {
            cb = b;
            ce = e2 + 1;
          }
        }
        clen = ce - cb;
        for (uint32_t i = 0; i < clen; ++i) {
          const uint32_t nd = g.r2n[plen - 1 - (cb + i)];
          out[i] = "ACGT"[NCode(g.nodeA[nd])];
          if (cov_dst) cov_dst[i] = coverage(cb + i);
        }
      }
    }
    cons_len[w] = clen;
    status[w] = static_cast<uint8_t>(st);
    if (cells && st != kPoaStatusCapacity) atomicAdd(cells, my_cells);
  }
}

}  // namespace
}  // namespace rvn
