// raven_b200 — POA register-row kernel (included by poa.cu): layers of at most 575 bases.
//
// The graph, its surgery and the consensus are poa.cu's, over PoaGraph<PoaNarrow>; only
// the DP fill and the traceback are this kernel's own:
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
//   * the per-node flags and ranks live in shared memory.
#pragma once

namespace rvn {
namespace {

constexpr uint8_t kDirDiag = 0x00, kDirVert = 0x40, kDirHorz = 0x80;

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
  using W = PoaNarrow;
  extern __shared__ __align__(16) unsigned char smem[];
  if (blockIdx.x >= n_windows) return;
  const uint32_t lane = threadIdx.x;
  const uint32_t w = win_list ? win_list[blockIdx.x] : blockIdx.x;
  const uint32_t s0 = win_first[w], s1 = win_first[w + 1];
  const uint32_t L0 = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
  uint8_t* out = cons + cons_off[w];
  uint32_t* cov_dst = cov_out ? cov_out + cons_off[w] : nullptr;
  const uint32_t nseq = KeptSequences(seq_off, seq_begin, seq_end, s0, s1, lane);
  if (WindowDone(nseq, s0, s1, L0, seq_off, bases, out, cov_dst, cons_len + w, status + w, lane)) {
    return;
  }

  uint8_t* base = scratch + scratch_stride * blockIdx.x;
  const PoaLayout L = MakePoaLayout<W>(shape, true);
  __shared__ PoaGraph<W> g;
  __shared__ uint32_t sh_fail;
  if (lane == 0) {
    // dynamic shared memory: ncap flags (rounded up to 16 bytes), r2n, n2r
    g.flags = smem;
    g.r2n = reinterpret_cast<uint16_t*>(smem + ((shape.ncap + 15) & ~15u));
    g.n2r = g.r2n + shape.ncap;
    sh_fail = SetupGraph(g, base, L, shape, seq_off, bases, quals, seq_begin, seq_end, s0, s1,
                         L0);
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
    const uint32_t rows = LayerGraph(g, lb < offset && le > L0 - offset, lb, le, len, m, n, gap, lane);
    if (g.overflow) break;
    my_cells += static_cast<unsigned long long>(rows + 1) * (len + 1);

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
      const PoaNodeA<uint16_t> va = Ld(g.node_a + v);
      const int vcode = va.code;
      int M[kS];
#pragma unroll
      for (int k = 0; k < kS; ++k) M[k] = W::kNoCell;
      int col0 = W::kNoCell;
      // predecessors inside the (sub)graph, in in-edge order; a node without
      // any uses the virtual start row 0
      auto next_pred = [&](uint32_t& e, bool& any, uint32_t& prow) -> bool {
        while (e != W::kNone) {
          const PoaEdge<uint16_t> ea = Ld(g.edge + e);
          e = ea.next_in;
          const uint32_t t = ea.tail;
          if (g.flags[t] & kInSub) {
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
        uint32_t e = va.in_head, prow = 0;
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
          if (lane == 0) left = W::kNoCell;
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
        int run = W::kNoCell;
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
        cin = lane == 0 ? W::kNoCell : cin + static_cast<int>(lane - 1) * kS * gap;
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
        uint32_t e = va.in_head, prow = 0, ord = 0;
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
          if (lane == 0) left = W::kNoCell;
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
        if ((g.flags[v] & kSink) && best_score < sc) {
          best_score = sc;
          best_row = static_cast<int>(r + 1);
        }
      }
    }
    __syncwarp();

    // ---- (lane 0) traceback from the stored directions ----
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
            const PoaNodeA<uint16_t> va = Ld(g.node_a + g.r2n[i - 1]);
            uint32_t ord = 0, prow = 0;
            bool found = false;
            const bool diag = !(d & kDirVert);
            const int h = H[static_cast<size_t>(i) * kFastCols + j];
            const int match = diag ? ((CodeOf(sv.bases[j - 1]) == va.code) ? m : n) : 0;
            for (uint32_t e = va.in_head; e != W::kNone;) {
              const PoaEdge<uint16_t> ea = Ld(g.edge + e);
              e = ea.next_in;
              const uint32_t t = ea.tail;
              if (!(g.flags[t] & kInSub)) continue;
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
      MergeLayer(g, sv, alen);
    }
    __syncwarp();
  }
  Consensus(g, sh_fail, nseq, trim, tgs, my_cells, out, cov_dst, cons_len + w, status + w,
            cells, lane);
}

}  // namespace
}  // namespace rvn
