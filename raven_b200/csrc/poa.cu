// raven_b200 — windowed partial-order-alignment consensus on sm_90a.
//
// Replaces the per-window consensus of racon::Polisher::Polish (un-vendored;
// the reference calls it at RavenLib/src/polish.cc:43-51 with w = 500,
// trim = true, m/n/g from PolishCfg polish.hpp:13-17): racon::Window::
// GenerateConsensus over spoa's Graph / AlignmentEngine (global alignment,
// linear gaps). Semantics restated in SURVEY.md App. A.4-A.5 and, as the
// parity oracle, in oracle/spoa_graph.cpp + oracle/racon_window.cpp.
//
// One warp per window, many windows in flight (the graph surgery between two
// layers is sequential pointer work; occupancy hides its latency):
//   * lane 0 keeps the partial order graph (nodes, in/out edge lists in
//     insertion order, aligned-node sets, per-node sequence counts) in a
//     per-window scratch slab, extracts the sub-graph a partial layer aligns
//     to, and sorts it topologically exactly like spoa's DFS;
//   * all 32 lanes fill the DP rows: coalesced int16 rows, the diagonal
//     neighbour through a shuffle, and the horizontal gap recurrence
//     H[i][j] = max(M[j], H[i][j-1] + g) solved as a warp max-scan of
//     M[j] - j*g (exact in integers);
//   * lane 0 walks the traceback with spoa's preference (diagonal over
//     predecessors in in-edge order, then vertical, then horizontal), merges
//     the layer into the graph, and finally runs the heaviest-bundle consensus
//     with branch completion and the coverage-based TGS trimming.
// A node's Coverage() (distinct sequence labels on its incident edges) equals
// the number of sequences (of >= 2 bases) whose path visits it, so a per-node
// counter replaces spoa's per-edge label lists.
// No tensor-core work exists here (no dense contraction).
#include <algorithm>

#include "engine.cuh"

namespace rvn {

namespace {

constexpr uint16_t kNone = 0xFFFF;
constexpr int kPoaStatusOk = 1;        // polished
constexpr int kPoaStatusChimeric = 2;  // trimming skipped (racon's warning)
constexpr int kPoaStatusCapacity = 64; // scratch too small: host retries bigger
constexpr int kPoaStatusInvalid = 128; // bad layer coordinates / letters
constexpr uint32_t kPoaMaxLayers = 4095;  // kept layers of one window (16-bit order slots)

struct PoaShape {
  uint32_t ncap;   // node capacity
  uint32_t ecap;   // edge capacity
  uint32_t lmax;   // longest layer
  uint32_t rows;   // DP rows = ncap + 1
  uint32_t width;  // DP row stride (lmax + 1 rounded up to 32)
};

// The two widths of the generic kernel: one definition of PoaKernel and its helpers,
// instantiated for each.
//   PoaNarrow: 16-bit node, edge and order ids and coverage, int16 layer positions and
//     DP cells - every window of the default contract (65000 window bases, 32000 layer
//     bases, 4095 layers, 65000 nodes or edges, the int16 score guard).
//   PoaWide: 32-bit ids, positions and coverage, int32 cells - the windows past those
//     limits (option "poa_wide"); its order slots are sized per launch.
struct PoaNarrow {
  using Id = uint16_t;   // node, edge, order and stack slots; coverage
  using Pos = int16_t;   // traceback node / layer position, -1 = gap
  using Cell = int16_t;  // DP cell
  using Shape = PoaShape;
  static constexpr Id kNone = 0xFFFF;
  // |score| <= max(|m|,|n|,|g|) * (rows + len + 2) must stay below this
  static constexpr long long kCellLimit = 32000;
  static constexpr int kNoCell = -1000000;     // M of a column past the layer
  static constexpr int kNoScan = -1000000000;  // scan value of a lane past the layer
  __host__ __device__ static uint32_t Layers(const Shape&) { return kPoaMaxLayers; }
};

struct PoaWideShape : PoaShape {
  uint32_t layers;  // order slots: the most kept layers of a window of the launch
};

struct PoaWide {
  using Id = uint32_t;
  using Pos = int32_t;
  using Cell = int32_t;
  using Shape = PoaWideShape;
  static constexpr Id kNone = 0xFFFFFFFFu;
  // far beyond any window (2^28 / 127 > 2 million rows + bases) and far inside int32
  static constexpr long long kCellLimit = 1LL << 28;
  static constexpr int kNoCell = -(1 << 29);
  static constexpr int kNoScan = -(1 << 30);
  __host__ __device__ static uint32_t Layers(const Shape& s) { return s.layers; }
};

// byte offsets of the arrays inside one window's scratch slab
struct PoaLayout {
  size_t code, n_aligned, marks, ignored, in_sub, sink;
  size_t in_head, in_tail, out_head, aligned, cov, r2n, n2r, stack, order;
  size_t e_tail, e_head, e_next_in, e_next_out, e_weight;
  size_t aln_node, aln_pos, pred, score, H, bytes;
};

template <class W>
__host__ __device__ inline PoaLayout MakePoaLayout(const typename W::Shape& s) {
  constexpr size_t id = sizeof(typename W::Id), pos = sizeof(typename W::Pos);
  PoaLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    size_t at = o;
    o += (bytes + 15) & ~size_t(15);
    return at;
  };
  L.code = take(s.ncap);
  L.n_aligned = take(s.ncap);
  L.marks = take(s.ncap);
  L.ignored = take(s.ncap);
  L.in_sub = take(s.ncap);
  L.sink = take(s.ncap);
  L.in_head = take(id * s.ncap);
  L.in_tail = take(id * s.ncap);
  L.out_head = take(id * s.ncap);
  L.aligned = take(id * 3 * s.ncap);
  L.cov = take(id * s.ncap);
  L.r2n = take(id * s.ncap);
  L.n2r = take(id * s.ncap);
  L.stack = take(id * 4 * s.ncap);
  L.order = take(id * (W::Layers(s) + 1));
  L.e_tail = take(id * s.ecap);
  L.e_head = take(id * s.ecap);
  L.e_next_in = take(id * s.ecap);
  L.e_next_out = take(id * s.ecap);
  L.e_weight = take(4ULL * s.ecap);
  L.aln_node = take(pos * (s.ncap + s.lmax + 2));
  L.aln_pos = take(pos * (s.ncap + s.lmax + 2));
  L.pred = take(4ULL * s.ncap);
  L.score = take(8ULL * s.ncap);
  L.H = take(sizeof(typename W::Cell) * s.rows * s.width);
  L.bytes = o;
  return L;
}

template <class W>
struct PoaGraph {
  using Id = typename W::Id;
  uint8_t *code, *n_aligned, *marks, *ignored, *in_sub, *sink;
  Id *in_head, *in_tail, *out_head, *aligned, *cov, *r2n, *n2r, *stack, *order;
  Id *e_tail, *e_head, *e_next_in, *e_next_out;
  int32_t* e_weight;
  typename W::Pos *aln_node, *aln_pos;
  int32_t* pred;
  long long* score;
  typename W::Cell* H;
  uint32_t n_nodes, n_edges, ncap, ecap, stack_cap;
  bool overflow;
};

// Upper-case ACGT only, which is all racon passes. spoa codes letters as they
// come (a lower-case letter is a fifth letter there and is printed as given), so
// anything else has no code here and fails the window.
__device__ __forceinline__ int CodeOf(uint8_t c) {
  switch (c) {
    case 'A': return 0;
    case 'C': return 1;
    case 'G': return 2;
    case 'T': return 3;
    default: return -1;
  }
}

// racon::Window::AddLayer drops a layer without bases or with begin == end
// before it looks at anything else: such an entry is not a sequence of its
// window. It does not count for "fewer than 3 sequences" or for the trimming
// threshold, and its coordinates are never checked.
__host__ __device__ inline bool LayerKept(const uint64_t* seq_off, const uint32_t* seq_begin,
                                          const uint32_t* seq_end, uint32_t s) {
  return seq_off[s + 1] != seq_off[s] && seq_begin[s] != seq_end[s];
}

// (all lanes) the sequences of window [s0, s1) under that rule, backbone included
__device__ uint32_t KeptSequences(const uint64_t* seq_off, const uint32_t* seq_begin,
                                  const uint32_t* seq_end, uint32_t s0, uint32_t s1,
                                  uint32_t lane) {
  uint32_t kept = 0;
  for (uint32_t s = s0 + 1 + lane; s < s1; s += 32) {
    kept += LayerKept(seq_off, seq_begin, seq_end, s);
  }
  return 1 + __reduce_add_sync(0xffffffffu, kept);
}

// (lane 0) order[] = the kept layers of the window as offsets from s0, by begin
// position, stable (equal begins keep their arrival order). Returns 0, or the
// status that ends the window: racon's coordinate check (with end < L0, as a
// layer's end is a node of the backbone chain), a layer beyond `lmax` bases, or
// more layers than order[] holds (PoaBatch refuses those before any launch).
template <class Order>
__device__ uint32_t OrderLayers(Order* order, const uint64_t* seq_off,
                                const uint32_t* seq_begin, const uint32_t* seq_end,
                                uint32_t s0, uint32_t s1, uint32_t L0, uint32_t lmax,
                                uint32_t max_layers = kPoaMaxLayers) {
  uint32_t n = 0;
  for (uint32_t s = s0 + 1; s < s1; ++s) {
    if (!LayerKept(seq_off, seq_begin, seq_end, s)) continue;
    if (n >= max_layers) return kPoaStatusCapacity;
    if (seq_begin[s] > seq_end[s] || seq_end[s] >= L0) return kPoaStatusInvalid;
    if (seq_off[s + 1] - seq_off[s] > lmax) return kPoaStatusInvalid;
    uint32_t b = n++;
    while (b > 0 && seq_begin[s0 + order[b - 1]] > seq_begin[s]) {
      order[b] = order[b - 1];
      --b;
    }
    order[b] = static_cast<Order>(s - s0);
  }
  return 0;
}

template <class W>
__device__ typename W::Id AddNode(PoaGraph<W>& g, uint32_t code) {
  if (g.n_nodes >= g.ncap) {
    g.overflow = true;
    return 0;
  }
  const uint32_t v = g.n_nodes++;
  g.code[v] = static_cast<uint8_t>(code);
  g.n_aligned[v] = 0;
  g.in_head[v] = g.in_tail[v] = g.out_head[v] = W::kNone;
  g.cov[v] = 0;
  return static_cast<typename W::Id>(v);
}

// spoa Graph::AddEdge: bump the weight of an existing edge or append a new
// one at the END of both adjacency lists (insertion order is observable)
template <class W>
__device__ void AddEdge(PoaGraph<W>& g, typename W::Id tail, typename W::Id head, int32_t w) {
  using Id = typename W::Id;
  Id last_out = W::kNone;
  for (Id e = g.out_head[tail]; e != W::kNone; e = g.e_next_out[e]) {
    if (g.e_head[e] == head) {
      g.e_weight[e] += w;
      return;
    }
    last_out = e;
  }
  if (g.n_edges >= g.ecap) {
    g.overflow = true;
    return;
  }
  const Id e = static_cast<Id>(g.n_edges++);
  g.e_tail[e] = tail;
  g.e_head[e] = head;
  g.e_weight[e] = w;
  g.e_next_in[e] = g.e_next_out[e] = W::kNone;
  if (last_out == W::kNone) {
    g.out_head[tail] = e;
  } else {
    g.e_next_out[last_out] = e;
  }
  if (g.in_head[head] == W::kNone) {
    g.in_head[head] = e;
  } else {
    g.e_next_in[g.in_tail[head]] = e;
  }
  g.in_tail[head] = e;
}

struct SeqView {
  const uint8_t* bases;
  const uint8_t* quals;  // nullptr = constant weight
  uint32_t len;
  int32_t flat;          // weight without qualities: layers 1, backbone 0
  __device__ __forceinline__ int32_t weight(uint32_t i) const {
    return quals ? static_cast<int32_t>(quals[i]) - 33 : flat;
  }
};

// a chain of fresh nodes for s[begin, end); returns its first node or W::kNone
template <class W>
__device__ typename W::Id AddChain(PoaGraph<W>& g, const SeqView& s, uint32_t begin,
                                   uint32_t end) {
  using Id = typename W::Id;
  if (begin == end) return W::kNone;
  Id first = W::kNone, prev = W::kNone;
  for (uint32_t i = begin; i < end && !g.overflow; ++i) {
    const Id cur = AddNode(g, CodeOf(s.bases[i]));
    if (prev != W::kNone) AddEdge(g, prev, cur, s.weight(i - 1) + s.weight(i));
    if (first == W::kNone) first = cur;
    prev = cur;
  }
  return first;
}

// spoa Graph::TopologicalSort restricted to the nodes with in_sub != 0
// (Graph::Subgraph keeps relative ids and adjacency order, so the restricted
// DFS over the full graph yields exactly the sub-graph's order)
template <class W>
__device__ uint32_t TopoSort(PoaGraph<W>& g) {
  using Id = typename W::Id;
  const uint32_t n = g.n_nodes;
  for (uint32_t v = 0; v < n; ++v) {
    g.marks[v] = 0;
    g.ignored[v] = 0;
  }
  uint32_t rank = 0, sp = 0;
  for (uint32_t root = 0; root < n; ++root) {
    if (!g.in_sub[root] || g.marks[root] != 0) continue;
    g.stack[sp++] = static_cast<Id>(root);
    while (sp > 0) {
      const Id cur = g.stack[sp - 1];
      bool valid = true;
      if (g.marks[cur] != 2) {
        for (Id e = g.in_head[cur]; e != W::kNone; e = g.e_next_in[e]) {
          const Id t = g.e_tail[e];
          if (g.in_sub[t] && g.marks[t] != 2) {
            if (sp >= g.stack_cap) {
              g.overflow = true;
              return 0;
            }
            g.stack[sp++] = t;
            valid = false;
          }
        }
        if (!g.ignored[cur]) {
          for (uint32_t a = 0; a < g.n_aligned[cur]; ++a) {
            const Id t = g.aligned[3 * cur + a];
            if (g.in_sub[t] && g.marks[t] != 2) {
              if (sp >= g.stack_cap) {
                g.overflow = true;
                return 0;
              }
              g.stack[sp++] = t;
              g.ignored[t] = 1;
              valid = false;
            }
          }
        }
        if (valid) {
          g.marks[cur] = 2;
          if (!g.ignored[cur]) {
            g.n2r[cur] = static_cast<Id>(rank);
            g.r2n[rank++] = cur;
            for (uint32_t a = 0; a < g.n_aligned[cur]; ++a) {
              const Id t = g.aligned[3 * cur + a];
              if (g.in_sub[t]) {
                g.n2r[t] = static_cast<Id>(rank);
                g.r2n[rank++] = t;
              }
            }
          }
        } else {
          g.marks[cur] = 1;
        }
      }
      if (valid) --sp;
    }
  }
  return rank;
}

// spoa Graph::ExtractSubgraph(nodes[end], nodes[begin]): backward reachability
// from `from` through in-edges and aligned nodes, keeping ids >= min_id
template <class W>
__device__ void MarkSubgraph(PoaGraph<W>& g, uint32_t from, uint32_t min_id) {
  using Id = typename W::Id;
  for (uint32_t v = 0; v < g.n_nodes; ++v) g.in_sub[v] = 0;
  uint32_t sp = 0;
  g.stack[sp++] = static_cast<Id>(from);
  while (sp > 0) {
    const Id cur = g.stack[--sp];
    if (g.in_sub[cur] || cur < min_id) continue;
    for (Id e = g.in_head[cur]; e != W::kNone; e = g.e_next_in[e]) {
      if (sp >= g.stack_cap) {
        g.overflow = true;
        return;
      }
      g.stack[sp++] = g.e_tail[e];
    }
    for (uint32_t a = 0; a < g.n_aligned[cur]; ++a) {
      if (sp >= g.stack_cap) {
        g.overflow = true;
        return;
      }
      g.stack[sp++] = g.aligned[3 * cur + a];
    }
    g.in_sub[cur] = 1;
  }
}

// spoa Graph::AddAlignment (alignment non-empty)
template <class W>
__device__ void AddAlignment(PoaGraph<W>& g, const SeqView& s, uint32_t aln_len) {
  using Id = typename W::Id;
  // valid = sequence positions that appear in the alignment
  int32_t first_pos = -1, last_pos = -1;
  for (uint32_t i = 0; i < aln_len; ++i) {
    if (g.aln_pos[i] != -1) {
      if (first_pos < 0) first_pos = g.aln_pos[i];
      last_pos = g.aln_pos[i];
    }
  }
  const uint32_t before = g.n_nodes;
  Id begin = AddChain(g, s, 0, first_pos);
  Id prev = before == g.n_nodes ? W::kNone : static_cast<Id>(g.n_nodes - 1);
  const Id last = AddChain(g, s, last_pos + 1, s.len);
  // count this sequence on the chains (coverage = sequences through a node)
  const bool counts = s.len >= 2;
  if (counts) {
    for (uint32_t v = before; v < g.n_nodes; ++v) g.cov[v] += 1;
  }
  for (uint32_t i = 0; i < aln_len && !g.overflow; ++i) {
    const int32_t pos = g.aln_pos[i];
    if (pos == -1) continue;
    const uint32_t code = CodeOf(s.bases[pos]);
    Id cur = W::kNone;
    if (g.aln_node[i] == -1) {
      cur = AddNode(g, code);
    } else {
      const Id jt = static_cast<Id>(g.aln_node[i]);
      if (g.code[jt] == code) {
        cur = jt;
      } else {
        for (uint32_t a = 0; a < g.n_aligned[jt]; ++a) {
          const Id kt = g.aligned[3 * jt + a];
          if (g.code[kt] == code) {
            cur = kt;
            break;
          }
        }
        if (cur == W::kNone) {  // a new letter for this column
          cur = AddNode(g, code);
          if (g.overflow) break;
          const uint32_t na = g.n_aligned[jt];
          for (uint32_t a = 0; a < na; ++a) {
            const Id kt = g.aligned[3 * jt + a];
            g.aligned[3 * kt + g.n_aligned[kt]++] = cur;
            g.aligned[3 * cur + g.n_aligned[cur]++] = kt;
          }
          g.aligned[3 * jt + g.n_aligned[jt]++] = cur;
          g.aligned[3 * cur + g.n_aligned[cur]++] = jt;
        }
      }
    }
    if (g.overflow) break;
    if (counts) g.cov[cur] += 1;
    if (begin == W::kNone) begin = cur;
    if (prev != W::kNone) AddEdge(g, prev, cur, s.weight(pos - 1) + s.weight(pos));
    prev = cur;
  }
  if (last != W::kNone && !g.overflow) {
    AddEdge(g, prev, last, s.weight(last_pos) + s.weight(last_pos + 1));
  }
}

template <class W>
__global__ void __launch_bounds__(32)
PoaKernel(uint32_t n_windows, const uint32_t* __restrict__ win_list,
          const uint32_t* __restrict__ win_first, const uint64_t* __restrict__ seq_off,
          const uint8_t* __restrict__ bases, const uint8_t* __restrict__ quals,
          const uint32_t* __restrict__ seq_begin, const uint32_t* __restrict__ seq_end,
          int m, int n, int gap, int trim, int tgs, typename W::Shape shape,
          uint8_t* __restrict__ scratch, size_t scratch_stride,
          uint8_t* __restrict__ cons, const uint64_t* __restrict__ cons_off,
          uint32_t* __restrict__ cons_len, uint32_t* __restrict__ cov_out,
          uint8_t* __restrict__ status, unsigned long long* __restrict__ cells) {
  using Id = typename W::Id;
  using Pos = typename W::Pos;
  using Cell = typename W::Cell;
  if (blockIdx.x >= n_windows) return;
  const uint32_t lane = threadIdx.x;
  const uint32_t w = win_list ? win_list[blockIdx.x] : blockIdx.x;
  const uint32_t s0 = win_first[w], s1 = win_first[w + 1];
  const uint32_t nseq = KeptSequences(seq_off, seq_begin, seq_end, s0, s1, lane);
  const uint32_t L0 = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
  uint8_t* out = cons + cons_off[w];
  uint32_t* cov_dst = cov_out ? cov_out + cons_off[w] : nullptr;

  if (nseq < 3) {  // fewer than 3 sequences: the backbone, "unpolished"
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

  // only ACGT letters are valid (racon feeds 2-bit reads)
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
  const PoaLayout L = MakePoaLayout<W>(shape);
  __shared__ PoaGraph<W> g;
  __shared__ uint32_t sh_rows, sh_fail;
  if (lane == 0) {
    g.code = base + L.code;
    g.n_aligned = base + L.n_aligned;
    g.marks = base + L.marks;
    g.ignored = base + L.ignored;
    g.in_sub = base + L.in_sub;
    g.sink = base + L.sink;
    g.in_head = reinterpret_cast<Id*>(base + L.in_head);
    g.in_tail = reinterpret_cast<Id*>(base + L.in_tail);
    g.out_head = reinterpret_cast<Id*>(base + L.out_head);
    g.aligned = reinterpret_cast<Id*>(base + L.aligned);
    g.cov = reinterpret_cast<Id*>(base + L.cov);
    g.r2n = reinterpret_cast<Id*>(base + L.r2n);
    g.n2r = reinterpret_cast<Id*>(base + L.n2r);
    g.stack = reinterpret_cast<Id*>(base + L.stack);
    g.order = reinterpret_cast<Id*>(base + L.order);
    g.e_tail = reinterpret_cast<Id*>(base + L.e_tail);
    g.e_head = reinterpret_cast<Id*>(base + L.e_head);
    g.e_next_in = reinterpret_cast<Id*>(base + L.e_next_in);
    g.e_next_out = reinterpret_cast<Id*>(base + L.e_next_out);
    g.e_weight = reinterpret_cast<int32_t*>(base + L.e_weight);
    g.aln_node = reinterpret_cast<Pos*>(base + L.aln_node);
    g.aln_pos = reinterpret_cast<Pos*>(base + L.aln_pos);
    g.pred = reinterpret_cast<int32_t*>(base + L.pred);
    g.score = reinterpret_cast<long long*>(base + L.score);
    g.H = reinterpret_cast<Cell*>(base + L.H);
    g.n_nodes = g.n_edges = 0;
    g.ncap = shape.ncap;
    g.ecap = shape.ecap;
    g.stack_cap = 4 * shape.ncap;
    g.overflow = false;
    // layer coordinates are validated up front
    sh_fail = OrderLayers(g.order, seq_off, seq_begin, seq_end, s0, s1, L0, shape.lmax,
                          W::Layers(shape));
    if (!sh_fail) {
      // backbone chain (spoa AddAlignment with an empty alignment): its edges weigh
      // by its own qualities when the batch has qualities, and 0 when it has none
      SeqView bb{bases + seq_off[s0], quals ? quals + seq_off[s0] : nullptr, L0, 0};
      AddChain(g, bb, 0, L0);
      if (L0 >= 2) {
        for (uint32_t v = 0; v < g.n_nodes; ++v) g.cov[v] += 1;
      }
    }
  }
  __syncwarp();

  const uint32_t offset = static_cast<uint32_t>(0.01 * L0);
  const uint32_t width = shape.width;
  unsigned long long my_cells = 0;

  for (uint32_t li = 0; li + 1 < nseq; ++li) {
    if (sh_fail || g.overflow) break;
    const uint32_t s = s0 + g.order[li];
    const SeqView sv{bases + seq_off[s], quals ? quals + seq_off[s] : nullptr,
                     static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]), 1};
    const uint32_t len = sv.len;

    // ---- (lane 0) the graph this layer aligns to, in topological order ----
    if (lane == 0) {
      const uint32_t lb = seq_begin[s], le = seq_end[s];
      if (lb < offset && le > L0 - offset) {
        for (uint32_t v = 0; v < g.n_nodes; ++v) g.in_sub[v] = 1;
      } else {
        MarkSubgraph(g, le, lb);
      }
      uint32_t rows = g.overflow ? 0 : TopoSort(g);
      // a node is a sink if it has no out-edge inside the (sub)graph
      for (uint32_t r = 0; r < rows; ++r) {
        const Id v = g.r2n[r];
        uint8_t sink = 1;
        for (Id e = g.out_head[v]; e != W::kNone; e = g.e_next_out[e]) {
          if (g.in_sub[g.e_head[e]]) {
            sink = 0;
            break;
          }
        }
        g.sink[v] = sink;
      }
      // the cells' range: |score| <= max|m,n,g| * (rows + columns)
      const int amax = max(max(abs(m), abs(n)), abs(gap));
      if (static_cast<long long>(amax) * (rows + len + 2) > W::kCellLimit) g.overflow = true;
      sh_rows = rows;
    }
    __syncwarp();
    const uint32_t rows = sh_rows;
    if (g.overflow) break;
    my_cells += static_cast<unsigned long long>(rows + 1) * (len + 1);

    // ---- DP (all lanes) ----
    Cell* H = g.H;
    for (uint32_t j = lane; j <= len; j += 32) H[j] = static_cast<Cell>(j * gap);
    __syncwarp();
    int best_score = -2147483647, best_row = -1;
    for (uint32_t r = 0; r < rows; ++r) {
      const Id v = g.r2n[r];
      const uint32_t vcode = g.code[v];
      Cell* row = H + static_cast<size_t>(r + 1) * width;
      // column 0
      int col0 = 0;
      {
        bool any = false;
        int pen = -2147483647;
        for (Id e = g.in_head[v]; e != W::kNone; e = g.e_next_in[e]) {
          const Id t = g.e_tail[e];
          if (!g.in_sub[t]) continue;
          any = true;
          pen = max(pen, static_cast<int>(H[static_cast<size_t>(g.n2r[t] + 1) * width]));
        }
        col0 = (any ? pen : 0) + gap;
      }
      int carry = col0;  // running max of M[k] - k*g over k < chunk start (k = 0 term)
      for (uint32_t c0 = 1; c0 <= len; c0 += 32) {
        const uint32_t j = c0 + lane;
        int M = W::kNoCell;
        if (j <= len) {
          const int match = (static_cast<uint32_t>(CodeOf(sv.bases[j - 1])) == vcode) ? m : n;
          bool any = false;
          for (Id e = g.in_head[v]; e != W::kNone; e = g.e_next_in[e]) {
            const Id t = g.e_tail[e];
            if (!g.in_sub[t]) continue;
            any = true;
            const Cell* pr = H + static_cast<size_t>(g.n2r[t] + 1) * width;
            M = max(M, max(static_cast<int>(pr[j - 1]) + match,
                           static_cast<int>(pr[j]) + gap));
          }
          if (!any) {
            M = max(static_cast<int>(H[j - 1]) + match, static_cast<int>(H[j]) + gap);
          }
        }
        // horizontal recurrence as a max-scan of T = M - j*g
        int T = j <= len ? M - static_cast<int>(j) * gap : W::kNoScan;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int o = __shfl_up_sync(0xffffffffu, T, d);
          if (static_cast<int>(lane) >= d) T = max(T, o);
        }
        T = max(T, carry);
        if (j <= len) row[j] = static_cast<Cell>(T + static_cast<int>(j) * gap);
        carry = __shfl_sync(0xffffffffu, T, 31);
      }
      if (lane == 0) row[0] = static_cast<Cell>(col0);
      __syncwarp();
      if (g.sink[v]) {
        const int sc = row[len];
        if (best_score < sc) {
          best_score = sc;
          best_row = static_cast<int>(r + 1);
        }
      }
    }

    // ---- (lane 0) traceback + merge ----
    if (lane == 0) {
      uint32_t alen = 0;
      uint32_t i = best_row < 0 ? 0 : static_cast<uint32_t>(best_row), j = len;
      if (best_row < 0) j = 0;
      const uint32_t acap = shape.ncap + shape.lmax + 2;
      while (!(i == 0 && j == 0)) {
        const int h = H[static_cast<size_t>(i) * width + j];
        uint32_t pi = 0, pj = 0;
        bool found = false;
        if (i != 0 && j != 0) {
          const Id v = g.r2n[i - 1];
          const int match =
              (static_cast<uint32_t>(CodeOf(sv.bases[j - 1])) == g.code[v]) ? m : n;
          bool any = false;
          for (Id e = g.in_head[v]; e != W::kNone && !found; e = g.e_next_in[e]) {
            const Id t = g.e_tail[e];
            if (!g.in_sub[t]) continue;
            any = true;
            const uint32_t p = g.n2r[t] + 1;
            if (h == H[static_cast<size_t>(p) * width + (j - 1)] + match) {
              pi = p;
              pj = j - 1;
              found = true;
            }
          }
          if (!any && h == H[j - 1] + match) {
            pi = 0;
            pj = j - 1;
            found = true;
          }
        }
        if (!found && i != 0) {
          const Id v = g.r2n[i - 1];
          bool any = false;
          for (Id e = g.in_head[v]; e != W::kNone && !found; e = g.e_next_in[e]) {
            const Id t = g.e_tail[e];
            if (!g.in_sub[t]) continue;
            any = true;
            const uint32_t p = g.n2r[t] + 1;
            if (h == H[static_cast<size_t>(p) * width + j] + gap) {
              pi = p;
              pj = j;
              found = true;
            }
          }
          if (!any && h == H[j] + gap) {
            pi = 0;
            pj = j;
            found = true;
          }
        }
        if (!found && j != 0 && h == H[static_cast<size_t>(i) * width + j - 1] + gap) {
          pi = i;
          pj = j - 1;
          found = true;
        }
        if (!found || alen >= acap) {  // cannot happen for a consistent matrix
          g.overflow = true;
          break;
        }
        g.aln_node[alen] = i == pi ? -1 : static_cast<Pos>(g.r2n[i - 1]);
        g.aln_pos[alen] = j == pj ? -1 : static_cast<Pos>(j - 1);
        ++alen;
        i = pi;
        j = pj;
      }
      // reverse into emission order
      for (uint32_t a = 0; a < alen / 2; ++a) {
        const Pos tn = g.aln_node[a], tp = g.aln_pos[a];
        g.aln_node[a] = g.aln_node[alen - 1 - a];
        g.aln_pos[a] = g.aln_pos[alen - 1 - a];
        g.aln_node[alen - 1 - a] = tn;
        g.aln_pos[alen - 1 - a] = tp;
      }
      if (!g.overflow) {
        if (alen == 0) {
          // spoa: an empty alignment appends the sequence as a separate chain
          const uint32_t before = g.n_nodes;
          AddChain(g, sv, 0, sv.len);
          if (sv.len >= 2) {
            for (uint32_t v = before; v < g.n_nodes; ++v) g.cov[v] += 1;
          }
        } else {
          AddAlignment(g, sv, alen);
        }
      }
    }
    __syncwarp();
  }

  // ---- (lane 0) consensus: heaviest bundle + branch completion + trimming ----
  if (lane == 0) {
    uint32_t st = 0;
    uint32_t clen = 0;
    if (sh_fail) {
      st = sh_fail;
    } else if (g.overflow) {
      st = kPoaStatusCapacity;
    } else {
      for (uint32_t v = 0; v < g.n_nodes; ++v) g.in_sub[v] = 1;
      const uint32_t rows = TopoSort(g);
      if (g.overflow) {
        st = kPoaStatusCapacity;
      } else {
        for (uint32_t v = 0; v < g.n_nodes; ++v) {
          g.pred[v] = -1;
          g.score[v] = -1;
        }
        auto relax = [&](Id v) {
          for (Id e = g.in_head[v]; e != W::kNone; e = g.e_next_in[e]) {
            const Id t = g.e_tail[e];
            const long long wgt = g.e_weight[e];
            if (g.score[v] < wgt ||
                (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
              g.score[v] = wgt;
              g.pred[v] = t;
            }
          }
          if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
        };
        int32_t mx = -1;
        for (uint32_t r = 0; r < rows; ++r) {
          const Id v = g.r2n[r];
          relax(v);
          if (mx < 0 || g.score[mx] < g.score[v]) mx = v;
        }
        while (g.out_head[mx] != W::kNone) {  // branch completion
          const uint32_t rank = g.n2r[mx];
          for (Id e = g.out_head[mx]; e != W::kNone; e = g.e_next_out[e]) {
            const Id hd = g.e_head[e];
            for (Id f = g.in_head[hd]; f != W::kNone; f = g.e_next_in[f]) {
              if (g.e_tail[f] != mx) g.score[g.e_tail[f]] = -1;
            }
          }
          int32_t nmx = -1;
          for (uint32_t r = rank + 1; r < rows; ++r) {
            const Id v = g.r2n[r];
            g.score[v] = -1;
            g.pred[v] = -1;
            for (Id e = g.in_head[v]; e != W::kNone; e = g.e_next_in[e]) {
              const Id t = g.e_tail[e];
              if (g.score[t] == -1) continue;
              const long long wgt = g.e_weight[e];
              if (g.score[v] < wgt ||
                  (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
                g.score[v] = wgt;
                g.pred[v] = t;
              }
            }
            if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
            if (nmx < 0 || g.score[nmx] < g.score[v]) nmx = v;
          }
          mx = nmx;
        }
        // walk back; r2n is free now and holds the reversed path
        uint32_t plen = 0;
        int32_t v = mx;
        while (g.pred[v] != -1) {
          g.r2n[plen++] = static_cast<Id>(v);
          v = g.pred[v];
        }
        g.r2n[plen++] = static_cast<Id>(v);
        // coverage of a consensus base = its node + the aligned nodes
        auto coverage = [&](uint32_t idx) -> uint32_t {
          const Id nd = g.r2n[plen - 1 - idx];
          uint32_t cvg = g.cov[nd];
          for (uint32_t a = 0; a < g.n_aligned[nd]; ++a) cvg += g.cov[g.aligned[3 * nd + a]];
          return cvg;
        };
        uint32_t cb = 0, ce = plen;  // [cb, ce)
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
          const Id nd = g.r2n[plen - 1 - (cb + i)];
          out[i] = "ACGT"[g.code[nd]];
          if (cov_dst) cov_dst[i] = coverage(cb + i);
        }
      }
    }
    cons_len[w] = clen;
    status[w] = static_cast<uint8_t>(st);
    // DP cells of this window (lanes hold the same count); an attempt that ran out
    // of capacity is run again and counted then
    if (cells && st != kPoaStatusCapacity) atomicAdd(cells, my_cells);
  }
}

}  // namespace
}  // namespace rvn

#include "poa_fast.cuh"

namespace rvn {

namespace {

// scratch of one launch: up to 16 GB, at most half of what the device has left (the
// stage-1 buffers of the same context stay resident on an 80 GB card), or option
// "poa_scratch_budget"
size_t PoaScratchBudget(Ctx& c) {
  if (c.poa_scratch_budget) return c.poa_scratch_budget;
  size_t free_b = 0, total_b = 0;
  RVN_CUDA(cudaMemGetInfo(&free_b, &total_b));
  return std::min<size_t>(16ULL << 30, (free_b + c.po_scratch.cap) / 2);
}

// The windows `todo` on PoaKernel<PoaWide>. A window's node capacity starts at an
// estimate (the first tier's, plus 1/16 of its layer bases for the columns the layers
// open) and doubles while the window reports kPoaStatusCapacity, up to its bases (every
// node holds one base of the window). Edges: 3 per node, and never more than the bases.
// Each round sorts the windows by scratch and launches runs of them that fit the budget
// at the largest shape of the run.
struct PoaWindowDims {
  const std::vector<uint32_t>& lmax;
  const std::vector<uint32_t>& bb;
  const std::vector<uint32_t>& kept;
  const std::vector<uint64_t>& tot;
};

void PoaWideRun(Ctx& c, std::vector<uint32_t> todo, const PoaWindowDims& d,
                uint32_t n_windows, const uint32_t* d_wf, const uint64_t* d_so,
                const uint8_t* d_bases, const uint8_t* d_quals, const uint32_t* d_sb,
                const uint32_t* d_se, int m, int n, int gap, bool trim, bool tgs,
                uint8_t* d_cons, const uint64_t* d_coff, uint32_t* d_clen, uint32_t* d_cov,
                uint8_t* d_status, uint64_t* d_cells) {
  std::vector<uint64_t> ncap(n_windows, 0);
  for (uint32_t w : todo) {
    ncap[w] = std::min<uint64_t>(d.tot[w], 3ULL * d.bb[w] + d.lmax[w] + 64 + d.tot[w] / 16);
  }
  const auto shape_of = [&](uint32_t w) {
    PoaWideShape s;
    s.ncap = static_cast<uint32_t>(ncap[w]);
    s.ecap = static_cast<uint32_t>(std::min<uint64_t>(3 * ncap[w], d.tot[w]));
    s.lmax = d.lmax[w];
    s.rows = s.ncap + 1;
    s.width = (s.lmax + 1 + 31) & ~31u;
    s.layers = d.kept[w];
    return s;
  };
  const auto widest = [](PoaWideShape a, const PoaWideShape& b) {
    a.ncap = std::max(a.ncap, b.ncap);
    a.ecap = std::max(a.ecap, b.ecap);
    a.lmax = std::max(a.lmax, b.lmax);
    a.rows = std::max(a.rows, b.rows);
    a.width = std::max(a.width, b.width);
    a.layers = std::max(a.layers, b.layers);
    return a;
  };
  const auto stride_of = [](const PoaWideShape& s) {
    return (MakePoaLayout<PoaWide>(s).bytes + 255) & ~size_t(255);
  };
  while (!todo.empty()) {
    std::vector<size_t> need(n_windows, 0);
    for (uint32_t w : todo) need[w] = stride_of(shape_of(w));
    std::stable_sort(todo.begin(), todo.end(),
                     [&](uint32_t a, uint32_t b) { return need[a] < need[b]; });
    const size_t budget = PoaScratchBudget(c);
    if (need[todo.back()] > budget) {
      throw LimitError("a POA window needs " + std::to_string(need[todo.back()]) +
                       " bytes of scratch, more than the budget of " +
                       std::to_string(budget) + " bytes");
    }
    // runs [first, first + count) of the sorted windows and their shapes
    struct Run {
      size_t first, count;
      PoaWideShape shape;
      size_t stride;
    };
    std::vector<Run> runs;
    size_t scratch_bytes = 0;
    for (size_t i = 0; i < todo.size();) {
      Run r{i, 1, shape_of(todo[i]), need[todo[i]]};
      while (i + r.count < todo.size()) {
        const PoaWideShape s = widest(r.shape, shape_of(todo[i + r.count]));
        const size_t st = stride_of(s);
        if (st * (r.count + 1) > budget) break;
        r.shape = s;
        r.stride = st;
        ++r.count;
      }
      scratch_bytes = std::max(scratch_bytes, r.stride * r.count);
      runs.push_back(r);
      i += r.count;
    }
    uint8_t* scratch = c.po_scratch.reserve(scratch_bytes);
    uint32_t* d_list = c.po_list.reserve(n_windows + 1ULL);
    RVN_CUDA(cudaMemcpyAsync(d_list, todo.data(), todo.size() * 4, cudaMemcpyHostToDevice, c.stream));
    for (const Run& r : runs) {
      PoaKernel<PoaWide><<<static_cast<uint32_t>(r.count), 32, 0, c.stream>>>(
          static_cast<uint32_t>(r.count), d_list + r.first, d_wf, d_so, d_bases, d_quals,
          d_sb, d_se, m, n, gap, trim, tgs, r.shape, scratch, r.stride, d_cons, d_coff,
          d_clen, d_cov, d_status, reinterpret_cast<unsigned long long*>(d_cells));
      RVN_LAUNCH_CHECK();
      ++c.launches;
      ++c.po_route_launches[2];
    }
    RVN_CUDA(cudaMemcpyAsync(c.po_h_status.data(), d_status, n_windows, cudaMemcpyDeviceToHost, c.stream));
    RVN_CUDA(cudaStreamSynchronize(c.stream));  // (also: todo / d_list are reusable)
    std::vector<uint32_t> again;
    for (uint32_t w : todo) {
      if (c.po_h_status[w] != kPoaStatusCapacity) continue;
      if (ncap[w] >= d.tot[w]) {  // cannot happen: the bound holds every base
        throw LimitError("a POA graph outgrew the bases of its window");
      }
      ncap[w] = std::min<uint64_t>(2 * ncap[w], d.tot[w]);
      again.push_back(w);
    }
    todo.swap(again);
  }
}

}  // namespace

// Host driver of windows whose flat layout is on the device (`d`); h_* are the host
// copies of its window and sequence tables. Windows in batches sized by the scratch
// budget; windows that outgrow the first-tier capacity are retried with the exact
// upper bound. With option "poa_wide", the windows past the 16-bit kernels' limits run
// on the wide one. Results (compacted) land in c.po_out_*, c.po_h_status, c.po_route_*.
void PoaRun(Ctx& c, uint32_t n_windows, const uint32_t* h_win_first, const uint64_t* h_seq_off,
            const uint32_t* h_seq_begin, const uint32_t* h_seq_end, const PoaInput& d, int m,
            int n, int gap, bool trim, bool tgs, bool want_coverage) {
  c.poa_valid = false;
  if (gap >= 0) {
    throw InvalidArgument("[racon::Polisher::Create] error: gap penalty must be negative");
  }
  const uint32_t* d_wf = d.win_first;
  const uint64_t* d_so = d.seq_off;
  const uint8_t* d_bases = d.bases;
  const uint8_t* d_quals = d.quals;
  const uint32_t* d_sb = d.seq_begin;
  const uint32_t* d_se = d.seq_end;

  // output slots: a consensus never has more bases than the window holds
  c.po_cons_off.assign(n_windows + 1ULL, 0);
  // per window: longest layer, backbone length, all bases - the kernel is chosen
  // PER WINDOW (one long layer must not send a whole batch to the generic kernel)
  std::vector<uint32_t> w_lmax(n_windows, 1), w_bb(n_windows, 1), w_kept(n_windows, 0);
  std::vector<uint64_t> w_tot(n_windows, 1);
  std::vector<uint8_t> w_wide(n_windows, 0);
  for (uint32_t w = 0; w < n_windows; ++w) {
    const uint32_t s0 = h_win_first[w], s1 = h_win_first[w + 1];
    uint64_t tot = 0, lmax = 0;
    uint32_t kept = 0;
    for (uint32_t s = s0; s < s1; ++s) {
      const uint64_t len = h_seq_off[s + 1] - h_seq_off[s];
      tot += len;
      if (s > s0) {
        lmax = std::max(lmax, len);
        kept += LayerKept(h_seq_off, h_seq_begin, h_seq_end, s);
      } else {
        w_bb[w] = std::max<uint32_t>(w_bb[w], static_cast<uint32_t>(len));
      }
    }
    // 16-bit node ids, int16 layer positions, 16-bit layer order slots
    const bool past = tot > 65000 || lmax > 32000 || kept > kPoaMaxLayers;
    if (c.poa_wide == 2 || (c.poa_wide == 1 && past)) {
      w_wide[w] = 1;
    } else {
      if (tot > 65000) throw LimitError("a POA window holds more than 65000 bases");
      if (lmax > 32000) throw LimitError("a layer of a POA window holds more than 32000 bases");
      if (kept > kPoaMaxLayers) throw LimitError("a POA window holds more than 4095 layers");
    }
    w_lmax[w] = std::max<uint32_t>(w_lmax[w], static_cast<uint32_t>(lmax));
    w_kept[w] = kept;
    w_tot[w] = std::max<uint64_t>(tot, 1);
    c.po_cons_off[w + 1] = c.po_cons_off[w] + tot;
  }
  const uint64_t out_total = c.po_cons_off[n_windows];
  uint64_t* d_coff = c.po_d_cons_off.reserve(n_windows + 2ULL);
  RVN_CUDA(cudaMemcpyAsync(d_coff, c.po_cons_off.data(), (n_windows + 1ULL) * 8, cudaMemcpyHostToDevice, c.stream));
  uint8_t* d_cons = c.po_cons.reserve(out_total + 16);
  uint32_t* d_cov = want_coverage ? c.po_cov.reserve(out_total + 16) : nullptr;
  uint32_t* d_clen = c.po_cons_len.reserve(n_windows + 2ULL);
  uint8_t* d_status = c.po_status.reserve(n_windows + 2ULL);
  uint64_t* d_cells = c.m_counter.reserve((1u << 16) + 8);
  RVN_CUDA(cudaMemsetAsync(d_cells, 0, 8, c.stream));
  RVN_CUDA(cudaMemsetAsync(d_status, 0, n_windows + 1ULL, c.stream));

  c.po_h_status.assign(n_windows, 0);
  std::vector<uint8_t> route(n_windows, 0);  // 0 fast, 1 generic, 2 wide
  for (int k = 0; k < 3; ++k) c.po_route_windows[k] = c.po_route_launches[k] = 0;
  TimerBegin(c, "poa");
  // group 0: every layer fits the register-row kernel; group 1: the generic kernel
  for (int group = 0; group < 2; ++group) {
    std::vector<uint32_t> todo;
    for (uint32_t w = 0; w < n_windows; ++w) {
      if (!w_wide[w] && (w_lmax[w] + 1 <= kFastCols) == (group == 0)) todo.push_back(w);
    }
    for (int tier = 0; tier < 2 && !todo.empty(); ++tier) {
      uint32_t lmax = 1, bb_max = 1;
      uint64_t total_max = 1;
      for (uint32_t w : todo) {
        lmax = std::max(lmax, w_lmax[w]);
        bb_max = std::max(bb_max, w_bb[w]);
        total_max = std::max(total_max, w_tot[w]);
      }
      PoaShape shape;
      shape.lmax = lmax;
      shape.ncap = tier == 0 ? std::min<uint64_t>(total_max, 3ULL * bb_max + lmax + 64)
                             : static_cast<uint32_t>(total_max);
      shape.ncap = std::min<uint32_t>(shape.ncap, 65000);
      shape.ecap = std::min<uint32_t>(3 * shape.ncap, 65000);
      shape.rows = shape.ncap + 1;
      shape.width = (lmax + 1 + 31) & ~31u;
      const size_t fast_smem = ((shape.ncap + 15) & ~15u) + 4ULL * shape.ncap + 16;
      const bool fast = group == 0 && fast_smem <= 220 * 1024;  // the register-row kernel
      const size_t stride = ((fast ? MakeFastLayout(shape).bytes
                                   : MakePoaLayout<PoaNarrow>(shape).bytes) +
                             255) & ~size_t(255);
      if (fast) {
        RVN_CUDA(cudaFuncSetAttribute(PoaKernelFast,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(fast_smem)));
      }
      const size_t budget = PoaScratchBudget(c);
      const uint32_t batch = static_cast<uint32_t>(
          std::max<size_t>(1, std::min<size_t>(todo.size(), budget / stride)));
      uint8_t* scratch = c.po_scratch.reserve(stride * batch);
      uint32_t* d_list = c.po_list.reserve(n_windows + 1ULL);
      RVN_CUDA(cudaMemcpyAsync(d_list, todo.data(), todo.size() * 4, cudaMemcpyHostToDevice, c.stream));
      for (size_t b0 = 0; b0 < todo.size(); b0 += batch) {
        const uint32_t nb = static_cast<uint32_t>(std::min<size_t>(batch, todo.size() - b0));
        if (fast) {
          PoaKernelFast<<<nb, 32, fast_smem, c.stream>>>(
              nb, d_list + b0, d_wf, d_so, d_bases, d_quals, d_sb, d_se, m, n, gap, trim,
              tgs, shape, scratch, stride, d_cons, d_coff, d_clen, d_cov, d_status,
              reinterpret_cast<unsigned long long*>(d_cells));
        } else {
          PoaKernel<PoaNarrow><<<nb, 32, 0, c.stream>>>(
              nb, d_list + b0, d_wf, d_so, d_bases, d_quals, d_sb, d_se, m, n, gap, trim,
              tgs, shape, scratch, stride, d_cons, d_coff, d_clen, d_cov, d_status,
              reinterpret_cast<unsigned long long*>(d_cells));
        }
        RVN_LAUNCH_CHECK();
        ++c.launches;
        ++c.po_route_launches[fast ? 0 : 1];
      }
      for (uint32_t w : todo) route[w] = fast ? 0 : 1;
      RVN_CUDA(cudaMemcpyAsync(c.po_h_status.data(), d_status, n_windows, cudaMemcpyDeviceToHost, c.stream));
      RVN_CUDA(cudaStreamSynchronize(c.stream));  // (also: todo / d_list are reusable)
      std::vector<uint32_t> again;
      for (uint32_t w : todo) {
        if (c.po_h_status[w] == kPoaStatusCapacity) again.push_back(w);
      }
      todo.swap(again);
    }
  }
  TimerEnd(c);
  // the wide kernel: windows past the 16-bit limits, and those still out of capacity
  // after the second tier (a graph beyond 65000 nodes or edges, or the int16 guard)
  std::vector<uint32_t> deep;
  for (uint32_t w = 0; w < n_windows; ++w) {
    if (w_wide[w] || (c.poa_wide && c.po_h_status[w] == kPoaStatusCapacity)) {
      deep.push_back(w);
      route[w] = 2;
    }
  }
  if (!deep.empty()) {
    TimerBegin(c, "poa_wide");
    PoaWideRun(c, deep, PoaWindowDims{w_lmax, w_bb, w_kept, w_tot}, n_windows, d_wf, d_so,
               d_bases, d_quals, d_sb, d_se, m, n, gap, trim, tgs, d_cons, d_coff, d_clen,
               d_cov, d_status, d_cells);
    TimerEnd(c);
  }
  for (uint32_t w = 0; w < n_windows; ++w) ++c.po_route_windows[route[w]];
  for (uint32_t w = 0; w < n_windows; ++w) {
    if (c.po_h_status[w] == kPoaStatusCapacity) {
      throw LimitError("a POA graph outgrew 65000 nodes/edges or the int16 score range");
    }
    if (c.po_h_status[w] == kPoaStatusInvalid) {
      throw InvalidArgument(
          "[racon::Window::AddLayer] error: layer begin and end positions are invalid");
    }
  }

  // results to the host, compacted
  TimerBegin(c, "poa_d2h");
  c.po_h_clen.assign(n_windows, 0);
  c.po_h_cons.resize(out_total);
  RVN_CUDA(cudaMemcpyAsync(c.po_h_clen.data(), d_clen, n_windows * 4ULL, cudaMemcpyDeviceToHost, c.stream));
  RVN_CUDA(cudaMemcpyAsync(c.po_h_cons.data(), d_cons, out_total, cudaMemcpyDeviceToHost, c.stream));
  if (want_coverage) {
    c.po_h_cov.resize(out_total);
    RVN_CUDA(cudaMemcpyAsync(c.po_h_cov.data(), d_cov, out_total * 4, cudaMemcpyDeviceToHost, c.stream));
  }
  c.po_cells = ReadU64(c, d_cells);
  TimerEnd(c);
  // compact the per-window slots
  c.po_out_off.assign(n_windows + 1ULL, 0);
  for (uint32_t w = 0; w < n_windows; ++w) c.po_out_off[w + 1] = c.po_out_off[w] + c.po_h_clen[w];
  c.po_out_cons.resize(c.po_out_off[n_windows]);
  if (want_coverage) c.po_out_cov.resize(c.po_out_off[n_windows]);
  for (uint32_t w = 0; w < n_windows; ++w) {
    std::copy(c.po_h_cons.begin() + c.po_cons_off[w],
              c.po_h_cons.begin() + c.po_cons_off[w] + c.po_h_clen[w],
              c.po_out_cons.begin() + c.po_out_off[w]);
    if (want_coverage) {
      std::copy(c.po_h_cov.begin() + c.po_cons_off[w],
                c.po_h_cov.begin() + c.po_cons_off[w] + c.po_h_clen[w],
                c.po_out_cov.begin() + c.po_out_off[w]);
    }
  }
  c.po_n_windows = n_windows;
  c.po_has_cov = want_coverage;
  c.poa_valid = true;
}

// rvn_poa_batch: the host's flat layout to the device, then PoaRun.
void PoaBatch(Ctx& c, uint32_t n_windows, const uint32_t* h_win_first,
              const uint64_t* h_seq_off, const uint8_t* h_bases, const uint8_t* h_quals,
              const uint32_t* h_seq_begin, const uint32_t* h_seq_end, int m, int n,
              int gap, bool trim, bool tgs, bool want_coverage) {
  c.poa_valid = false;
  if (gap >= 0) {
    throw InvalidArgument("[racon::Polisher::Create] error: gap penalty must be negative");
  }
  const uint32_t n_seqs = n_windows ? h_win_first[n_windows] : 0;
  const uint64_t n_bases = n_seqs ? h_seq_off[n_seqs] : 0;
  TimerBegin(c, "poa_h2d");
  PoaInput d;
  uint32_t* d_wf = c.po_win_first.reserve(n_windows + 2ULL);
  uint64_t* d_so = c.po_seq_off.reserve(n_seqs + 2ULL);
  uint8_t* d_bases = c.po_bases.reserve(n_bases + 16);
  uint8_t* d_quals = h_quals ? c.po_quals.reserve(n_bases + 16) : nullptr;
  uint32_t* d_sb = c.po_seq_begin.reserve(n_seqs + 2ULL);
  uint32_t* d_se = c.po_seq_end.reserve(n_seqs + 2ULL);
  RVN_CUDA(cudaMemcpyAsync(d_wf, h_win_first, (n_windows + 1ULL) * 4, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_so, h_seq_off, (n_seqs + 1ULL) * 8, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_bases, h_bases, n_bases, cudaMemcpyHostToDevice, c.stream));
  if (h_quals) RVN_CUDA(cudaMemcpyAsync(d_quals, h_quals, n_bases, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_sb, h_seq_begin, n_seqs * 4ULL, cudaMemcpyHostToDevice, c.stream));
  RVN_CUDA(cudaMemcpyAsync(d_se, h_seq_end, n_seqs * 4ULL, cudaMemcpyHostToDevice, c.stream));
  TimerEnd(c);
  d.win_first = d_wf;
  d.seq_off = d_so;
  d.bases = d_bases;
  d.quals = d_quals;
  d.seq_begin = d_sb;
  d.seq_end = d_se;
  PoaRun(c, n_windows, h_win_first, h_seq_off, h_seq_begin, h_seq_end, d, m, n, gap, trim, tgs,
         want_coverage);
}

}  // namespace rvn
