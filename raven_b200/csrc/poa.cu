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
// layers is sequential pointer work; occupancy hides its latency). Three kernels
// share one definition of the graph and of everything but the DP:
//   * lane 0 keeps the partial order graph (nodes, in/out edge lists in
//     insertion order, aligned-node sets, per-node sequence counts) as packed
//     records in a per-window scratch slab, with one flag byte per node, extracts
//     the sub-graph a partial layer aligns to, and sorts it topologically exactly
//     like spoa's DFS;
//   * all 32 lanes fill the DP rows, and lane 0 walks the traceback with spoa's
//     preference (diagonal over predecessors in in-edge order, then vertical, then
//     horizontal). These two steps are each kernel's own: PoaKernelFast
//     (poa_fast.cuh) keeps rows in registers, for layers of at most 575 bases;
//     PoaKernel fills coalesced rows, the diagonal neighbour through a shuffle and
//     the horizontal gap recurrence H[i][j] = max(M[j], H[i][j-1] + g) as a warp
//     max-scan of M[j] - j*g (exact in integers), with 16-bit (PoaNarrow) or
//     32-bit (PoaWide) ids;
//   * lane 0 merges the layer into the graph, and finally runs the heaviest-bundle
//     consensus with branch completion and the coverage-based TGS trimming.
// A node's Coverage() (distinct sequence labels on its incident edges) equals
// the number of sequences (of >= 2 bases) whose path visits it, so a per-node
// counter replaces spoa's per-edge label lists.
// No tensor-core work exists here (no dense contraction).
#include <algorithm>
#include <cstddef>
#include <cstring>
#include <type_traits>

#include "engine.cuh"

namespace rvn {

namespace {

constexpr int kPoaStatusOk = 1;        // polished
constexpr int kPoaStatusChimeric = 2;  // trimming skipped (racon's warning)
constexpr int kPoaStatusCapacity = 64; // scratch too small: host retries bigger
constexpr int kPoaStatusInvalid = 128; // bad layer coordinates / letters
constexpr uint32_t kPoaMaxLayers = 4095;  // kept layers of one window (16-bit order slots)

// the register-row kernel's DP (poa_fast.cuh): kS contiguous columns per lane
constexpr int kS = 18;
constexpr uint32_t kFastCols = 32 * kS;  // 576 = longest layer + 1
constexpr uint32_t kDirStride = 32 * 20; // bytes per direction row (20 per lane)

struct PoaShape {
  uint32_t ncap;   // node capacity
  uint32_t ecap;   // edge capacity
  uint32_t lmax;   // longest layer
  uint32_t rows;   // DP rows = ncap + 1
  uint32_t width;  // DP row stride (lmax + 1 rounded up to 32)
};

// The two widths of the graph and the consensus: one definition of each, instantiated
// for both.
//   PoaNarrow: 16-bit node, edge and order ids and coverage, int16 layer positions and
//     DP cells - every window of the default contract (65000 window bases, 32000 layer
//     bases, 4095 layers, 65000 nodes or edges, the int16 score guard). Both the
//     register-row kernel and PoaKernel<PoaNarrow> use it.
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

// Nodes and edges as packed records, so one load reads what the surgery needs of a node
// or an edge: 8 bytes each for 16-bit ids, 16 bytes for 32-bit ids.
template <class Id>
struct alignas(4 * sizeof(Id)) PoaNodeA {  // in-edge list, out-edge list, letter
  Id in_head, in_tail, out_head;
  uint8_t code, n_aligned;
};
template <class Id>
struct alignas(4 * sizeof(Id)) PoaNodeB {  // aligned nodes (one per other letter), coverage
  Id aligned[3];
  Id cov;
};
template <class Id>
struct alignas(4 * sizeof(Id)) PoaEdge {  // adjacency lists in insertion order
  Id tail, head, next_in, next_out;
};
static_assert(sizeof(PoaNodeA<uint16_t>) == 8 && offsetof(PoaNodeA<uint16_t>, code) == 6 &&
              sizeof(PoaNodeB<uint16_t>) == 8 && sizeof(PoaEdge<uint16_t>) == 8,
              "16-bit records are 8 bytes");
static_assert(sizeof(PoaNodeA<uint32_t>) == 16 && sizeof(PoaNodeB<uint32_t>) == 16 &&
              sizeof(PoaEdge<uint32_t>) == 16, "32-bit records are 16 bytes");

// one vector load / store for a whole record
template <class T>
using PoaVec = typename std::conditional<sizeof(T) == 8, uint2, uint4>::type;
template <class T>
__device__ __forceinline__ T Ld(const T* p) {
  const PoaVec<T> v = *reinterpret_cast<const PoaVec<T>*>(p);
  T t;
  memcpy(&t, &v, sizeof t);
  return t;
}
template <class T>
__device__ __forceinline__ void St(T* p, const T& t) {
  PoaVec<T> v;
  memcpy(&v, &t, sizeof v);
  *reinterpret_cast<PoaVec<T>*>(p) = v;
}
template <class Id>
__device__ __forceinline__ uint32_t AlignedAt(const PoaNodeB<Id>& b, uint32_t i) {
  return i == 0 ? b.aligned[0] : i == 1 ? b.aligned[1] : b.aligned[2];
}

// node flags: topological mark (0 new, 1 on the stack, 2 done), ignored by the sort,
// inside the (sub)graph of the layer, sink of that (sub)graph
constexpr uint8_t kMarks = 3, kIgnored = 4, kInSub = 8, kSink = 16;

// Byte offsets of the arrays inside one window's scratch slab: the graph's, then the
// kernel's own. PoaKernelFast keeps flags, r2n and n2r in shared memory and has its DP
// matrix at kFastCols columns with one direction byte per cell; PoaKernel keeps them
// here and has its matrix at shape.width columns.
struct PoaLayout {
  size_t node_a, node_b, edge, edge_w, stack, order, aln_node, aln_pos, pred, score;
  size_t flags, r2n, n2r, H, DIR, bytes;
};

template <class W>
__host__ __device__ inline PoaLayout MakePoaLayout(const typename W::Shape& s, bool fast) {
  using Id = typename W::Id;
  constexpr size_t id = sizeof(Id), pos = sizeof(typename W::Pos);
  PoaLayout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) {
    size_t at = o;
    o += (bytes + 15) & ~size_t(15);
    return at;
  };
  L.node_a = take(sizeof(PoaNodeA<Id>) * s.ncap);
  L.node_b = take(sizeof(PoaNodeB<Id>) * s.ncap);
  L.edge = take(sizeof(PoaEdge<Id>) * s.ecap);
  L.edge_w = take(4ULL * s.ecap);
  L.stack = take(id * 4 * s.ncap);
  L.order = take(id * (W::Layers(s) + 1));
  L.aln_node = take(pos * (s.ncap + s.lmax + 2));
  L.aln_pos = take(pos * (s.ncap + s.lmax + 2));
  L.pred = take(4ULL * s.ncap);
  L.score = take(8ULL * s.ncap);
  if (fast) {
    L.H = take(sizeof(typename W::Cell) * s.rows * kFastCols);
    L.DIR = take(1ULL * s.rows * kDirStride);
  } else {
    L.flags = take(s.ncap);
    L.r2n = take(id * s.ncap);
    L.n2r = take(id * s.ncap);
    L.H = take(sizeof(typename W::Cell) * s.rows * s.width);
  }
  L.bytes = o;
  return L;
}

template <class W>
struct PoaGraph {
  using Id = typename W::Id;
  PoaNodeA<Id>* node_a;
  PoaNodeB<Id>* node_b;
  PoaEdge<Id>* edge;
  int32_t* edge_w;
  Id *stack, *order;
  typename W::Pos *aln_node, *aln_pos;
  int32_t* pred;
  long long* score;
  uint8_t* flags;
  Id *r2n, *n2r;  // rank -> node and node -> rank of the last TopoSort
  typename W::Cell* H;
  uint8_t* DIR;  // PoaKernelFast only
  uint32_t n_nodes, n_edges, ncap, ecap, stack_cap;
  uint32_t rows;  // of the layer's (sub)graph
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
                                uint32_t max_layers) {
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
__device__ uint32_t AddNode(PoaGraph<W>& g, uint32_t code) {
  if (g.n_nodes >= g.ncap) {
    g.overflow = true;
    return 0;
  }
  const uint32_t v = g.n_nodes++;
  St(g.node_a + v, PoaNodeA<typename W::Id>{W::kNone, W::kNone, W::kNone,
                                            static_cast<uint8_t>(code), 0});
  St(g.node_b + v, PoaNodeB<typename W::Id>{});
  return v;
}

// spoa Graph::AddEdge: bump the weight of an existing edge or append a new
// one at the END of both adjacency lists (insertion order is observable)
template <class W>
__device__ void AddEdge(PoaGraph<W>& g, uint32_t tail, uint32_t head, int32_t w) {
  using Id = typename W::Id;
  uint32_t last_out = W::kNone;
  for (uint32_t e = Ld(g.node_a + tail).out_head; e != W::kNone;) {
    const PoaEdge<Id> ea = Ld(g.edge + e);
    if (ea.head == head) {
      g.edge_w[e] += w;
      return;
    }
    last_out = e;
    e = ea.next_out;
  }
  if (g.n_edges >= g.ecap) {
    g.overflow = true;
    return;
  }
  const uint32_t e = g.n_edges++;
  St(g.edge + e, PoaEdge<Id>{static_cast<Id>(tail), static_cast<Id>(head), W::kNone, W::kNone});
  g.edge_w[e] = w;
  if (last_out == W::kNone) {
    g.node_a[tail].out_head = static_cast<Id>(e);
  } else {
    g.edge[last_out].next_out = static_cast<Id>(e);
  }
  const PoaNodeA<Id> h = Ld(g.node_a + head);
  if (h.in_head == W::kNone) {
    g.node_a[head].in_head = static_cast<Id>(e);
  } else {
    g.edge[h.in_tail].next_in = static_cast<Id>(e);
  }
  g.node_a[head].in_tail = static_cast<Id>(e);
}

// coverage = the sequences (of >= 2 bases) whose path visits the node
template <class W>
__device__ __forceinline__ void AddCov(PoaGraph<W>& g, uint32_t v) {
  g.node_b[v].cov += 1;
}

// append b to a's aligned nodes
template <class W>
__device__ void LinkAligned(PoaGraph<W>& g, uint32_t a, uint32_t b) {
  const uint32_t k = g.node_a[a].n_aligned++;
  g.node_b[a].aligned[k] = static_cast<typename W::Id>(b);
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
__device__ uint32_t AddChain(PoaGraph<W>& g, const SeqView& s, uint32_t begin, uint32_t end) {
  if (begin == end) return W::kNone;
  uint32_t first = W::kNone, prev = W::kNone;
  for (uint32_t i = begin; i < end && !g.overflow; ++i) {
    const uint32_t cur = AddNode(g, CodeOf(s.bases[i]));
    if (prev != W::kNone) AddEdge(g, prev, cur, s.weight(i - 1) + s.weight(i));
    if (first == W::kNone) first = cur;
    prev = cur;
  }
  return first;
}

// spoa Graph::TopologicalSort restricted to the nodes flagged kInSub, whose marks and
// ignored bits are clear (Graph::Subgraph keeps relative ids and adjacency order, so
// the restricted DFS over the full graph yields exactly the sub-graph's order)
template <class W>
__device__ uint32_t TopoSort(PoaGraph<W>& g) {
  using Id = typename W::Id;
  const uint32_t n = g.n_nodes;
  uint32_t rank = 0, sp = 0;
  for (uint32_t root = 0; root < n; ++root) {
    if (!(g.flags[root] & kInSub) || (g.flags[root] & kMarks)) continue;
    g.stack[sp++] = static_cast<Id>(root);
    while (sp > 0) {
      const uint32_t cur = g.stack[sp - 1];
      bool valid = true;
      if ((g.flags[cur] & kMarks) != 2) {
        const PoaNodeA<Id> a = Ld(g.node_a + cur);
        for (uint32_t e = a.in_head; e != W::kNone;) {
          const PoaEdge<Id> ea = Ld(g.edge + e);
          const uint32_t t = ea.tail;
          const uint8_t ft = g.flags[t];
          if ((ft & kInSub) && (ft & kMarks) != 2) {
            if (sp >= g.stack_cap) {
              g.overflow = true;
              return 0;
            }
            g.stack[sp++] = static_cast<Id>(t);
            valid = false;
          }
          e = ea.next_in;
        }
        const uint32_t na = a.n_aligned;
        PoaNodeB<Id> b{};
        if (na) b = Ld(g.node_b + cur);
        if (!(g.flags[cur] & kIgnored)) {
          for (uint32_t i = 0; i < na; ++i) {
            const uint32_t t = AlignedAt(b, i);
            const uint8_t ft = g.flags[t];
            if ((ft & kInSub) && (ft & kMarks) != 2) {
              if (sp >= g.stack_cap) {
                g.overflow = true;
                return 0;
              }
              g.stack[sp++] = static_cast<Id>(t);
              g.flags[t] = ft | kIgnored;
              valid = false;
            }
          }
        }
        if (valid) {
          g.flags[cur] = (g.flags[cur] & ~kMarks) | 2;
          if (!(g.flags[cur] & kIgnored)) {
            g.n2r[cur] = static_cast<Id>(rank);
            g.r2n[rank++] = static_cast<Id>(cur);
            for (uint32_t i = 0; i < na; ++i) {
              const uint32_t t = AlignedAt(b, i);
              if (g.flags[t] & kInSub) {
                g.n2r[t] = static_cast<Id>(rank);
                g.r2n[rank++] = static_cast<Id>(t);
              }
            }
          }
        } else {
          g.flags[cur] = (g.flags[cur] & ~kMarks) | 1;
        }
      }
      if (valid) --sp;
    }
  }
  return rank;
}

// spoa Graph::ExtractSubgraph(nodes[end], nodes[begin]): backward reachability from
// `from` through in-edges and aligned nodes, keeping ids >= min_id, into clear flags
template <class W>
__device__ void MarkSubgraph(PoaGraph<W>& g, uint32_t from, uint32_t min_id) {
  using Id = typename W::Id;
  uint32_t sp = 0;
  g.stack[sp++] = static_cast<Id>(from);
  while (sp > 0) {
    const uint32_t cur = g.stack[--sp];
    if ((g.flags[cur] & kInSub) || cur < min_id) continue;
    const PoaNodeA<Id> a = Ld(g.node_a + cur);
    for (uint32_t e = a.in_head; e != W::kNone;) {
      const PoaEdge<Id> ea = Ld(g.edge + e);
      if (sp >= g.stack_cap) {
        g.overflow = true;
        return;
      }
      g.stack[sp++] = ea.tail;
      e = ea.next_in;
    }
    const uint32_t na = a.n_aligned;
    if (na) {
      const PoaNodeB<Id> b = Ld(g.node_b + cur);
      for (uint32_t i = 0; i < na; ++i) {
        if (sp >= g.stack_cap) {
          g.overflow = true;
          return;
        }
        g.stack[sp++] = static_cast<Id>(AlignedAt(b, i));
      }
    }
    g.flags[cur] |= kInSub;
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
  uint32_t begin = AddChain(g, s, 0, first_pos);
  uint32_t prev = before == g.n_nodes ? W::kNone : g.n_nodes - 1;
  const uint32_t last = AddChain(g, s, last_pos + 1, s.len);
  // count this sequence on the chains
  const bool counts = s.len >= 2;
  if (counts) {
    for (uint32_t v = before; v < g.n_nodes; ++v) AddCov(g, v);
  }
  for (uint32_t i = 0; i < aln_len && !g.overflow; ++i) {
    const int32_t pos = g.aln_pos[i];
    if (pos == -1) continue;
    const uint32_t code = CodeOf(s.bases[pos]);
    uint32_t cur = W::kNone;
    if (g.aln_node[i] == -1) {
      cur = AddNode(g, code);
    } else {
      const uint32_t jt = static_cast<Id>(g.aln_node[i]);
      const PoaNodeA<Id> ja = Ld(g.node_a + jt);
      if (ja.code == code) {
        cur = jt;
      } else {
        const uint32_t na = ja.n_aligned;
        const PoaNodeB<Id> jb = Ld(g.node_b + jt);
        for (uint32_t a = 0; a < na; ++a) {
          const uint32_t kt = AlignedAt(jb, a);
          if (Ld(g.node_a + kt).code == code) {
            cur = kt;
            break;
          }
        }
        if (cur == W::kNone) {  // a new letter for this column
          cur = AddNode(g, code);
          if (g.overflow) break;
          for (uint32_t a = 0; a < na; ++a) {
            const uint32_t kt = AlignedAt(jb, a);
            LinkAligned(g, kt, cur);
            LinkAligned(g, cur, kt);
          }
          LinkAligned(g, jt, cur);
          LinkAligned(g, cur, jt);
        }
      }
    }
    if (g.overflow) break;
    if (counts) AddCov(g, cur);
    if (begin == W::kNone) begin = cur;
    if (prev != W::kNone) AddEdge(g, prev, cur, s.weight(pos - 1) + s.weight(pos));
    prev = cur;
  }
  if (last != W::kNone && !g.overflow) {
    AddEdge(g, prev, last, s.weight(last_pos) + s.weight(last_pos + 1));
  }
}

// (all lanes) racon's window prologue, over the window's `nseq` kept sequences. Returns
// true when it is done here: fewer than 3 give the backbone, "unpolished"; a letter
// other than ACGT fails it (racon feeds 2-bit reads).
__device__ __forceinline__ bool WindowDone(uint32_t nseq, uint32_t s0, uint32_t s1, uint32_t L0,
                                           const uint64_t* seq_off, const uint8_t* bases,
                                           uint8_t* out, uint32_t* cov_dst, uint32_t* cons_len,
                                           uint8_t* status, uint32_t lane) {
  if (nseq < 3) {
    for (uint32_t i = lane; i < L0; i += 32) {
      out[i] = bases[seq_off[s0] + i];
      if (cov_dst) cov_dst[i] = 0;
    }
    if (lane == 0) {
      *cons_len = L0;
      *status = 0;
    }
    return true;
  }
  bool bad_letter = false;
  for (uint64_t i = seq_off[s0] + lane; i < seq_off[s1]; i += 32) {
    if (CodeOf(bases[i]) < 0) bad_letter = true;
  }
  if (__any_sync(0xffffffffu, bad_letter)) {
    if (lane == 0) {
      *cons_len = 0;
      *status = kPoaStatusInvalid;
    }
    return true;
  }
  return false;
}

// (lane 0) the graph's arrays in the window's scratch slab (the kernel sets flags, r2n
// and n2r), the layers' order, and the backbone chain (spoa AddAlignment with an empty
// alignment: its edges weigh by its own qualities when the batch has qualities, and 0
// when it has none). Returns 0 or the status that ends the window.
template <class W>
__device__ uint32_t SetupGraph(PoaGraph<W>& g, uint8_t* base, const PoaLayout& L,
                               const typename W::Shape& shape, const uint64_t* seq_off,
                               const uint8_t* bases, const uint8_t* quals,
                               const uint32_t* seq_begin, const uint32_t* seq_end,
                               uint32_t s0, uint32_t s1, uint32_t L0) {
  using Id = typename W::Id;
  g.node_a = reinterpret_cast<PoaNodeA<Id>*>(base + L.node_a);
  g.node_b = reinterpret_cast<PoaNodeB<Id>*>(base + L.node_b);
  g.edge = reinterpret_cast<PoaEdge<Id>*>(base + L.edge);
  g.edge_w = reinterpret_cast<int32_t*>(base + L.edge_w);
  g.stack = reinterpret_cast<Id*>(base + L.stack);
  g.order = reinterpret_cast<Id*>(base + L.order);
  g.aln_node = reinterpret_cast<typename W::Pos*>(base + L.aln_node);
  g.aln_pos = reinterpret_cast<typename W::Pos*>(base + L.aln_pos);
  g.pred = reinterpret_cast<int32_t*>(base + L.pred);
  g.score = reinterpret_cast<long long*>(base + L.score);
  g.H = reinterpret_cast<typename W::Cell*>(base + L.H);
  g.DIR = base + L.DIR;
  g.n_nodes = g.n_edges = 0;
  g.ncap = shape.ncap;
  g.ecap = shape.ecap;
  g.stack_cap = 4 * shape.ncap;
  g.overflow = false;
  // layer coordinates are validated up front
  const uint32_t fail = OrderLayers(g.order, seq_off, seq_begin, seq_end, s0, s1, L0,
                                    shape.lmax, W::Layers(shape));
  if (!fail) {
    const SeqView bb{bases + seq_off[s0], quals ? quals + seq_off[s0] : nullptr, L0, 0};
    AddChain(g, bb, 0, L0);
    if (L0 >= 2) {
      for (uint32_t v = 0; v < g.n_nodes; ++v) AddCov(g, v);
    }
  }
  return fail;
}

// (all lanes) the graph a layer aligns to, in topological order: the whole graph, or
// the sub-graph between the layer's begin and end nodes; the cell guard; the sinks
// (no out-edge inside the (sub)graph). Returns the rows; on overflow the window stops.
template <class W>
__device__ __forceinline__ uint32_t LayerGraph(PoaGraph<W>& g, bool full, uint32_t lb,
                                               uint32_t le, uint32_t len, int m, int n,
                                               int gap, uint32_t lane) {
  const uint32_t nn = g.n_nodes;
  for (uint32_t v = lane; v < nn; v += 32) g.flags[v] = full ? kInSub : 0;
  __syncwarp();
  if (lane == 0) {
    if (!full) MarkSubgraph(g, le, lb);
    const uint32_t rows = g.overflow ? 0 : TopoSort(g);
    // the cells' range: |score| <= max|m,n,g| * (rows + columns)
    const int amax = max(max(abs(m), abs(n)), abs(gap));
    if (static_cast<long long>(amax) * (rows + len + 2) > W::kCellLimit) g.overflow = true;
    g.rows = rows;
  }
  __syncwarp();
  const uint32_t rows = g.rows;
  if (g.overflow) return rows;
  for (uint32_t r = lane; r < rows; r += 32) {
    const uint32_t v = g.r2n[r];
    bool sink = true;
    for (uint32_t e = Ld(g.node_a + v).out_head; e != W::kNone;) {
      const PoaEdge<typename W::Id> ea = Ld(g.edge + e);
      if (g.flags[ea.head] & kInSub) {
        sink = false;
        break;
      }
      e = ea.next_out;
    }
    if (sink) g.flags[v] |= kSink;
  }
  __syncwarp();
  return rows;
}

// (lane 0) the traceback of `alen` steps, written from its end, into emission order,
// and the layer into the graph
template <class W>
__device__ void MergeLayer(PoaGraph<W>& g, const SeqView& sv, uint32_t alen) {
  for (uint32_t a = 0; a < alen / 2; ++a) {
    const typename W::Pos tn = g.aln_node[a], tp = g.aln_pos[a];
    g.aln_node[a] = g.aln_node[alen - 1 - a];
    g.aln_pos[a] = g.aln_pos[alen - 1 - a];
    g.aln_node[alen - 1 - a] = tn;
    g.aln_pos[alen - 1 - a] = tp;
  }
  if (g.overflow) return;
  if (alen == 0) {
    // spoa: an empty alignment appends the sequence as a separate chain
    const uint32_t before = g.n_nodes;
    AddChain(g, sv, 0, sv.len);
    if (sv.len >= 2) {
      for (uint32_t v = before; v < g.n_nodes; ++v) AddCov(g, v);
    }
  } else {
    AddAlignment(g, sv, alen);
  }
}

// (all lanes) the window's result: spoa's heaviest bundle with branch completion,
// racon's coverage-based TGS trimming, the consensus and its coverage, the status, and
// the window's DP cells
template <class W>
__device__ __forceinline__ void Consensus(PoaGraph<W>& g, uint32_t fail, uint32_t nseq,
                                          int trim, int tgs, unsigned long long my_cells,
                                          uint8_t* out, uint32_t* cov_dst, uint32_t* cons_len,
                                          uint8_t* status, unsigned long long* cells,
                                          uint32_t lane) {
  using Id = typename W::Id;
  const uint32_t nn = g.n_nodes;
  for (uint32_t v = lane; v < nn; v += 32) g.flags[v] = kInSub;
  __syncwarp();
  if (lane != 0) return;
  uint32_t st = 0, clen = 0;
  if (fail) {
    st = fail;
  } else if (g.overflow) {
    st = kPoaStatusCapacity;
  } else {
    const uint32_t rows = TopoSort(g);
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
        for (uint32_t e = Ld(g.node_a + v).in_head; e != W::kNone;) {
          const PoaEdge<Id> ea = Ld(g.edge + e);
          const uint32_t t = ea.tail;
          const long long wgt = g.edge_w[e];
          if (g.score[v] < wgt || (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
            g.score[v] = wgt;
            g.pred[v] = static_cast<int32_t>(t);
          }
          e = ea.next_in;
        }
        if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
        if (mx < 0 || g.score[mx] < g.score[v]) mx = static_cast<int32_t>(v);
      }
      while (Ld(g.node_a + mx).out_head != W::kNone) {  // branch completion
        const uint32_t rank = g.n2r[mx];
        for (uint32_t e = Ld(g.node_a + mx).out_head; e != W::kNone;) {
          const PoaEdge<Id> ea = Ld(g.edge + e);
          for (uint32_t f = Ld(g.node_a + ea.head).in_head; f != W::kNone;) {
            const PoaEdge<Id> fa = Ld(g.edge + f);
            if (fa.tail != static_cast<uint32_t>(mx)) g.score[fa.tail] = -1;
            f = fa.next_in;
          }
          e = ea.next_out;
        }
        int32_t nmx = -1;
        for (uint32_t r = rank + 1; r < rows; ++r) {
          const uint32_t v = g.r2n[r];
          g.score[v] = -1;
          g.pred[v] = -1;
          for (uint32_t e = Ld(g.node_a + v).in_head; e != W::kNone;) {
            const PoaEdge<Id> ea = Ld(g.edge + e);
            const uint32_t t = ea.tail;
            const long long wgt = g.edge_w[e];
            e = ea.next_in;
            if (g.score[t] == -1) continue;
            if (g.score[v] < wgt || (g.score[v] == wgt && g.score[g.pred[v]] <= g.score[t])) {
              g.score[v] = wgt;
              g.pred[v] = static_cast<int32_t>(t);
            }
          }
          if (g.pred[v] != -1) g.score[v] += g.score[g.pred[v]];
          if (nmx < 0 || g.score[nmx] < g.score[v]) nmx = static_cast<int32_t>(v);
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
        const uint32_t nd = g.r2n[plen - 1 - idx];
        uint32_t cvg = g.node_b[nd].cov;
        const uint32_t na = Ld(g.node_a + nd).n_aligned;
        if (na) {
          const PoaNodeB<Id> b = Ld(g.node_b + nd);
          for (uint32_t a = 0; a < na; ++a) cvg += g.node_b[AlignedAt(b, a)].cov;
        }
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
        const uint32_t nd = g.r2n[plen - 1 - (cb + i)];
        out[i] = "ACGT"[Ld(g.node_a + nd).code];
        if (cov_dst) cov_dst[i] = coverage(cb + i);
      }
    }
  }
  *cons_len = clen;
  *status = static_cast<uint8_t>(st);
  // DP cells of this window (lanes hold the same count); an attempt that ran out
  // of capacity is run again and counted then
  if (cells && st != kPoaStatusCapacity) atomicAdd(cells, my_cells);
}

// The generic DP: all lanes fill a row 32 columns at a time, the diagonal neighbour
// from the row above, the horizontal gap recurrence H[i][j] = max(M[j], H[i][j-1] + g)
// as a warp max-scan of M[j] - j*g (exact in integers); lane 0's traceback re-derives
// each step from H with spoa's preference.
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
  const uint32_t L0 = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
  uint8_t* out = cons + cons_off[w];
  uint32_t* cov_dst = cov_out ? cov_out + cons_off[w] : nullptr;
  const uint32_t nseq = KeptSequences(seq_off, seq_begin, seq_end, s0, s1, lane);
  if (WindowDone(nseq, s0, s1, L0, seq_off, bases, out, cov_dst, cons_len + w, status + w, lane)) {
    return;
  }

  uint8_t* base = scratch + scratch_stride * blockIdx.x;
  const PoaLayout L = MakePoaLayout<W>(shape, false);
  __shared__ PoaGraph<W> g;
  __shared__ uint32_t sh_fail;
  if (lane == 0) {
    g.flags = base + L.flags;
    g.r2n = reinterpret_cast<Id*>(base + L.r2n);
    g.n2r = reinterpret_cast<Id*>(base + L.n2r);
    sh_fail = SetupGraph(g, base, L, shape, seq_off, bases, quals, seq_begin, seq_end, s0, s1,
                         L0);
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
    const uint32_t lb = seq_begin[s], le = seq_end[s];
    const uint32_t rows = LayerGraph(g, lb < offset && le > L0 - offset, lb, le, len, m, n, gap, lane);
    if (g.overflow) break;
    my_cells += static_cast<unsigned long long>(rows + 1) * (len + 1);

    // ---- DP (all lanes) ----
    Cell* H = g.H;
    for (uint32_t j = lane; j <= len; j += 32) H[j] = static_cast<Cell>(j * gap);
    __syncwarp();
    int best_score = -2147483647, best_row = -1;
    for (uint32_t r = 0; r < rows; ++r) {
      const uint32_t v = g.r2n[r];
      const PoaNodeA<Id> va = Ld(g.node_a + v);
      Cell* row = H + static_cast<size_t>(r + 1) * width;
      // column 0
      int col0 = 0;
      {
        bool any = false;
        int pen = -2147483647;
        for (uint32_t e = va.in_head; e != W::kNone;) {
          const PoaEdge<Id> ea = Ld(g.edge + e);
          e = ea.next_in;
          if (!(g.flags[ea.tail] & kInSub)) continue;
          any = true;
          pen = max(pen, static_cast<int>(H[static_cast<size_t>(g.n2r[ea.tail] + 1) * width]));
        }
        col0 = (any ? pen : 0) + gap;
      }
      int carry = col0;  // running max of M[k] - k*g over k < chunk start (k = 0 term)
      for (uint32_t c0 = 1; c0 <= len; c0 += 32) {
        const uint32_t j = c0 + lane;
        int M = W::kNoCell;
        if (j <= len) {
          const int match = (static_cast<uint32_t>(CodeOf(sv.bases[j - 1])) == va.code) ? m : n;
          bool any = false;
          for (uint32_t e = va.in_head; e != W::kNone;) {
            const PoaEdge<Id> ea = Ld(g.edge + e);
            e = ea.next_in;
            if (!(g.flags[ea.tail] & kInSub)) continue;
            any = true;
            const Cell* pr = H + static_cast<size_t>(g.n2r[ea.tail] + 1) * width;
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
      if (g.flags[v] & kSink) {
        const int sc = row[len];
        if (best_score < sc) {
          best_score = sc;
          best_row = static_cast<int>(r + 1);
        }
      }
    }

    // ---- (lane 0) traceback: diagonal over predecessors in in-edge order, then
    // vertical, then horizontal ----
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
          const PoaNodeA<Id> va = Ld(g.node_a + g.r2n[i - 1]);
          const int match = (static_cast<uint32_t>(CodeOf(sv.bases[j - 1])) == va.code) ? m : n;
          bool any = false;
          for (uint32_t e = va.in_head; e != W::kNone && !found;) {
            const PoaEdge<Id> ea = Ld(g.edge + e);
            e = ea.next_in;
            if (!(g.flags[ea.tail] & kInSub)) continue;
            any = true;
            const uint32_t p = g.n2r[ea.tail] + 1;
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
          bool any = false;
          for (uint32_t e = Ld(g.node_a + g.r2n[i - 1]).in_head; e != W::kNone && !found;) {
            const PoaEdge<Id> ea = Ld(g.edge + e);
            e = ea.next_in;
            if (!(g.flags[ea.tail] & kInSub)) continue;
            any = true;
            const uint32_t p = g.n2r[ea.tail] + 1;
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
      MergeLayer(g, sv, alen);
    }
    __syncwarp();
  }
  Consensus(g, sh_fail, nseq, trim, tgs, my_cells, out, cov_dst, cons_len + w, status + w,
            cells, lane);
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
    return (MakePoaLayout<PoaWide>(s, false).bytes + 255) & ~size_t(255);
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
      const size_t stride = (MakePoaLayout<PoaNarrow>(shape, fast).bytes + 255) & ~size_t(255);
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
