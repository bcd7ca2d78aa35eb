// raven_b200 — overlap engine context and stage entry points (host side).
//
// Data layout in HBM (all SoA, 8-byte fields, see DESIGN.md):
//   reads      words[]           2-bit packed, biosoup layout, 0.25 B/base
//   sketch     sk.val, sk.org    minimizer records in (read, position) order
//   queries    mm.val, mm.org    micromizers (len/k smallest per read)
//   index      i_val[], i_org[]  sketch stably sorted by value + bucket table
//   hits       h_grp[], h_pos[]  ram "Match" records grouped by query read
//   overlaps   rvn_overlap[]     32 B records grouped by query read
#pragma once

#include <functional>
#include <string>
#include <vector>

#include "../../include/raven_b200.h"
#include "common.cuh"

namespace rvn {

struct Params {
  uint32_t k = 15, w = 5, bandwidth = 500, chain = 4, matches = 100;
  uint32_t gap = 10000;
};

// k-mer positions handled by one CTA of the sketch kernels
constexpr uint32_t kSketchTile = 2048;
constexpr uint32_t kSketchThreads = 256;
constexpr uint32_t kMaxWindow = 256;  // w limit (halo staged in shared memory)

// The reads one stage-1 flush touches, as dense slots: the index batch [b0, b1)
// first, then the flush's queries [a0, a1) that lie before it (a1 <= b0, possibly
// empty). Piles, list counts and offsets of a flush are indexed by slot. The
// resident layout is the window of all n reads, where slot == id.
struct Window {
  uint32_t b0 = 0, b1 = 0, a0 = 0, a1 = 0;
  static Window All(uint32_t n) { return Window{0, n, 0, 0}; }
  __host__ __device__ __forceinline__ uint32_t size() const { return (b1 - b0) + (a1 - a0); }
  __host__ __device__ __forceinline__ uint32_t Slot(uint32_t id) const {
    return id >= b0 ? id - b0 : (b1 - b0) + (id - a0);
  }
  __host__ __device__ __forceinline__ uint32_t Id(uint32_t s) const {
    return s < b1 - b0 ? b0 + s : a0 + (s - (b1 - b0));
  }
};

// one substring pair of the edit-distance tiers (editdist.cu)
struct PairDesc {
  uint64_t q_word;   // first word of the lhs read in `words`
  uint64_t t_word;   // first word of the rhs read
  uint32_t q_begin, q_len;
  uint32_t t_begin, t_len;
  uint32_t strand;   // 1 = same strand; 0 = rhs substring reverse complemented
  uint32_t slot;     // index of the pair in the caller's arrays
};

struct PhaseTimer {
  std::vector<const char*> names;
  std::vector<float> ms;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
  std::vector<cudaEvent_t> pool;
};

// The words of a read range copied to the device on the context's copy stream in pieces cut
// at read boundaries (bases.cu): reads [.., read_end[i]) have arrived once events[i] has
// completed. n: the pieces of the last copy (the events are reused).
struct CopyPieces {
  std::vector<cudaEvent_t> events;
  std::vector<uint32_t> read_end;
  uint32_t n = 0;
};

// One half of the staging window of packed bases (host_bases mode): the words of the read
// range [first, last), word w of the set at words[w - woff[first]], arriving in `copy`.
// `used` is recorded on the context's stream behind the last kernel that read the half; a
// new copy into it waits for that.
struct BaseHalf {
  DevBuf<uint64_t> words;
  uint32_t first = 0, last = 0;
  bool valid = false;
  CopyPieces copy;
  cudaEvent_t used = nullptr;
  bool used_recorded = false;
};

// Where the sketch kernels of a read range find their bases: word w of the set at
// words[w - base]. pieces > 0: copies still in flight, reads [.., read_end[i]) complete once
// events[i] has (the async_upload chunks, or a staged range's pieces). half: the staging
// window's half that holds them, -1 = the device copy of the set (d_words).
struct BaseView {
  const uint64_t* words = nullptr;
  uint64_t base = 0;
  const cudaEvent_t* events = nullptr;
  const uint32_t* read_end = nullptr;
  uint32_t pieces = 0;
  int half = -1;
};

// Where the packed bases of the uploaded reads are (bases.cu)
struct Bases {
  // option "host_bases": where rvn_reads_upload / rvn_reads_upload_ids keep the bases: 0 in
  // d_words, 1 in the pinned host copy h_words (the sketch kernels read them from the staging
  // window half[]), -1 (default) on the host only when a stage-1 pass at the reference's
  // batch sizes would fit the device with them there and not without ("host_bases_budget"
  // replaces the usable device memory when it is not 0)
  int64_t host_bases = -1;
  uint64_t host_bases_budget = 0;
  bool on_host = false;  // the current upload's bases are in h_words only
  PinBuf<uint64_t> h_words;
  BaseHalf half[2];
  int cur = 0;  // the half of the range a sketch asked for last
  // reads whose bases the next sketch launch should be followed by a copy of (the range the
  // driver sketches after it; empty: none)
  uint32_t next_first = 0, next_last = 0;
  uint32_t res_first = 0, res_last = 0;  // reads whose bases are in d_words
  // option "async_upload": the bases travel to d_words on the copy stream in pieces, behind
  // up_fence (recorded on the context's stream: kernels of earlier calls may still read the
  // old bases). The next sketch launch starts on the pieces that have arrived, any other call
  // waits for all of them (WaitUpload); upload.n = 0: none in flight.
  int64_t async_upload = 0;
  cudaStream_t copy_stream = nullptr;  // (the staging window's copies too)
  cudaEvent_t up_fence = nullptr;
  CopyPieces upload;
};

// The records of reads [first, last) in (read, position) order: the sketch or the
// micromizers. Read first + i has records [h_off[i], h_off[i + 1]) of val / org, n in all
// (off: the same offsets on the device, bound at construction); the values are u32 when
// is32 (2k <= 30), else u64.
struct RecordSet {
  RecordSet(DevBuf<uint64_t>& o, std::vector<uint64_t>& h) : off(o), h_off(h) {}
  bool valid = false;
  uint32_t first = 0, last = 0;
  uint64_t n = 0;
  bool is32 = false;
  DevBuf<uint64_t> val, org;
  DevBuf<uint64_t>& off;
  std::vector<uint64_t>& h_off;
  bool Exactly(uint32_t f, uint32_t l) const { return valid && first == f && last == l; }
  bool Covers(uint32_t f, uint32_t l) const { return valid && first <= f && l <= last; }
  ValView Values() const { return ValView{val.get(), is32 ? 1 : 0}; }
  void Hold(uint32_t f, uint32_t l, uint64_t records, bool v32) {  // (once val / org are written)
    first = f;
    last = l;
    n = records;
    is32 = v32;
    valid = true;
  }
};

// Micromizer thresholds of reads [first, last): record (value, position) of read r is a
// micromizer iff value < val[r - first] || (value == val[r - first] && position <
// pos[r - first]). Read first + i has h_off[i + 1] - h_off[i] micromizers (off: the same
// counts on the device, where Micromize selects by them).
struct Thresholds {
  bool valid = false;
  uint32_t first = 0, last = 0;
  DevBuf<uint64_t> val;
  DevBuf<uint32_t> pos;
  DevBuf<uint64_t> off;
  std::vector<uint64_t> h_off;
  bool Exactly(uint32_t f, uint32_t l) const { return valid && first == f && last == l; }
  bool Covers(uint32_t f, uint32_t l) const { return valid && first <= f && l <= last; }
  // an empty table of reads [f, f) with room for the values of `reads` reads
  void Reset(uint32_t f, uint32_t reads) {
    first = last = f;
    val.reserve(reads + 1ULL);
    pos.reserve(reads + 1ULL);
    h_off.assign(1, 0);
  }
  // the table of the reads that follow (t.first == last) behind this one (no device counts)
  void Append(const Thresholds& t, cudaStream_t stream) {
    const uint32_t nr = t.last - t.first;
    RVN_CUDA(cudaMemcpyAsync(val.get() + (t.first - first), t.val.get(), nr * sizeof(uint64_t),
                             cudaMemcpyDeviceToDevice, stream));
    RVN_CUDA(cudaMemcpyAsync(pos.get() + (t.first - first), t.pos.get(), nr * sizeof(uint32_t),
                             cudaMemcpyDeviceToDevice, stream));
    const uint64_t base = h_off.back();
    for (uint32_t r = 1; r <= nr; ++r) h_off.push_back(base + t.h_off[r]);
    last = t.last;
  }
};

struct Ctx {
  // device bytes held by this context's buffers (first member: it outlives them)
  uint64_t held_bytes = 0;
  int device = 0;
  int sms = 132;  // multiprocessors of `device` (grid caps of the grid-stride kernels)
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  bool p_off_uploaded = false;  // stage-1 pile offsets already on the device
  std::string err;
  Params prm;
  bool keep_hits = false;
  rvn_stats stats{};

  // ---- reads ----
  uint32_t n_reads = 0;
  uint64_t n_words = 0;
  DevBuf<uint64_t> d_words, d_woff;
  DevBuf<uint32_t> d_len, d_ids;
  std::vector<uint64_t> h_woff;
  std::vector<uint32_t> h_len, h_ids;
  // first pile bin of every read (len >> 4 bins), n_reads + 1 entries (before the first
  // upload too: a context starts as an empty read set)
  std::vector<uint64_t> h_pile_off{0};
  bool ids_identity = true;  // id == index (needed by the device-side gather)
  Bases bases;
  // ---- rvn_reads_upload_files (fastx.cu) ----
  // option "fastx_chunk_bytes": text bytes parsed per chunk (0: 256 MiB)
  uint64_t fastx_chunk_bytes = 0;
  bool reads_unset = false;  // a failed rvn_reads_upload_files left no read set
  // the current set was made by rvn_reads_upload_files: its block qualities (bq_off as
  // rvn_polish_windows takes it) and names (name i = fx_names[fx_name_off[i], [i + 1]))
  bool fx_valid = false;
  std::vector<uint8_t> fx_bq;
  std::vector<uint64_t> fx_bq_off, fx_name_off;
  std::string fx_names;
  // sketch tiles: tile_off[r] = first tile of read r (depends on k)
  std::vector<uint64_t> h_tile_off;
  DevBuf<uint64_t> d_tile_off;
  DevBuf<uint32_t> d_tile_read;  // read of every tile
  uint32_t tiles_k = 0;

  // ---- current sketch: the full minimizers of reads [sk.first, sk.last) ----
  DevBuf<uint64_t> sk_off;
  std::vector<uint64_t> h_sk_off;
  RecordSet sk{sk_off, h_sk_off};
  DevBuf<uint32_t> tile_cnt;
  DevBuf<uint64_t> tile_out, tile_status;

  // ---- current micromizer thresholds and micromizer set ----
  Thresholds qt;
  // One buffer pair: the micromizers' offsets are the counts of the thresholds. A Micromize
  // of thresholds only rewrites them, and the set stays valid only for the same reads.
  RecordSet mm{qt.off, qt.h_off};
  int t_b_low = 0;  // the bare keys of the upper tier are sorted above this many low bits
  uint64_t group_count_min = 0;  // fewer keys per group of equal upper bits: full sort instead
  bool i_from_sketch = false;  // the index holds the FULL sketches of reads [i_first, i_last)
  int64_t self_join = 1;       // option: stage-1 hits by a self-join over the index
  // option: multiplicities of the bare keys by one partition pass + cluster counters
  // (1: clusters of 8 CTAs, 8 or 16: that cluster size) instead of a sort (0)
  int64_t bare_count = 1;

  // ---- index ----
  bool i_valid = false;
  uint32_t i_first = 0, i_last = 0;
  uint64_t i_n = 0, i_keys = 0;
  DevBuf<uint64_t> i_val, i_org, i_val_alt, i_org_alt;
  bool i_is32 = false;  // i_val holds u32 values
  int i_shift = 0;             // bucket = value >> i_shift
  uint64_t i_limit = ~0ULL;    // tiered build: only values <= i_limit are in the index
  // tiers (index.cu): staging of the probe-able tier and the bare keys beyond it
  DevBuf<uint32_t> t_cnt;
  DevBuf<uint64_t> t_off, t_aval, t_aorg, t_b0, t_b1, t_b2, t_narrow;
  const uint32_t* t_sorted_b = nullptr;
  uint64_t t_nb = 0;
  bool t_b_sorted = true;       // t_sorted_b is in full key order (else: partitioned or unsorted)
  DevBuf<uint32_t> t_bstart;    // first bare key of every bucket of the partition
  int bare_cluster = 0;         // cluster size of BareCountKernel on this device (0: not chosen)
  int bare_clusters = 0;        // clusters of that size resident at once
  uint64_t tier_min_records = 1ULL << 18;  // smaller index batches are not worth a partition
  DevBuf<uint64_t> t_hist;  // chunked build: coarse value histogram (capacity of the tiers)
  // Chunked build (BuildIndexChunked): the micromizer thresholds and counts of the index
  // batch [i_first, i_last), kept apart from c.qt, which the probe-path flushes of reads
  // before the batch overwrite; valid while jt_gen == i_gen
  uint64_t jt_gen = 0;
  Thresholds jt;
  DevBuf<uint32_t> i_bucket;
  int i_bucket_bits = 0;
  DevBuf<uint64_t> i_gaps;  // long empty stretches of the bucket table (index.cu)
  DevBuf<uint64_t> i_hist;  // run-length histogram of the keys + #keys (index.cu)
  uint32_t occurrence = 0xFFFFFFFFu;
  bool i_sorted_ids = false;  // postings of a key are in ascending read-id order
  bool ids_ascending = true;  // read ids never decrease with the read index
  DevBuf<uint8_t> sort_tmp;
  // option "radix_portion_tiles": a radix sort or partition runs in portions of at
  // most that many tiles (0: the longest portion its status words allow)
  int64_t radix_portion_tiles = 0;

  // ---- map ----
  DevBuf<uint32_t> m_cnt, m_first;
  DevBuf<uint8_t> m_filt;
  DevBuf<uint64_t> m_hit_off;  // per query record (+1)
  DevBuf<uint64_t> m_sq_key, m_sq_key2;  // queries sorted by value (probe order)
  DevBuf<uint32_t> m_sq_idx, m_sq_idx2;
  DevBuf<uint64_t> h_grp, h_pos;
  DevBuf<uint64_t> m_read_hit_off;  // per query read (+1)
  // stage-1 self-join (map.cu): per micromizer slot of reads [j_first, i_last), its
  // query posting << 32 | hit count; valid for index build j_gen filtered at
  // j_occurrence
  uint64_t i_gen = 0, j_gen = 0;
  uint32_t j_occurrence = 0, j_first = 0;
  std::vector<uint64_t> h_j_off;
  DevBuf<uint64_t> j_off, j_packed;
  DevBuf<uint32_t> j_cursor;
  DevBuf<uint64_t> m_scratch64;     // oversize chain scratch
  DevBuf<uint32_t> m_scratch32, m_fallback;
  // split chain path: pair descriptors, pair-contiguous hits, overlap keys
  DevBuf<uint32_t> m_desc, m_desc_cnt, m_desc_idx, m_desc_cnt2, m_desc_idx2, m_gdiag,
      m_oidx, m_oidx2;
  DevBuf<uint64_t> m_gpos, m_group_loc, m_okey, m_okey2, m_starts;
  DevBuf<uint32_t> m_bounds;
  DevBuf<rvn_overlap> m_ovl_raw, m_ovl, m_ovl_tmp;
  DevBuf<uint64_t> m_ovl_loc;  // per read: base<<24 | count  (raw placement)
  DevBuf<uint64_t> m_ovl_off;
  DevBuf<uint64_t> m_counter;
  DevBuf<uint32_t> m_filtered;
  DevBuf<uint64_t> m_filtered_off;  // per query read (+1): its slice of m_filtered
  uint64_t m_n_filtered = 0;
  bool m_filtered_host = true;  // FilteredPositions also copies them to r_filtered
  DevBuf<uint64_t> m_filt_off;
  DevBuf<uint64_t> scan_tmp;
  uint64_t m_hits = 0;
  uint32_t m_first_read = 0, m_last_read = 0;

  // host-side results of the last map
  PinBuf<rvn_overlap> r_ovl;
  PinBuf<uint64_t> r_ovl_off;
  PinBuf<uint32_t> r_filtered;
  PinBuf<uint64_t> r_filt_off;
  uint64_t r_n_ovl = 0;
  bool r_valid = false;
  PinBuf<uint64_t> r_hit_grp, r_hit_pos, r_hit_off;
  // rvn_map in several flushes: the results gathered so far (they become r_* at the end)
  PinBuf<rvn_overlap> a_ovl;
  PinBuf<uint64_t> a_ovl_off, a_filt_off;
  PinBuf<uint32_t> a_filtered;
  uint64_t r_n_hits = 0;

  // introspection staging
  PinBuf<uint64_t> x_val, x_org, x_off;

  // ---- piles ----
  DevBuf<int32_t> p_diff;
  DevBuf<uint16_t> p_data;
  DevBuf<uint64_t> p_off;
  DevBuf<rvn_overlap> p_ovl;

  // ---- per-read overlap lists (gather.cu) ----
  int g_cur = 0;
  uint64_t g_total = 0;
  DevBuf<rvn_overlap> g_list[2], g_stage;
  DevBuf<uint64_t> g_off, g_off_alt, g_rhs_off, g_t_off, g_pairs;
  DevBuf<uint32_t> g_cnt, g_kept, g_key, g_idx, g_key2, g_idx2, g_rhs_cnt,
      g_total_cnt;

  // ---- windowed stage 1 (stage.cu): piles and lists of all reads on the host,
  // a flush's window of them on the device ----
  // option "stage1_window": 0 resident, 1 windowed, -1 (default) windowed only when
  // the resident estimate exceeds the free device memory ("stage1_window_budget"
  // replaces that free memory when it is not 0)
  int64_t stage1_window = -1;
  uint64_t stage1_window_budget = 0;
  bool st_windowed = false;  // the last stage-1 call ran windowed
  // option "index_chunk_bases": -1 (default) chunks of 2^30 bases only when the one-shot
  // pass does not fit the device ("index_chunk_budget" replaces the free memory when it
  // is not 0), 0 one-shot index build, N > 0 always chunks of >= N bases
  int64_t index_chunk_bases = -1;
  uint64_t index_chunk_budget = 0;
  // rvn_minimize built the index in chunks and rvn_filter has not yet freed what only the
  // build used (ReleaseIndexBuild)
  bool i_build_held = false;
  // option "map_flush_bases": rvn_map works its query range in flushes of >= N bases;
  // 0 (default) = from the usable device memory, at most the reference's 2^30
  uint64_t map_flush_bases = 0;
  // option "stage2_batch_bases": rvn_find_overlaps_and_repetitive_regions cuts its index
  // batches at >= N bases; 0 (default) = the reference's 2^30
  uint64_t stage2_batch_bases = 0;
  PinBuf<rvn_overlap> w_rows;  // kmax records per read
  PinBuf<uint32_t> w_cnt;      // kept records per read
  DevBuf<uint64_t> w_pile_off, w_row_off;  // per slot (+1) of the current window

  // ---- POA (poa.cu) ----
  DevBuf<uint32_t> po_win_first, po_seq_begin, po_seq_end, po_cons_len, po_cov, po_list;
  DevBuf<uint64_t> po_seq_off, po_d_cons_off;
  DevBuf<uint8_t> po_bases, po_quals, po_cons, po_status, po_scratch;
  std::vector<uint64_t> po_cons_off, po_out_off;
  std::vector<uint8_t> po_h_status, po_h_cons, po_out_cons;
  std::vector<uint32_t> po_h_clen, po_h_cov, po_out_cov;
  uint64_t po_cells = 0;
  uint32_t po_n_windows = 0;
  bool po_has_cov = false, poa_valid = false;
  // option "poa_wide": 0 (default) windows past the 16-bit kernels' limits fail the call;
  // 1 they run on the 32-bit kernel; 2 every window does. "poa_scratch_budget" (bytes)
  // replaces the scratch budget of a launch when it is not 0
  int64_t poa_wide = 0;
  uint64_t poa_scratch_budget = 0;
  // windows and launches of the last rvn_poa_batch per kernel: fast, generic, wide
  uint32_t po_route_windows[3] = {0, 0, 0}, po_route_launches[3] = {0, 0, 0};
  // rvn_polish_windows (layers.cu): per alignment and per breaking-point slot, the
  // window key and slot order of the stable sort, per window its kept layers and their
  // bases, per window of a batch its source; option "poa_batch_bytes" (0 = from the
  // free device memory) bounds the flat inputs of one window batch
  DevBuf<uint8_t> pl_aln, pl_bq, pl_win;
  DevBuf<uint32_t> pl_bp, pl_key[2], pl_cnt, pl_seq_len;
  DevBuf<uint64_t> pl_ord[2], pl_bases, pl_err;
  uint64_t poa_batch_bytes = 0;
  uint32_t po_batches = 0;  // window batches of the last rvn_polish_windows

  // ---- stage-1 results ----
  PinBuf<rvn_overlap> st_ovl;  // pinned: the D2H of the results runs at link speed
  PinBuf<uint64_t> st_ovl_off;
  PinBuf<uint16_t> st_pile;
  uint64_t st_mapped = 0;
  bool st_valid = false;
  bool st_piles_on_device = false;  // c.p_data / c.p_off still hold the piles of that call
  // option "stage1_stream": a resident pass copies the piles and lists of the reads no
  // later flush touches to the host while the later flushes run (1, default), or all
  // of them after the last flush (0). d2h_stream carries those copies; d2h_ready is
  // recorded on `stream` when a source is final, d2h_done after the copies
  int64_t stage1_stream = 1;
  cudaStream_t d2h_stream = nullptr;
  cudaEvent_t d2h_ready = nullptr, d2h_done = nullptr;

  // ---- stage 2 (stage.cu Stage2): per valid read its pile region, the k-mer marks (one
  // bit per pile bin and one past the end, bins + 1 bits in whole u32 words) and the
  // touched flag, resident for the whole call; the kept overlaps of every batch ----
  DevBuf<uint32_t> s2_pos_of, s2_rbeg, s2_rend, s2_bits;
  DevBuf<uint64_t> s2_bit_off;
  DevBuf<uint8_t> s2_touched;
  DevBuf<rvn_overlap> s2_kept;
  DevBuf<uint64_t> s2_kept_off;
  PinBuf<rvn_overlap> s2_ovl;
  PinBuf<uint64_t> s2_ovl_off, s2_bit_off_h;
  PinBuf<uint32_t> s2_bits_h;
  PinBuf<uint8_t> s2_touched_h;
  // edit-distance tiers and the clip/filter of one flush (editdist.cu)
  DevBuf<PairDesc> e_pairs;
  DevBuf<uint32_t> e_list, e_list2, e_key, e_key2, e_flag, e_sflag;
  DevBuf<int32_t> e_limit, e_dist;
  DevBuf<uint64_t> e_scan, e_sscan;
  DevBuf<rvn_overlap> e_ovl;
  uint32_t s2_n_valid = 0;
  uint64_t s2_mapped = 0;
  bool s2_valid = false;

  // ---- read ownership of the stage-1 tail: read r is owned iff r % own_mod ==
  // own_rem (1 / 0 = every read: the single-GPU path) ----
  uint32_t own_mod = 1, own_rem = 0;

  // ---- multi-GPU partition / exchange staging (dist.cu) ----
  DevBuf<uint64_t> ds_split_val, ds_split_org, ds_qsplit_val, ds_qsplit_org;
  DevBuf<uint64_t> ds_grouped_grp, ds_grouped_pos, ds_rel_off, ds_seg_start, ds_seg_base,
      ds_bounds, ds_q_off;
  DevBuf<uint32_t> ds_masked, ds_hit_lhs, ds_read_cnt, ds_flag, ds_own_ids;
  DevBuf<rvn_overlap> ds_ovl_split, ds_merged;
  // results of the owned reads (pinned host)
  PinBuf<rvn_overlap> ds_r_ovl;
  PinBuf<uint64_t> ds_r_ovl_off, ds_r_pile_off;
  PinBuf<uint16_t> ds_r_pile;
  uint32_t ds_n_own = 0;
  bool ds_results_valid = false;
  // peer-memory exchange: own receive arena + the peers' arenas (CUDA IPC)
  void* x_arena = nullptr;
  uint64_t x_cap = 0;
  uint32_t x_rank = 0;
  std::vector<void*> x_peers;
  std::vector<cudaStream_t> x_streams;

  // pinned scalars for small D2H reads
  PinBuf<uint64_t> pin64;

  PhaseTimer timer;
  uint64_t launches = 0;
};

// The cached sets a change makes stale (each level also clears those of the levels before it)
enum class Stale { kRecords, kThresholds, kIndex, kStage1 };
inline void MarkStale(Ctx& c, Stale s) {
  c.sk.valid = c.mm.valid = false;  // kRecords: a new sketch, or the tile table changed
  if (s >= Stale::kThresholds) c.qt.valid = false;  // a rider read joined or left the set
  if (s >= Stale::kIndex) c.i_valid = c.r_valid = false;  // new parameters, a stage-1 pass
  if (s >= Stale::kStage1) c.st_valid = false;  // a new read set
}

// ---- utilities (scan.cu) ----
// out[i] = sum_{j<i} in[j] for i in [0, n]; out has n + 1 entries.
void ExclusiveScanU32(Ctx& c, const uint32_t* in, uint64_t* out, uint64_t n);
// sync D2H of one value (and of a second one into *value2 when value2 is not null)
uint64_t ReadU64(Ctx& c, const uint64_t* dptr, const uint64_t* dptr2 = nullptr,
                 uint64_t* value2 = nullptr);

void TimerBegin(Ctx& c, const char* name);
void TimerEnd(Ctx& c);
void TimerCollect(Ctx& c);
void TimerReset(Ctx& c);

// ---- bases.cu ----
// rvn_reads_upload*: the read tables and the bases (whole_set: rvn_reads_upload /
// rvn_reads_upload_ids, where option host_bases applies)
void UploadReads(Ctx& c, const uint64_t* words, const uint64_t* word_off, const uint32_t* lens,
                 const uint32_t* ids, uint32_t n_reads, uint32_t res_first = 0,
                 uint32_t res_last = 0xFFFFFFFFu, bool whole_set = false);
// rvn_reads_upload_files: the set whose words the parse left in d_words (word_off, lens:
// its tables) becomes the context's read set as after UploadReads of the same words
void AdoptParsedReads(Ctx& c, const uint64_t* word_off, const uint32_t* lens, uint32_t n_reads);
// RVN_ERR_STATE unless the bases of reads [first, last) can be read: the range is empty, the
// bases are on the host (a sketch stages its range), or it lies inside the resident range
void CheckResident(const Ctx& c, uint32_t first, uint32_t last);
void WaitUpload(Ctx& c);  // the context's stream waits for an asynchronous upload
// The bases of reads [first, last) for a sketch launch: the device copy of the set, or
// (host_bases) a half of the staging window that holds them, copied there now unless a half
// already does. The caller checks the range (CheckResident), waits for the view's pieces,
// launches, then calls BasesLaunched.
BaseView SketchBases(Ctx& c, uint32_t first, uint32_t last);
// after the launches that read v: the half may be overwritten behind them, and the range
// BasesNext named is copied into the other half now, beside the kernels that follow
void BasesLaunched(Ctx& c, const BaseView& v);
// the read range the caller sketches next: staged right after the next sketch launch
// (no-op with the bases on the device)
void BasesNext(Ctx& c, uint32_t first, uint32_t last);
uint64_t StagedBaseBytes(const Ctx& c);  // device bytes of the staging window
// the calls that read bases at random positions: a set whose bases are on the host goes to
// d_words whole first (the context is then in device mode until the next upload);
// RVN_ERR_LIMIT when it does not fit the usable memory ("host_bases_budget" when not 0)
void EnsureDeviceBases(Ctx& c);
// rvn_map_external's rider: a read outside the uploaded set, its words in the caller's host
// memory, rides in the spare slot n_reads while the guard lives: in the host and device
// tables, as the resident range and, with the bases on the host, in a half of the staging
// window. The destructor restores the set.
struct RiderRead {
  RiderRead(Ctx& c, const uint64_t* words, uint32_t len, uint32_t id);
  RiderRead(const RiderRead&) = delete;
  ~RiderRead();
  Ctx& c;
  const uint32_t n, res_first, res_last;  // the set's reads and resident range
};
void ReleaseBases(Ctx& c);  // rvn_ctx_destroy: the copy stream and the events

// ---- fastx.cu ----
// rvn_reads_upload_files and rvn_reads_parsed (include/raven_b200.h)
void UploadFiles(Ctx& c, const char* const* paths, uint32_t n_paths);
void ParsedReads(Ctx& c, uint64_t* words, uint64_t* word_off, uint32_t* lens,
                 uint8_t* block_quality, uint64_t* bq_off, char* names, uint64_t* name_off);

// ---- sketch.cu ----
void EnsureTiles(Ctx& c);
// full minimizers of reads [first,last) into c.sk (no-op if already there)
void EnsureSketch(Ctx& c, uint32_t first, uint32_t last);
// micromizers of reads [first,last) into c.mm and their thresholds into c.qt (needs the
// sketch of a range that contains [first,last))
void EnsureMicromizers(Ctx& c, uint32_t first, uint32_t last);
// only the thresholds and counts of reads [first, last) into c.qt
void EnsureThresholds(Ctx& c, uint32_t first, uint32_t last);
// The sketch records of reads [first, last) straight into the two tiers of an index build
// (SketchFastKernel's tier-output mode; raven's stage-1 parameters k <= 15, w = 5 only,
// SketchTiersFused): value <= limit as (value, origin) to a_val / a_org, the others as bare
// keys to b_val, each in (read, position) order. *n_a / *n_b: the records of each stream;
// a stream beyond its capacity (cap_a, cap_b) is only counted, and the caller repeats the
// call with room for all of them.
bool SketchTiersFused(const Ctx& c);
void SketchTiers(Ctx& c, uint32_t first, uint32_t last, uint32_t limit, uint32_t* a_val,
                 uint64_t* a_org, uint64_t cap_a, uint32_t* b_val, uint64_t cap_b,
                 uint64_t* n_a, uint64_t* n_b);

// The sketch records of reads [first, last) behind the `base` records that out_val / out_org
// (room for cap records in all) already hold, in (read, position) order (SketchFastKernel's
// append mode, SketchTiersFused parameters only): sweep 2 of the untiered chunked build
// calls it chunk after chunk, `base` being the records of the chunks before, without a
// copy of the chunk's sketch. Records past cap are only counted. SketchAppendTotal: the
// records of the stream after the last call, base included (synchronises).
void SketchAppend(Ctx& c, uint32_t first, uint32_t last, uint32_t* out_val, uint64_t* out_org,
                  uint64_t base, uint64_t cap);
uint64_t SketchAppendTotal(Ctx& c);

// ---- index.cu ----
// value_limit: records whose value exceeds it are counted (occurrence threshold)
// but not indexed - the caller guarantees that no query value is larger
void BuildIndex(Ctx& c, uint32_t first, uint32_t last, bool minhash,
                uint64_t value_limit = ~0ULL);
uint64_t MaxMicromizerValue(Ctx& c, uint32_t first, uint32_t last);
// The same index as BuildIndex(c, first, last, minhash, limit) with limit = the largest of
// `tmax` and the batch's micromizer values (returned; tmax itself with minhash), built
// from chunks of reads of >= chunk bases: no sketch of the whole batch is ever held.
// minhash: one sweep appends each chunk's micromizers to the sort's input. Otherwise
// sweep 1 sketches each chunk and keeps its thresholds (c.jt); sweep 2 sketches it
// again and appends its records to the sort's input - tiered: split into tier A
// (c.i_val_alt / c.i_org_alt) and bare keys (c.t_b0), at k <= 15, w = 5 straight from
// the sketch kernel (SketchTiers).
// tiers = false: the untiered index BuildIndex(c, first, last, minhash) builds, which full
// sketches may probe (tmax is returned as it came); its records go to c.i_val_alt /
// c.i_org_alt, at k <= 15, w = 5 straight from the sketch kernel (SketchAppend).
uint64_t BuildIndexChunked(Ctx& c, uint32_t first, uint32_t last, bool minhash,
                           uint64_t chunk, uint64_t tmax, bool tiers = true);
// bases of reads [first, last)
uint64_t ReadBases(const Ctx& c, uint32_t first, uint32_t last);
// reads [first, last) cut into ranges of >= chunk bases at read boundaries, by the rule
// that cuts index batches (construct.cc:36-44): boundaries first, ..., last
std::vector<uint32_t> ChunkCuts(const Ctx& c, uint32_t first, uint32_t last, uint64_t chunk);
// after the frequency filter of a chunked build: frees what only the build used (the
// chunk sketch, the sort's second buffers, the tiers' staging and bare keys)
void ReleaseIndexBuild(Ctx& c);
// index from device records already in (read, position) order (values as u32
// or u64, see ValView)
// count_bare: the bare keys of a tiered build are counted by partition + BareCountKernel
// (c.bare_count permitting) instead of being sorted
void BuildIndexFrom(Ctx& c, ValView src_val, const uint64_t* src_org, uint64_t n,
                    uint64_t index_bases, uint64_t value_limit = ~0ULL, bool count_bare = false);

// ---- radix.cu ---- stable LSD radix sort on key bits [begin_bit, end_bit).
// The source arrays are only read (src may alias buffer b: it is dead once the
// first pass is through); the result lands in buffer a (return 0) or b (return
// 1); -1 = nothing to do, the source order is the result.
int RadixSortPairs(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b,
                   const uint64_t* src_vals, uint64_t* vals_a, uint64_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending = false);
int RadixSortPairs(Ctx& c, const uint64_t* src_keys, uint64_t* keys_a, uint64_t* keys_b,
                   const uint64_t* src_vals, uint64_t* vals_a, uint64_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending = false);
int RadixSortPairs(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b,
                   const uint32_t* src_vals, uint32_t* vals_a, uint32_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending = false);
int RadixSortPairs(Ctx& c, const uint64_t* src_keys, uint64_t* keys_a, uint64_t* keys_b,
                   const uint32_t* src_vals, uint32_t* vals_a, uint32_t* vals_b, uint64_t n,
                   int begin_bit, int end_bit, bool descending = false);
int RadixSortKeys(Ctx& c, const uint32_t* src_keys, uint32_t* keys_a, uint32_t* keys_b,
                  uint64_t n, int begin_bit, int end_bit);
// unstable partition of u32 keys on bits [begin_bit, end_bit) (at most 10): digit d's
// keys land in dst[bin_start[d], bin_start[d + 1]) (n past the last digit), in any order
void RadixPartitionKeys(Ctx& c, const uint32_t* src, uint32_t* dst, uint64_t n, int begin_bit,
                        int end_bit, uint32_t* bin_start);
// run-length histogram of the index keys (c.i_hist: 65536 u64 bins + #keys), filled by the build
uint64_t* IndexHistogram(Ctx& c);
uint32_t ThresholdFromHistogram(Ctx& c, const uint64_t* h_hist, uint64_t n_keys,
                                double frequency, bool* needs_long_runs);
uint32_t FilterIndex(Ctx& c, double frequency);

// ---- map.cu ----
// fetch = copy the ordered overlaps to the host (rvn_map); stage 1 keeps them
// on the device (c.m_ovl, c.m_ovl_off, c.r_n_ovl)
void MapRange(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal,
              bool avoid_symmetric, bool minhash, bool want_filtered,
              bool fetch = true);

// chains hits grouped by query read (see map.cu); overlaps land in c.m_ovl
// lhs_ids[i] = id of query read i of the batch (device)
uint64_t ChainGroupedHits(Ctx& c, const uint64_t* hg, const uint64_t* hp,
                          const uint64_t* read_hit_off,
                          const std::vector<uint64_t>& h_rho, const uint32_t* lhs_ids,
                          uint32_t nr, uint64_t n_hits, uint64_t n_q);

// ---- gather.cu ----
void GatherReset(Ctx& c);
// one flush over the reads of window `w` (lists, counts and offsets by slot).
// row_off null: the lists are compact (c.g_off) and are re-compacted; otherwise
// every slot owns a fixed row of row_stride records at row_off[slot] and the lists
// stay in their rows
// mark_off (compact lists only): set to the new compact offset of slot `mark`, read
// back with the lists' total
void GatherFlush(Ctx& c, const rvn_overlap* ovl, const uint64_t* q_ovl_off,
                 uint64_t m, uint32_t k0, uint32_t k1, uint64_t kmax, const Window& w,
                 const uint64_t* row_off = nullptr, uint64_t row_stride = 0,
                 uint32_t mark = 0, uint64_t* mark_off = nullptr);
void GatherFetch(Ctx& c);
// the window tables: row_off[s] = s * stride, pile_off[s] = first bin of slot s
// in a pile buffer that holds the window's piles in slot order (both nw + 1)
void WindowTables(Ctx& c, const Window& w, const uint64_t* d_poff, uint64_t stride,
                  uint64_t* row_off, uint64_t* pile_off);

// ---- dist.cu ---- key-partitioned index, reads owned by id mod parts
// which: 0 = full minimizers, 1 = micromizers; records of reads [first,last)
// stably partitioned by value % parts; counts[parts]
void DistSketchSplit(Ctx& c, uint32_t first, uint32_t last, int which, uint32_t parts,
                     const uint64_t** d_val, const uint64_t** d_org, uint64_t* counts);
void DistHitsSplit(Ctx& c, const uint64_t* d_qval, const uint64_t* d_qorg, uint64_t n_q,
                   bool avoid_equal, bool avoid_symmetric, uint32_t parts, uint32_t n_query,
                   const uint64_t** d_grp, const uint64_t** d_pos, const uint32_t** d_lhs,
                   uint64_t* counts);
void DistChainOwned(Ctx& c, const uint64_t* d_grp, const uint64_t* d_pos,
                    const uint32_t* d_lhs, uint64_t n_hits, uint32_t n_seg,
                    const uint64_t* h_seg_off, uint32_t mod, uint32_t rem, uint32_t n_query,
                    const rvn_overlap** d_ovl, uint64_t* n_ovl);
void DistOverlapsSplit(Ctx& c, uint32_t parts, uint32_t self, const rvn_overlap** d_out,
                       uint64_t* counts);
void DistStage1Begin(Ctx& c, uint32_t parts, uint32_t rank);
void DistStage1Add(Ctx& c, const rvn_overlap* d_ovl, uint64_t n_ovl, uint32_t n_seg,
                   const uint64_t* h_seg_off, uint32_t n_query, uint64_t kmax, uint64_t qb);
void DistStage1End(Ctx& c);
void ArenaClosePeers(Ctx& c);
void ArenaExport(Ctx& c, uint64_t bytes, void* handle64);
void ArenaImport(Ctx& c, uint32_t parts, uint32_t rank, const void* handles);
void ArenaPut(Ctx& c, uint32_t dest, uint64_t dst_off, const void* d_src, uint64_t bytes);
void ArenaFlush(Ctx& c);
void ArenaRelease(Ctx& c);

// ---- editdist.cu ---- batched global edit distance of read substrings
void StagePileRegions(Ctx& c, uint32_t coverage, uint32_t* h_begin, uint32_t* h_end,
                      uint16_t* h_median, uint8_t* h_invalid);
void AlignBreakingPoints(Ctx& c, uint64_t n, const uint32_t* q_read, const uint32_t* q_begin,
                         const uint32_t* q_len, const uint8_t* strand, const uint32_t* t_read,
                         const uint32_t* t_begin, const uint32_t* t_len, uint32_t window,
                         const uint64_t* bp_off, int32_t* distance, uint32_t* bp);
void EditDistanceBatch(Ctx& c, uint64_t n, const uint32_t* lhs_read, const uint32_t* lhs_begin,
                       const uint32_t* lhs_len, const uint32_t* rhs_read,
                       const uint32_t* rhs_begin, const uint32_t* rhs_len,
                       const uint8_t* strand, const int32_t* limit, int32_t* out);

// The device half of the edit-distance tiers: distances of the n pairs listed in d_list
// (indices into d_pairs, in any order; the list is reordered), out[slot] per pair: the
// distance, or -1 when it exceeds the pair's limit (limit[slot] >= 0) - above the limit a
// distance may also come back exact. max_q_len: the longest lhs substring of the pairs.
void MyersTiers(Ctx& c, const PairDesc* d_pairs, uint32_t* d_list, uint32_t n,
                const int32_t* d_limit, int32_t* d_out);

// Stage 2's clip and identity filter (construct.cc:385-424) of the flush's n overlaps,
// grouped by query read (d_off, nr + 1 entries): OverlapClip against the pile regions of
// c.s2_rbeg / c.s2_rend, the edit distance of each clipped overlap that keeps one, and the
// kept clipped overlaps compacted stably into d_out with per-read offsets d_out_off.
// Returns how many were kept.
uint64_t Stage2ClipFilter(Ctx& c, const rvn_overlap* d_ovl, const uint64_t* d_off, uint32_t nr,
                          uint64_t n, double identity, rvn_overlap* d_out, uint64_t* d_out_off);

// ---- pile.cu ----
// Pile::AddKmers (pile.cc:64-120) for the filtered positions the last MapRange left on
// the device (c.m_filtered, c.m_filtered_off) of query reads [first, first + nr): marks
// bit pos >> 4 of the read's bitmap in c.s2_bits when the k-mer passes the complexity
// test, and sets the touched flag of every read with a filtered position.
void Stage2KmerMarks(Ctx& c, uint32_t first, uint32_t nr, uint32_t k);

// data: device u16 bins of the piles of window `w` in slot order, off: their device
// u64 offsets (w.size() + 1), `bins` of them in all. No overlap may name a pile of a
// slot below `first`: the coverage pass skips those piles, and neither reads nor
// writes their bins.
void PileAddLayersDevice(Ctx& c, uint16_t* d_data, const uint64_t* d_off, uint64_t bins,
                         const Window& w, const rvn_overlap* d_ovl, uint64_t n_ovl,
                         uint32_t first = 0);

// ---- stage.cu ---- the overlap stages' host drivers
// raven::FindOverlapsAndCreatePiles: index batches of >= ib bases, query flushes of >= qb
// bases (0: the reference's 2^32 and 2^30)
void Stage1(Ctx& c, double freq, uint64_t kmax, bool minhash, uint64_t ib, uint64_t qb);
// raven::FindOverlapsAndRepetetiveRegions' device work over the first n uploaded reads,
// with their valid regions [h_rbeg, h_rend)
void Stage2(Ctx& c, double freq, double identity, uint32_t n, const uint32_t* h_rbeg,
            const uint32_t* h_rend);
// rvn_map over reads [first, last) in flushes; each: called after every flush instead of
// gathering its results on the host (stage 2)
void MapFlushes(Ctx& c, uint32_t first, uint32_t last, bool avoid_equal, bool avoid_symmetric,
                bool minhash, bool want_filtered,
                const std::function<void(uint32_t, uint32_t)>& each = nullptr);
// option "host_bases" at an upload of the whole set (h_woff, h_len, h_pile_off are the new
// set's): whether its bases stay on the host
bool UseHostBases(const Ctx& c);
// device memory a pass can use: `budget`, or when that is 0 the free memory plus the
// buffers this context already holds (a pass re-uses them)
double UsableMemory(const Ctx& c, uint64_t budget);
// rvn_minimize and rvn_filter (returns the occurrence threshold)
void Minimize(Ctx& c, uint32_t first, uint32_t last, bool minhash);
uint32_t Filter(Ctx& c, double freq);
// the estimates rvn_stage1_footprint, rvn_index_footprint and rvn_minimize_footprint
// return, into the outputs that are not null
void Stage1Footprints(const Ctx& c, uint64_t kmax, uint64_t ib, uint64_t qb,
                      uint64_t* resident, uint64_t* windowed_device, uint64_t* windowed_host);
void IndexFootprints(const Ctx& c, uint64_t ib, uint64_t* one_shot, uint64_t* chunked);
void MinimizeFootprints(const Ctx& c, uint32_t first, uint32_t last, uint64_t* one_shot,
                        uint64_t* chunked, uint64_t* chunk);

// ---- poa.cu ---- racon window consensus over a flat batch of windows
// the flat layout of a batch of windows in device memory (rvn_poa_batch's arguments)
struct PoaInput {
  const uint32_t* win_first = nullptr;
  const uint64_t* seq_off = nullptr;
  const uint8_t* bases = nullptr;
  const uint8_t* quals = nullptr;  // null: no qualities
  const uint32_t* seq_begin = nullptr;
  const uint32_t* seq_end = nullptr;
};
// the consensus of windows already on the device; h_*: host copies of the tables
void PoaRun(Ctx& c, uint32_t n_windows, const uint32_t* h_win_first, const uint64_t* h_seq_off,
            const uint32_t* h_seq_begin, const uint32_t* h_seq_end, const PoaInput& d, int m,
            int n, int gap, bool trim, bool tgs, bool want_coverage);
void PoaBatch(Ctx& c, uint32_t n_windows, const uint32_t* h_win_first,
              const uint64_t* h_seq_off, const uint8_t* h_bases, const uint8_t* h_quals,
              const uint32_t* h_seq_begin, const uint32_t* h_seq_end, int m, int n,
              int gap, bool trim, bool tgs, bool want_coverage);

// ---- layers.cu ---- racon's layers of every window built on the device from the
// uploaded reads and the breaking points, then PoaRun over batches of windows
// (include/raven_b200.h, rvn_polish_windows)
struct PolishArgs {
  uint64_t n_aln;
  const uint32_t *q_read, *q_begin, *q_len;
  const uint8_t* strand;
  const uint32_t* t_read;
  const uint64_t* bp_off;
  const uint32_t* bp;
  uint32_t n_targets, window;
  const uint8_t* bq;
  const uint64_t* bq_off;
  const uint8_t* rc;
  double q;
  int m, n, gap;
  bool trim, tgs;
};
void PolishWindows(Ctx& c, const PolishArgs& a);

// Pile::AddKmers low-complexity test for (read index, position) pairs
void KmerComplexity(Ctx& c, const uint32_t* h_read_idx, const uint32_t* h_pos,
                    uint64_t n, uint32_t k, uint8_t* h_keep);

}  // namespace rvn
