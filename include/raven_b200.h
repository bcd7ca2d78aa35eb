/* raven_b200 — C ABI of the H100-native (sm_90a) overlap engine.
 *
 * This is the drop-in boundary for the reference's overlap hot path. The
 * reference has no FFI layer of its own: RavenLib calls C++ classes of
 * un-vendored dependencies directly. Every entry point below replaces one of
 * those call sites (file:line are into lbcb-sci/raven @ v1.8.3):
 *
 *   rvn_engine_configure   ram::MinimizerEngine ctor   RavenLib/src/construct.cc:661-662
 *   rvn_reads_upload       biosoup::NucleicAcid fields RavenLib/include/raven/graph/graph.h:13-18
 *   rvn_minimize           MinimizerEngine::Minimize   RavenLib/src/construct.cc:42-43,363
 *   rvn_filter             MinimizerEngine::Filter     RavenLib/src/construct.cc:44,372
 *   rvn_map / rvn_map_external
 *                          MinimizerEngine::Map        RavenLib/src/construct.cc:59-64,377-381
 *   rvn_pile_add_layers    raven::Pile::AddLayers      RavenLib/src/pile.cc:33-62
 *   rvn_kmer_complexity    raven::Pile::AddKmers       RavenLib/src/pile.cc:64-120
 *   rvn_poa_batch          racon::Polisher::Polish (window consensus: racon::Window +
 *                          spoa)                       RavenLib/src/polish.cc:43-51
 *   rvn_edit_distance_batch
 *                          edlibAlign(lhs, rhs, edlibDefaultAlignConfig()) of the
 *                          identity filter      RavenLib/src/construct.cc:176-199,
 *                                                                        :393-416
 *   rvn_stage1_pile_regions
 *                          raven::Pile::FindValidRegion + FindMedian of
 *                          raven::TrimAndAnnotatePiles RavenLib/src/construct.cc:123-152
 *   rvn_align_breaking_points
 *                          edlibAlign(read, unitig, NW, EDLIB_TASK_PATH) + the window
 *                          breaking points of racon::Polisher::Polish
 *                                                      RavenLib/src/polish.cc:43-51
 *   rvn_polish_windows     the window layers and consensus of racon::Polisher::Polish
 *                                                      RavenLib/src/polish.cc:43-51
 *   rvn_find_overlaps_and_create_piles
 *                          raven::FindOverlapsAndCreatePiles
 *                                                      RavenLib/src/construct.cc:14-121
 *   rvn_find_overlaps_and_repetitive_regions
 *                          the map, Pile::AddKmers and identity-filter part of
 *                          raven::FindOverlapsAndRepetetiveRegions
 *                                                      RavenLib/src/construct.cc:352-424
 *
 * The C++ facade over this ABI (include/ram/minimizer_engine.hpp and
 * raven_b200/host/) keeps the reference's class and function signatures, so
 * RavenLib's own sources compile against it unchanged (INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes, POD structs, `int` status (0 = ok,
 * negative = error; text via rvn_last_error). No exceptions or C++ types
 * cross this line. Output arrays are owned by the context and stay valid
 * until the next call on the same context that produces the same kind of
 * output, or rvn_ctx_destroy. A context is not thread-safe; use one per
 * host thread / GPU. There is NO CPU fallback: every compute entry point
 * fails with RVN_ERR_CUDA when no sm_90 (H100) device is usable.
 */
#ifndef RAVEN_B200_H_
#define RAVEN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RVN_OK 0
#define RVN_ERR_INVALID (-1) /* bad argument (mirrors std::invalid_argument) */
#define RVN_ERR_CUDA (-2)    /* CUDA runtime / no device */
#define RVN_ERR_STATE (-3)   /* call order (e.g. map before minimize) */
#define RVN_ERR_LIMIT (-4)   /* input beyond a documented limit */

typedef struct rvn_ctx rvn_ctx;

/* biosoup::Overlap without the alignment string
 * (field order: RavenLib/src/overlap_utils.cc:5-8) */
typedef struct rvn_overlap {
  uint32_t lhs_id, lhs_begin, lhs_end;
  uint32_t rhs_id, rhs_begin, rhs_end;
  uint32_t score;
  uint32_t strand; /* 1 = same strand */
} rvn_overlap;

/* Counters of the last rvn_map / stage-1 call; the roofline's algorithmic
 * bytes are computed from these (DESIGN.md "algorithmic bytes"). */
typedef struct rvn_stats {
  uint64_t index_bases;     /* bases sketched for the index */
  uint64_t index_records;   /* minimizer records indexed */
  uint64_t index_keys;      /* distinct minimizer values */
  uint64_t query_bases;     /* bases sketched as queries */
  uint64_t query_records;   /* query minimizers probed */
  uint64_t hits;            /* seed hits expanded */
  uint64_t overlaps;        /* overlaps emitted by chaining */
  uint64_t pile_bins;       /* pile bins updated */
  uint64_t kernel_launches; /* kernels of this library launched */
  uint32_t occurrence;      /* frequency threshold in force */
  uint32_t reserved;
} rvn_stats;

int rvn_version(void);

/* device: CUDA ordinal. stream: a cudaStream_t to run on (e.g. torch's
 * current stream) or NULL for a stream owned by the context. The environment variable
 * RVN_SET_OPTIONS="name=value,..." sets rvn_set_option options on every context created
 * (for programs that reach the library only through a facade); a bad entry fails the
 * call with RVN_ERR_INVALID. */
int rvn_ctx_create(int device, void* stream, rvn_ctx** out);
void rvn_ctx_destroy(rvn_ctx* ctx);
const char* rvn_last_error(const rvn_ctx* ctx);

/* ram::MinimizerEngine(pool, k, w, bandwidth, chain, matches, gap);
 * k is clamped to [1, 31] like the reference engine. Drops any index. */
int rvn_engine_configure(rvn_ctx* ctx, uint32_t k, uint32_t w,
                         uint32_t bandwidth, uint32_t chain, uint32_t matches,
                         uint32_t gap);

/* The read set, in the biosoup wire format: read i is words[word_off[i] ..
 * word_off[i+1]) (32 bases per word, base j at bits [(j<<1)&63,+1] of word
 * j>>5), lens[i] bases, id = i. Host buffers; copied to the device. */
int rvn_reads_upload(rvn_ctx* ctx, const uint64_t* words,
                     const uint64_t* word_off, const uint32_t* lens,
                     uint32_t n_reads);

/* As rvn_reads_upload, but only the bases of reads [first,last) are copied to
 * the device (lengths of all reads are): a rank of a partitioned run only
 * sketches its own range. Sketching any other read is RVN_ERR_STATE. */
int rvn_reads_upload_range(rvn_ctx* ctx, const uint64_t* words,
                           const uint64_t* word_off, const uint32_t* lens,
                           uint32_t n_reads, uint32_t first, uint32_t last);


/* Same, with explicit sequence ids (biosoup::NucleicAcid::id): origins and
 * overlap ids carry ids[i] instead of i. raven re-sorts its sequence vector
 * before stage 2 (construct.cc:324-349), so id != position there. */
int rvn_reads_upload_ids(rvn_ctx* ctx, const uint64_t* words,
                         const uint64_t* word_off, const uint32_t* lens,
                         const uint32_t* ids, uint32_t n_reads);

/* raven's input loop (RavenExe/src/main.cc:258-299: raven::CreateParser, RavenLib/src/io.cc:7-41,
 * then Parse(-1) per file, files concatenated in order, empty files skipped) with the records
 * parsed and packed on the device; the result is the context's read set (ids 0..n-1), as after
 * rvn_reads_upload. sizes (may be NULL): reads, words, block qualities, name bytes.
 * Plain and gzip files (multi-member included) are read with zlib's gzread on a thread of the
 * library's own, in chunks of option "fastx_chunk_bytes" (results do not depend on it). A file
 * whose first member is a whole BGZF member (bgzip, samtools; any suffix) is read raw instead
 * and its members are inflated on the device, to the same text: at the first gzip member that
 * is not a whole BGZF member the rest of the file goes to zlib, and bytes after the last member
 * that do not begin a gzip header are ignored, as zlib ignores them.
 * Option "host_bases" applies to the parsed set. Errors: RVN_ERR_INVALID with the message
 * the reference's loop prints for the first failing record in file order (an unsupported
 * suffix, a file that cannot be opened, "invalid file format" wherever the drop-in FASTA or
 * FASTQ parser throws, "not a nucleotide"); RVN_ERR_LIMIT for a read of 2^31 bases or more,
 * or words that do not fit the device while the set is parsed (naming the bytes). After a
 * failed call the context holds no read set (the calls on reads are RVN_ERR_STATE until the
 * next upload). Phases in rvn_get_timings: "fastx_read" (host read or inflate that nothing
 * hid), "fastx_copy" (text, or a BGZF file's compressed bytes), "fastx_inflate" (BGZF files
 * only) and "fastx_parse" (per chunk). A BGZF member that does not inflate to its CRC and
 * ISIZE fails the call with the drop-in's "unable to read file". */
int rvn_reads_upload_files(rvn_ctx* ctx, const char* const* paths, uint32_t n_paths,
                           uint64_t sizes[4]);

/* Host copies of the parsed set; any pointer may be NULL. bq_off as rvn_polish_windows takes it
 * (an empty range for a FASTA read); names are cut at the first white space, as raven's parser
 * does, name i = names[name_off[i] .. name_off[i+1]). RVN_ERR_STATE if the current set was not
 * made by rvn_reads_upload_files. */
int rvn_reads_parsed(rvn_ctx* ctx, uint64_t* words, uint64_t* word_off, uint32_t* lens,
                     uint8_t* block_quality, uint64_t* bq_off, char* names, uint64_t* name_off);

/* Where the packed bases of the current upload live (option "host_bases"): *on_host = 1
 * when they stay in the context's pinned host copy and the sketch kernels read them from a
 * staging window, 0 when the device holds the whole set; *device_word_bytes = the device
 * bytes of packed words held for them (the staging window, or the whole set). Either
 * output may be NULL. */
int rvn_reads_residency(rvn_ctx* ctx, int* on_host, uint64_t* device_word_bytes);

/* Minimize(reads[first..last), minhash): sketch and index. The index holds every record
 * (full sketches may probe it). Option "index_chunk_bases" applies: built in chunks, no
 * sketch of the whole range is held, and the rvn_filter that follows frees the build's
 * buffers; the index, the threshold and every map result are the one-shot build's. */
int rvn_minimize(rvn_ctx* ctx, uint32_t first, uint32_t last, int minhash);

/* Filter(frequency): occurrence threshold of the current index.
 * frequency outside [0,1] -> RVN_ERR_INVALID (reference throws). */
int rvn_filter(rvn_ctx* ctx, double frequency, uint32_t* occurrence);

/* Map(read, avoid_equal, avoid_symmetric, minhash[, &filtered]) for every
 * read in [first, last) against the current index. Overlaps come back
 * grouped by query in ascending id, each group in the reference engine's
 * emission order; ovl_off has (last-first)+1 entries. `filtered` are the
 * positions of over-frequent query minimizers (only if want_filtered). */
/* The range is worked in flushes of query bases, as the reference cuts its queries
 * (construct.cc:67): 2^30 bases, fewer when the device has less room; the hits, chain
 * scratch and overlaps of one flush are on the device at a time and the results are those
 * of one piece. A multi-flush call leaves one phase "map_flush" per flush in
 * rvn_get_timings. */
int rvn_map(rvn_ctx* ctx, uint32_t first, uint32_t last, int avoid_equal,
            int avoid_symmetric, int minhash, int want_filtered);
/* Map one read that is NOT in the uploaded set (e.g. a query of an earlier
 * index batch, construct.cc:59; plasmids vs unitigs, assemble.cc:757,780).
 * Results through rvn_map_results with a single query. */
int rvn_map_external(rvn_ctx* ctx, const uint64_t* words, uint32_t len,
                     uint32_t id, int avoid_equal, int avoid_symmetric,
                     int minhash, int want_filtered);
int rvn_map_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                    const uint64_t** ovl_off, uint64_t* n_overlaps,
                    const uint32_t** filtered, const uint64_t** filt_off);

/* Pile::AddLayers on a batch of piles: pile i has bins[i] uint16 counters at
 * data + bin_off[i]; every overlap adds +1 to bins [(begin>>4)+1, (end>>4)-1)
 * of the pile of its lhs and of its rhs read, saturating at 65535.
 * Precondition (holds for every chained overlap): *_end >= 16. */
int rvn_pile_add_layers(rvn_ctx* ctx, uint16_t* data, const uint64_t* bin_off,
                        uint32_t n_piles, const rvn_overlap* overlaps,
                        uint64_t n_overlaps);

/* The low-complexity test of Pile::AddKmers (RavenLib/src/pile.cc:64-120) for
 * n (read index, position) pairs - the positions rvn_map reports as filtered
 * (construct.cc:377-383): keep[i] = 1 iff the k-mer at positions[i] survives
 * the three compressions, i.e. iff the reference sets kmers_[position >> 4]. */
int rvn_kmer_complexity(rvn_ctx* ctx, const uint32_t* read_index,
                        const uint32_t* positions, uint64_t n, uint32_t kmer_len,
                        uint8_t* keep);

/* The identity filter's edlibAlign(lhs, rhs, edlibDefaultAlignConfig()).editDistance
 * (RavenLib/src/construct.cc:176-199 and :393-416) for n_pairs overlaps at once:
 * pair i aligns bases [lhs_begin, +lhs_len) of uploaded read lhs_read[i] with
 * [rhs_begin, +rhs_len) of read rhs_read[i], the latter reverse complemented when
 * strand[i] == 0 (construct.cc:184-188). Reads are addressed by their index in
 * the uploaded set. limit (may be NULL): limit[i] >= 0 bounds the search -
 * distance[i] = -1 if the distance exceeds it (the filter only needs to know that
 * 1 - ed/max(len) < identity); limit[i] < 0: exact distance, whatever it takes. */
int rvn_edit_distance_batch(rvn_ctx* ctx, uint64_t n_pairs, const uint32_t* lhs_read,
                            const uint32_t* lhs_begin, const uint32_t* lhs_len,
                            const uint32_t* rhs_read, const uint32_t* rhs_begin,
                            const uint32_t* rhs_len, const uint8_t* strand,
                            const int32_t* limit, int32_t* distance);

/* raven::TrimAndAnnotatePiles' first two steps for every pile (RavenLib/src/construct.cc:
 * 123-152: Pile::FindValidRegion(coverage) and Pile::FindMedian, pile.cc:122-172), on
 * the piles the last rvn_find_overlaps_and_create_piles call left on the device - no
 * round trip of the histograms. Per read i: invalid[i] = 1 if the reference marks the
 * pile invalid (no run of bins >= coverage followed by a lower bin, or one shorter than
 * 1260 >> 4 bins; begin/end then stay 0 / bins like the reference's fields); else
 * [begin[i], end[i]) is the valid region in bins and median[i] the element of rank
 * size/2 of it. The caller zeroes the bins outside the region like UpdateValidRegion.
 * After a windowed call (option "stage1_window") the piles are in host memory and pass
 * through the device in chunks of reads; the outputs are the same.
 * RVN_ERR_STATE if another call has replaced the device piles since. */
int rvn_stage1_pile_regions(rvn_ctx* ctx, uint32_t coverage, uint32_t* begin, uint32_t* end,
                            uint16_t* median, uint8_t* invalid);

/* The read-to-target alignments of racon::Polisher::Polish (RavenLib/src/polish.cc:43-51:
 * edlibAlign(query, target, EDLIB_MODE_NW, EDLIB_TASK_PATH) per read) and the walk along
 * each path that cuts it at the target's windows, for n_pairs alignments at once.
 * Pair i: query = bases [q_begin, +q_len) of uploaded read q_read[i], reverse
 * complemented as a whole when strand[i] == 0; target = bases [t_begin, +t_len) of read
 * t_read[i]. The path is the ONE upstream edlib returns (its traceback order and its
 * Hirschberg split of large problems are kept), so the cuts are the reference's.
 * Output: distance[i] = the edit distance, and for every window x of `window` target
 * bases that the target substring touches (x = t_begin/window .. (t_begin+t_len-1)/window)
 * the slot s = bp_off[i] + (x - t_begin/window) of breaking_points (4 values per slot):
 *   [4s+0] target position of the first match/mismatch column inside the window,
 *   [4s+1] its query position (0-based inside the oriented query substring),
 *   [4s+2], [4s+3] one past the last such pair;
 * all four 0xFFFFFFFF when no match/mismatch falls into the window. bp_off (n_pairs + 1
 * entries, computed by the caller) must count exactly those windows. */
int rvn_align_breaking_points(rvn_ctx* ctx, uint64_t n_pairs, const uint32_t* q_read,
                              const uint32_t* q_begin, const uint32_t* q_len,
                              const uint8_t* strand, const uint32_t* t_read,
                              const uint32_t* t_begin, const uint32_t* t_len, uint32_t window,
                              const uint64_t* bp_off, int32_t* distance,
                              uint32_t* breaking_points);

/* raven::FindOverlapsAndRepetetiveRegions up to its classification loop
 * (RavenLib/src/construct.cc:352-424; the loop, :430-455, and what follows it stay with
 * the caller). The caller uploads the reads in the reference's sorted order (valid
 * piles first, then by id, construct.cc:325-334), with their ids (rvn_reads_upload_ids);
 * n_valid is that order's s (construct.cc:343-349: 0 when no pile is invalid, and then
 * nothing is mapped). region_begin[i] / region_end[i]: Pile::begin() / end() of valid
 * read i, in bases.
 * Schedule, as the reference's: index batches [j, i + 1) of the valid reads, cut when
 * they reach 1U << 30 bases (option "stage2_batch_bases" forces a smaller cut), each an
 * untiered full-sketch index (Minimize) filtered at `frequency` (Filter); then every
 * valid read of [0, i + 1) is mapped (avoid equal, avoid symmetric, no minhash, filtered
 * positions kept: construct.cc:377-381) in rvn_map's flushes. On the device, per flush:
 *  - the filtered positions that pass Pile::AddKmers' complexity test (pile.cc:64-120)
 *    set bit position >> 4 of their read's bitmap, ORed over all batches;
 *  - identity != 0: each overlap is clipped to the valid regions (raven::OverlapUpdate,
 *    overlap_utils.cc:14-60) and kept iff 1 - ed / max(len) >= identity (edlibAlign of
 *    the clipped substrings, construct.cc:385-424); identity == 0: overlaps unchanged.
 * Results by rvn_stage2_results. */
int rvn_find_overlaps_and_repetitive_regions(rvn_ctx* ctx, double frequency, double identity,
                                             uint32_t n_valid, const uint32_t* region_begin,
                                             const uint32_t* region_end);
/* Results of the last rvn_find_overlaps_and_repetitive_regions call:
 *  - overlaps: the final (clipped, kept) overlaps of every batch in the order the
 *    reference's classification loop consumes them: batch by batch, query read by query
 *    read, in emission order; overlap_off (n_valid + 1): a batch that ends at valid read i
 *    holds overlaps [overlap_off[i], overlap_off[i + 1]) (an empty range for every other
 *    read);
 *  - kmer_bits: per valid read i the words [kmer_off[i], kmer_off[i + 1]) (n_valid + 1
 *    offsets), bit b of the read at word b >> 5, bit b & 31: Pile::kmers_[b], of
 *    (len >> 4) + 1 bits;
 *  - kmer_touched[i] = 1 iff some batch reported a filtered position of read i, i.e. iff
 *    the reference resized kmers_ (pile.cc:67-72; it may stay all zero);
 *  - n_mapped: the overlaps the map produced, before the clip and the identity filter. */
int rvn_stage2_results(rvn_ctx* ctx, const rvn_overlap** overlaps, const uint64_t** overlap_off,
                       const uint32_t** kmer_bits, const uint64_t** kmer_off,
                       const uint8_t** kmer_touched, uint64_t* n_mapped);

/* The estimates behind option "stage1_window" -1 (auto) for a stage-1 call over the
 * uploaded reads with these arguments (0 = the defaults, as in
 * rvn_find_overlaps_and_create_piles), in bytes: device memory of a resident pass, device
 * memory of a windowed pass, pinned host memory of a windowed pass. Auto runs windowed
 * only when the resident estimate exceeds the free device memory (plus the buffers the
 * context already holds), max_overlaps <= 65536 and both windowed estimates fit. */
int rvn_stage1_footprint(rvn_ctx* ctx, uint64_t max_overlaps, uint64_t index_batch_bases,
                         uint64_t query_batch_bases, uint64_t* resident,
                         uint64_t* windowed_device, uint64_t* windowed_host);

/* The device working set of the largest index batch of a stage-1 call over the uploaded
 * reads with index batches of index_batch_bases (0 = 2^32), in bytes: built in one piece,
 * and built in chunks (option "index_chunk_bases": its chunk size when it is > 0, else
 * 2^30 bases). The estimates of rvn_stage1_footprint use the chunked one when the call
 * would chunk. */
int rvn_index_footprint(rvn_ctx* ctx, uint64_t index_batch_bases, uint64_t* one_shot,
                        uint64_t* chunked);

/* Estimated device memory of rvn_minimize(first, last), in bytes: the reads, the index of
 * every record with the sort's second buffers, and the sketch of the whole range
 * (one_shot) or of one chunk (chunked: option "index_chunk_bases" when it is > 0, else
 * 2^30 bases). chunk: what the call would do under the options in force, 0 = one piece,
 * else its chunk size. */
int rvn_minimize_footprint(rvn_ctx* ctx, uint32_t first, uint32_t last, uint64_t* one_shot,
                           uint64_t* chunked, uint64_t* chunk);

/* raven::FindOverlapsAndCreatePiles over the uploaded read set: index batches
 * of >= index_batch_bases (reference: 1<<32), query flushes of >=
 * query_batch_bases (reference: 1<<30); pass 0 for the reference values.
 * Results: per read the kept overlaps (<= max_overlaps after the reference's
 * truncation rule) and the pile histogram (len>>4 uint16 bins). */
int rvn_find_overlaps_and_create_piles(rvn_ctx* ctx, double frequency,
                                       uint64_t max_overlaps, int minhash,
                                       uint64_t index_batch_bases,
                                       uint64_t query_batch_bases);
int rvn_stage1_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                       const uint64_t** ovl_off, const uint16_t** pile,
                       const uint64_t** pile_off, uint64_t* n_mapped);

/* racon::Window::GenerateConsensus over a batch of windows - the unit of the
 * "POA windows/s" metric; stands in for the consensus phase of
 * racon::Polisher::Polish (RavenLib/src/polish.cc:43-51; raven passes w = 500,
 * trim = true, m/n/g = PolishCfg polish.hpp:13-17). Flat layout: window w owns
 * sequences [win_first[w], win_first[w+1]); the first is the backbone (draft),
 * the others are layers aligned to backbone positions [seq_begin, seq_end]
 * (inclusive, < backbone length); sequence s = bases[seq_off[s]..seq_off[s+1])
 * as upper-case ACGT letters (any other byte -> RVN_ERR_INVALID), quals
 * (Phred+33) at the same offsets, the backbone's included, or NULL (layers weigh
 * 1, the backbone 0 like racon's dummy '!' quality).
 * A layer without bases or with seq_begin == seq_end is dropped like
 * racon::Window::AddLayer drops it: it is no sequence of its window (not for
 * "fewer than 3 sequences", not for the trimming threshold) and its coordinates
 * are not looked at. Any other layer needs seq_begin < seq_end < backbone length
 * (racon itself lets seq_end reach the backbone length) -> RVN_ERR_INVALID.
 * g must be negative (racon throws otherwise -> RVN_ERR_INVALID).
 * Limits, each RVN_ERR_LIMIT for the whole call: 65000 bases in one window
 * (backbone + layers; about 130 layers of a 500-base window), 32000 bases in one
 * layer, 4095 kept layers in one window, a graph beyond 65000 nodes or edges,
 * and int16 scores: max(|m|,|n|,|g|) * (graph nodes + layer bases + 2) <= 32000
 * for every layer. After a failed call rvn_poa_results is RVN_ERR_STATE.
 * Option "poa_wide" (rvn_set_option) lifts those limits: 0 (default) as above; 1 the
 * windows past them - refused up front, or out of graph capacity or int16 range after
 * the retry at their exact bound - run on a kernel with 32-bit ids and int32 cells
 * (same results; the other windows take their usual kernels); 2 every window runs on
 * that kernel (for tests). A wide window's scratch is sized from an estimate and
 * doubled while it runs out, up to its exact bound; one that does not fit the scratch
 * budget of a launch even alone is RVN_ERR_LIMIT, naming the bytes it needs. The budget
 * is 16 GB or half the free device memory, or option "poa_scratch_budget" (bytes) when
 * that is not 0. Phase "poa_wide" in rvn_get_timings is the wide kernel's share.
 * Results: consensus letters per window (cons_off has n_windows+1 entries),
 * status bit 0 = polished (>= 3 sequences), bit 1 = trimming skipped
 * ("might be chimeric"), coverage per consensus base if requested. */
int rvn_poa_batch(rvn_ctx* ctx, uint32_t n_windows, const uint32_t* win_first,
                  const uint64_t* seq_off, const char* bases, const char* quals,
                  const uint32_t* seq_begin, const uint32_t* seq_end, int8_t m,
                  int8_t n, int8_t g, int trim, int tgs, int want_coverage);
int rvn_poa_results(rvn_ctx* ctx, const char** consensus, const uint64_t** cons_off,
                    const uint8_t** status, const uint32_t** coverage,
                    uint64_t* cells);
/* The kernels of the last successful rvn_poa_batch: windows[k] = windows that finished
 * on kernel k, launches[k] = its launches, for k = 0 the register-row (fast) kernel,
 * 1 the generic kernel, 2 the wide kernel ("poa_wide"). Either pointer may be NULL
 * (else 3 entries). RVN_ERR_STATE when there are no POA results. */
int rvn_poa_routes(rvn_ctx* ctx, uint32_t* windows, uint32_t* launches);

/* The window layers and consensus of racon::Polisher::Polish (RavenLib/src/polish.cc:43-51)
 * after the alignments of rvn_align_breaking_points, with the layers built on the device
 * from the uploaded reads: no base of a layer passes through the host.
 * Targets are uploaded reads [0, n_targets); target t owns windows first_window[t] ..
 * first_window[t+1] - 1, ceil(len_t / window) of them, numbered over the targets in order.
 * The backbone of window j of target t is its bases [j*window, min((j+1)*window, len_t)).
 * Alignment a: query = uploaded read q_read[a] (length L), aligned on strand[a] (0 = the
 * read reverse complemented as a whole) to target t_read[a] (< n_targets); its window
 * slots bp_off[a] .. bp_off[a+1] - 1 (bp_off[0] = 0) hold 4 breaking points each, as
 * rvn_align_breaking_points writes them. Per slot x, in order of alignment and slot:
 *   - skipped if bp[4x] == 0xFFFFFFFF;
 *   - qb = q_begin[a], or L - (q_begin[a] + q_len[a]) when strand[a] == 0;
 *     fq = qb + bp[4x+1], lq = qb + bp[4x+3], ft = bp[4x], lt = bp[4x+2];
 *   - dropped unless (double)(lq - fq) >= 0.02 * window;
 *   - if the read has block qualities: dropped if avg < q, avg = the sum of Score(x) over
 *     x in [fq, lq) divided by lq - fq, where Score(x) = block_quality[(f ? L-1-x : x) >> 6]
 *     and f = reverse_complement[read] XOR (strand[a] == 0) (biosoup's Score of the view
 *     the reference aligns);
 *   - ws = (ft / window) * window; dropped if ft - ws >= lt - ws - 1 (unsigned);
 *   - else a layer of window first_window[t] + ft / window with begin = ft - ws and
 *     end = lt - ws - 1: bases [fq, lq) of the read in its aligned orientation, qualities
 *     Score + '!' (a read without qualities: '!' + 1, and no qualities at all when no read
 *     has any); the backbone's quality is '!'.
 * A window's layers keep that order. Qualities: block_quality[bq_off[r] .. bq_off[r+1])
 * for uploaded read r (bq_off has one entry per uploaded read + 1; an empty range = no
 * qualities, else at least one per 64 bases), or block_quality NULL. reverse_complement:
 * biosoup's is_reverse_complement per uploaded read, or NULL (all 0); it only turns the
 * quality index around - the uploaded bases are the read as it reads.
 * The consensus is rvn_poa_batch's (m, n, g, trim, tgs and its options) over that flat
 * layout, run on consecutive windows in batches whose device inputs fit a budget: per
 * window 2 bytes per base (backbone and layers; 3 when some read has qualities), 20 per
 * sequence and 64; the budget is a quarter of the free device memory (with the batch
 * buffers the context holds), or option "poa_batch_bytes" when that is not 0; a batch holds
 * at least one window. *window_batches (may be NULL) = the batches. Results as for
 * rvn_poa_batch, for every window of the call: rvn_poa_results (no coverage),
 * rvn_poa_routes (summed over the batches). Phases "poa_layers" (rules and sort) and
 * "poa_pack" (one per batch) in rvn_get_timings are the device layer build.
 * RVN_ERR_INVALID for bad indices or coordinates, breaking points outside their read or
 * their target's windows, too few block qualities, or g >= 0; RVN_ERR_LIMIT as
 * rvn_poa_batch; RVN_ERR_STATE when the reads were not uploaded. */
int rvn_polish_windows(rvn_ctx* ctx, uint64_t n_alignments, const uint32_t* q_read,
                       const uint32_t* q_begin, const uint32_t* q_len, const uint8_t* strand,
                       const uint32_t* t_read, const uint64_t* bp_off,
                       const uint32_t* breaking_points, uint32_t n_targets, uint32_t window,
                       const uint8_t* block_quality, const uint64_t* bq_off,
                       const uint8_t* reverse_complement, double q, int8_t m, int8_t n, int8_t g,
                       int trim, int tgs, uint32_t* window_batches);

/* ---- introspection (parity tests, profiling) ---- */

/* Per-read sketches of reads [first,last) exactly as the reference engine's
 * Minimize(sequence, minhash) returns them: value[], origin[] and
 * (last-first)+1 offsets. */
int rvn_sketch(rvn_ctx* ctx, uint32_t first, uint32_t last, int minhash,
               const uint64_t** value, const uint64_t** origin,
               const uint64_t** offsets, uint64_t* n_records);

/* The index as sorted (value, origin) records + distinct-key statistics. */
int rvn_index_records(rvn_ctx* ctx, const uint64_t** value,
                      const uint64_t** origin, uint64_t* n_records,
                      uint64_t* n_keys);

/* Seed hits of the last rvn_map call with keep_hits set via rvn_set_option:
 * group[], positions[] and per-query offsets, unsorted within a query. */
int rvn_map_hits(rvn_ctx* ctx, const uint64_t** group,
                 const uint64_t** positions, const uint64_t** hit_off,
                 uint64_t* n_hits);

/* The engine's stable LSD radix sort (raven_b200/csrc/radix.cu - it orders the
 * minimizer index, construct.cc:42-43), in place: keys of 4 or 8 bytes, values of
 * 0 (u32 keys only), 4 or 8 bytes, key bits [begin_bit, end_bit), n < 2^32 - 1;
 * equal keys keep their input order. keys and vals are both host or both device
 * memory; device arrays are sorted where they are, with one more buffer per array. */
int rvn_debug_sort_pairs(rvn_ctx* ctx, int key_bytes, int val_bytes, void* keys,
                         void* vals, uint64_t n, int begin_bit, int end_bit,
                         int descending);

/* The engine's unstable radix partition of u32 keys on bits [begin_bit, end_bit)
 * (1 to 10 bits), in place: the keys of digit d end in keys[bin_start[d],
 * bin_start[d + 1]) in any order (bin_start: 1024 entries, n for the digits past
 * the bit range). keys and bin_start are host or device memory, each on its own. */
int rvn_debug_partition_keys(rvn_ctx* ctx, uint32_t* keys, uint64_t n, int begin_bit,
                             int end_bit, uint32_t* bin_start);

/* The engine's exclusive scan of u32 counts into u64 offsets: out[i] = in[0] + ... +
 * in[i - 1] for i in [0, n] (n + 1 entries). in and out are host or device memory,
 * each on its own. */
int rvn_debug_exclusive_scan(rvn_ctx* ctx, const uint32_t* in, uint64_t n, uint64_t* out);

int rvn_get_stats(rvn_ctx* ctx, rvn_stats* out);

/* options: "keep_hits" (0/1); "tier_min_records" (stage 1 splits an index batch of
 * at least that many minimizers into a probe-able tier and bare keys, default
 * 2^18; 0 = always); "self_join" (0/1, default 1: the seed hits of a stage-1 flush
 * whose reads are inside the index batch come from a self-join over the sorted
 * index instead of a probe per micromizer); "async_upload" (0/1, default 0: with 1,
 * rvn_reads_upload* returns while the packed bases still travel - in chunks, on a
 * copy stream - and the sketch kernel of the next call starts on the reads that
 * have arrived; the caller must keep `words` unchanged until the next call on the
 * context has returned; meant for pinned host memory; ignored when the bases stay on the
 * host); "host_bases" (where rvn_reads_upload and rvn_reads_upload_ids keep the packed
 * bases: 0 = on the device for as long as the upload lives; 1 = in a pinned host copy the
 * context makes during the upload (the caller may change its words once the call returns),
 * and every sketch copies the words of its read range - an index batch, one chunk of a
 * chunked build, or one map flush - into one of two device halves of a staging window,
 * the drivers copying the next range while the current one is sketched and the kernels
 * that read no bases run; -1 = auto, the default: on the host only when the windowed,
 * chunked stage-1 estimate of the reference's schedule (2^32-base index batches, 2^30-base
 * flushes, max_overlaps 32) exceeds the usable device memory with the bases on the device
 * and fits with the staging window instead. rvn_reads_upload_range always keeps them on the
 * device. rvn_edit_distance_batch, rvn_align_breaking_points, rvn_polish_windows,
 * rvn_kmer_complexity and rvn_find_overlaps_and_repetitive_regions read bases at random
 * positions: on a context whose bases are on the host they first copy the whole set to the
 * device (which then holds it until the next upload), or return RVN_ERR_LIMIT naming the
 * bytes when it does not fit. Results are identical in every mode; phase "stage_bases" in
 * rvn_get_timings is the copy time no kernel hid; rvn_reads_residency tells where the bases
 * are); "host_bases_budget" (bytes: replaces the usable device memory in the auto decision
 * and in that fit test, 0 = the free memory); "stage1_window" (where
 * rvn_find_overlaps_and_create_piles keeps the piles and overlap lists of all reads:
 * 0 = on the device for the whole pass; 1 = windowed: in pinned host memory, and
 * each flush brings only the reads it touches - its queries and the current index
 * batch - to the device, so the device holds the packed bases, one index batch and
 * one window; -1 = auto, the default: windowed only when an estimate of the
 * resident pass exceeds the free device memory and the windowed pass fits
 * (rvn_stage1_footprint), else resident. Results are identical in every
 * mode; a windowed pass takes max_overlaps <= 65536 and leaves phase
 * "stage1_window" in rvn_get_timings); "stage1_window_budget" (bytes: replaces the
 * free device memory in the auto decision, 0 = the free memory); "stage1_stream" (0/1,
 * default 1: a resident rvn_find_overlaps_and_create_piles copies the piles and lists of
 * the reads no later flush touches to the host on a stream of its own while the later
 * flushes run, lists only at max_overlaps <= 256 and up to 8 GiB of them (the pinned
 * buffer is sized for max_overlaps records per read); with 0 all of them follow the last
 * flush. Either way the call returns with every result on the host, the same results,
 * and phase "results" in rvn_get_timings is the copying that no kernel hides);
 * "index_chunk_bases"
 * (how rvn_find_overlaps_and_create_piles and rvn_minimize build an index batch: 0 = in one piece,
 * with a sketch of the whole batch; N > 0 = in chunks of reads of >= N bases, cut like
 * the index batches: each chunk is sketched twice, once for its micromizer thresholds and
 * once for its records, which go straight into the index's tiers, and the build's buffers
 * are freed before the first flush; -1 = auto, the default: chunks of 2^30 bases only
 * when the one-shot pass fits neither resident nor windowed (rvn_minimize: when its
 * one-shot estimate, rvn_minimize_footprint, exceeds the memory), else one piece. Results
 * are identical in every mode; a chunked call leaves phase "sketch_tiers" in
 * rvn_get_timings; with "async_upload" a chunked build first waits for the whole
 * upload); "index_chunk_budget" (bytes: replaces the free device memory in that auto
 * decision, 0 = the free memory); "map_flush_bases" (rvn_map cuts its range into flushes of
 * >= N query bases; 0 = the default, from the device memory; for tests of the flush
 * path, results do not depend on it); "fastx_chunk_bytes" (text bytes rvn_reads_upload_files
 * parses per chunk; 0 = the default, 256 MiB; results do not depend on it); "stage2_batch_bases" (rvn_find_overlaps_and_repetitive_
 * regions cuts its index batches at >= N bases instead of the reference's 1U << 30; 0 = the
 * reference's cut; for tests of the multi-batch path: it changes what the reference's
 * schedule would compute at that cut); "poa_wide" and "poa_scratch_budget" (rvn_poa_batch and
 * rvn_polish_windows); "poa_batch_bytes" (rvn_polish_windows: the device inputs of one window
 * batch, 0 = the default, from the free device memory; results do not depend on it);
 * "radix_portion_tiles" (a radix sort or partition over more than about 2^30 records
 * runs in portions, the last tile of each handing the running bin ends to the next;
 * N > 0 cuts portions of N tiles - 8192 records for u32 keys, 4096 for u64 keys -
 * or of as few more as keep the launches of a sort within 64; 0 = the default, the
 * longest portion; for tests of the portion path, results do not depend on it);
 * "reset_stats".
 * Unknown name or value out of range -> RVN_ERR_INVALID. */
int rvn_set_option(rvn_ctx* ctx, const char* name, int64_t value);

/* Device time (ms, CUDA events on the context's stream) of the phases of the
 * last stage-1 / minimize / map call: names[] are static strings. */
int rvn_get_timings(rvn_ctx* ctx, const char* const** names,
                    const float** ms, uint32_t* n);

/* ---- multi-GPU building blocks -------------------------------------------
 * One context per rank (one process per GPU); the collectives between the
 * steps are the caller's (raven_b200/distributed.py: torch.distributed over
 * NCCL). With n_parts ranks: index keys are owned by value mod n_parts; a read
 * (as a query, and its pile and overlap list) by id mod n_parts; sketching is
 * split by any contiguous read ranges, ascending with the rank.
 * Every d_* pointer is DEVICE memory, owned by the context (outputs: valid
 * until the next call on it) or by the caller (inputs). Per index batch of
 * raven::FindOverlapsAndCreatePiles (RavenLib/src/construct.cc:36-112):
 *   sketch_split -> all-to-all -> index -> histogram -> all-reduce ->
 *   set_occurrence -> hits_split -> all-to-all -> chain -> overlaps_split ->
 *   all-to-all -> stage1_add; then stage1_end and rvn_dist_stage1_results
 *   (the piles and overlap lists of the reads this rank owns).
 * "runs": an all-to-all delivers one run per source rank; run_off (host,
 * n_runs + 1 entries) are their offsets in the received array. */
int rvn_dist_sketch_split(rvn_ctx* ctx, uint32_t first, uint32_t last, int minhash,
                          uint32_t n_parts, const uint64_t** d_value,
                          const uint64_t** d_origin, uint64_t* counts);
int rvn_dist_index(rvn_ctx* ctx, const uint64_t* d_value, const uint64_t* d_origin,
                   uint64_t n_records, uint64_t index_bases);
/* The same with the tiers of stage 1 (index.cu): records whose value exceeds
 * value_limit - the largest micromizer value of ANY read that can query this batch,
 * i.e. the maximum over the ranks of rvn_dist_max_threshold - are only counted for
 * the occurrence threshold. ~0: no tiers. */
int rvn_dist_index_limited(rvn_ctx* ctx, const uint64_t* d_value, const uint64_t* d_origin,
                           uint64_t n_records, uint64_t index_bases, uint64_t value_limit);
/* Largest micromizer value of the reads [first, last) this rank sketches (0 if empty). */
int rvn_dist_max_threshold(rvn_ctx* ctx, uint32_t first, uint32_t last, uint64_t* value);
/* run-length histogram of this rank's keys (u64 bins; bin i = keys with i
 * postings, last bin = longer runs) */
int rvn_dist_histogram(rvn_ctx* ctx, const uint64_t** d_hist, uint32_t* n_bins,
                       uint64_t* n_keys);
/* MinimizerEngine::Filter on the summed (host) histogram: one global threshold */
int rvn_dist_set_occurrence(rvn_ctx* ctx, const uint64_t* hist, uint64_t n_keys,
                            double frequency, uint32_t* occurrence);
/* seed hits of the received query records (sorted by read id; reads
 * [0, n_query_reads)) against this rank's keys, written as n_parts runs by the
 * owner of the query read; d_lhs = query read of every hit */
int rvn_dist_hits_split(rvn_ctx* ctx, const uint64_t* d_qvalue,
                        const uint64_t* d_qorigin, uint64_t n_queries,
                        int avoid_equal, int avoid_symmetric, uint32_t n_parts,
                        uint32_t n_query_reads, const uint64_t** d_group,
                        const uint64_t** d_positions, const uint32_t** d_lhs,
                        uint64_t* counts);
/* chains the hits of the owned reads below n_query_reads (runs sorted by query
 * read): overlaps in query order */
int rvn_dist_chain(rvn_ctx* ctx, const uint64_t* d_group, const uint64_t* d_positions,
                   const uint32_t* d_lhs, uint64_t n_hits, uint32_t n_runs,
                   const uint64_t* run_off, uint32_t n_parts, uint32_t rank,
                   uint32_t n_query_reads, const rvn_overlap** d_overlaps,
                   uint64_t* n_overlaps);
/* the overlaps of the last rvn_dist_chain as n_parts runs: run d != rank holds
 * those whose rhs read rank d owns, run `rank` holds all of them */
int rvn_dist_overlaps_split(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank,
                            const rvn_overlap** d_overlaps, uint64_t* counts);
/* piles + per-read overlap lists of the owned reads: begin once, add once per
 * index batch (runs sorted by query read; reference flush schedule), end */
int rvn_dist_stage1_begin(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank);
int rvn_dist_stage1_add(rvn_ctx* ctx, const rvn_overlap* d_overlaps,
                        uint64_t n_overlaps, uint32_t n_runs, const uint64_t* run_off,
                        uint32_t n_query_reads, uint64_t max_overlaps,
                        uint64_t query_batch_bases);
int rvn_dist_stage1_end(rvn_ctx* ctx);
/* owned read j is read rank + j * n_parts; arrays as rvn_stage1_results, over
 * the n_owned owned reads; n_mapped = overlaps found by this rank's queries */
int rvn_dist_stage1_results(rvn_ctx* ctx, const rvn_overlap** overlaps,
                            const uint64_t** overlap_off, const uint16_t** pile,
                            const uint64_t** pile_off, uint32_t* n_owned,
                            uint64_t* n_mapped);

/* ---- peer-memory exchange: the all-to-alls of the schedule as direct DMA
 * writes into the destination rank's receive arena over NVLink (CUDA IPC; one
 * process per GPU on one node). export: (re)allocate this rank's arena, 64-byte
 * handle out; import: map the peers' arenas from all n_parts handles (own slot
 * ignored); put: asynchronous copy of device memory into rank dest's arena at
 * dst_offset; put_flush: wait for this rank's puts. All arenas must have the
 * same size (the caller checks offsets against it); the caller brackets a
 * round of puts with barriers and closes the peers before any re-export. */
int rvn_dist_arena_export(rvn_ctx* ctx, uint64_t bytes, void* handle64);
int rvn_dist_arena_import(rvn_ctx* ctx, uint32_t n_parts, uint32_t rank,
                          const void* handles);
int rvn_dist_arena_close_peers(rvn_ctx* ctx);
int rvn_dist_arena(rvn_ctx* ctx, void** d_arena, uint64_t* bytes);
int rvn_dist_put(rvn_ctx* ctx, uint32_t dest, uint64_t dst_offset, const void* d_src,
                 uint64_t bytes);
int rvn_dist_put_flush(rvn_ctx* ctx);

#ifdef __cplusplus
}
#endif

#endif /* RAVEN_B200_H_ */
