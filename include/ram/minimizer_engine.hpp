// raven-b200: drop-in `ram/minimizer_engine.hpp`.
//
// The reference includes this header from the un-vendored `ram` library
// (RavenLib/include/raven/graph/construct.h:1) and uses
//   ram::MinimizerEngine{thread_pool, k, w}        construct.cc:661-662, assemble.cc:753
//   Minimize(first, last, minhash)                 construct.cc:42-43,363; assemble.cc:754,777
//   Filter(frequency)                              construct.cc:44,372; assemble.cc:755,778
//   Map(sequence, avoid_equal, avoid_symmetric, minhash, &filtered)
//                                                  construct.cc:62,377-381; assemble.cc:757,780
// This class keeps those signatures and forwards to the GPU engine through
// the C ABI (include/raven_b200.h). `Map` stays callable concurrently from pool
// workers like the reference's (a mutex serialises the device calls); the
// batched entry points below are the fast path our FindOverlapsAndCreatePiles
// replacement uses (include/raven_b200/construct_b200.hpp).
//
// A per-read Map result depends only on the index, the occurrence threshold,
// the engine parameters, the read and the flags. So the first Map of a read the
// device holds maps every read it holds in one batched call, and later Map
// calls with the same flags are served from those results on the host. A pass
// of index batches (each Minimize starting at the slot right after the last
// one's range, construct.cc:32-43) keeps the earlier batches' reads on the
// device, so they are served the same way.
#ifndef RAM_MINIMIZER_ENGINE_HPP_
#define RAM_MINIMIZER_ENGINE_HPP_

#include <cstdint>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "biosoup/nucleic_acid.hpp"
#include "biosoup/overlap.hpp"
#include "raven_b200.h"
#include "thread_pool/thread_pool.hpp"

namespace ram {

class MinimizerEngine {
 public:
  MinimizerEngine(std::shared_ptr<thread_pool::ThreadPool> thread_pool = nullptr,
                  std::uint32_t k = 15,  // element of [1, 31]
                  std::uint32_t w = 5,
                  std::uint32_t bandwidth = 500,
                  std::uint32_t chain = 4,
                  std::uint32_t matches = 100,
                  std::uint32_t gap = 10000);

  MinimizerEngine(const MinimizerEngine&) = delete;
  MinimizerEngine& operator=(const MinimizerEngine&) = delete;
  MinimizerEngine(MinimizerEngine&&) noexcept;
  MinimizerEngine& operator=(MinimizerEngine&&) noexcept;
  ~MinimizerEngine();

  // transform set of sequences to minimizer index
  // minhash = pick only the smallest sequence->data.size() / k minimizers
  void Minimize(
      std::vector<std::unique_ptr<biosoup::NucleicAcid>>::const_iterator first,
      std::vector<std::unique_ptr<biosoup::NucleicAcid>>::const_iterator last,
      bool minhash = false);

  // set occurrence frequency threshold (throws std::invalid_argument)
  void Filter(double frequency);

  // find overlaps in preconstructed minimizer index
  std::vector<biosoup::Overlap> Map(
      const std::unique_ptr<biosoup::NucleicAcid>& sequence,
      bool avoid_equal,      // ignore overlaps in which lhs_id == rhs_id
      bool avoid_symmetric,  // ignore overlaps in which lhs_id > rhs_id
      bool minhash = false,  // only lhs
      std::vector<std::uint32_t>* filtered = nullptr) const;

  // ---- GPU extensions ----
  // the whole read set on the device (ids must equal positions); lets stage 1
  // run without per-batch uploads
  void Upload(const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences);
  // any range, with its own ids (stage 2: the valid reads, sorted by id)
  void Upload(std::vector<std::unique_ptr<biosoup::NucleicAcid>>::const_iterator first,
              std::vector<std::unique_ptr<biosoup::NucleicAcid>>::const_iterator last);
  // (a caller that changes the index or the threshold through the context
  // follows with Minimize, Filter or Upload before the next Map)
  rvn_ctx* context() const { return ctx_; }
  std::mutex& mutex() const { return *mutex_; }
  std::uint32_t occurrence() const { return occurrence_; }

  // How Map calls were answered since construction.
  struct MapCounters {
    std::uint64_t batch_maps;   // device maps of a range of resident reads
    std::uint64_t served;       // Map calls answered from those results
    std::uint64_t single_maps;  // Map calls that mapped their read alone
  };
  MapCounters map_counters() const;

 private:
  using Iterator = std::vector<std::unique_ptr<biosoup::NucleicAcid>>::const_iterator;

  // The reads on the device, in order: the earlier index batches of the pass,
  // then the current one. The packed words are copies: callers may free or
  // change their reads (assemble.cc:758 resets them between Map calls).
  struct Resident {
    std::vector<std::uint64_t> words;
    std::vector<std::uint64_t> off{0};
    std::vector<std::uint32_t> lens, ids;
    std::vector<const biosoup::NucleicAcid*> objects;  // as uploaded
    std::unordered_map<std::uint32_t, std::uint32_t> position;  // id -> read
    std::uint32_t batch_first = 0;  // first read of the index batch
    // the slot after the last Minimize's range: a Minimize from there continues
    // the pass
    const std::unique_ptr<biosoup::NucleicAcid>* next = nullptr;
  };

  // Map results of every resident read for one set of flags.
  struct BatchResults {
    bool avoid_equal, avoid_symmetric, minhash, want_filtered;
    std::vector<rvn_overlap> overlaps;
    std::vector<std::uint64_t> overlap_off;
    std::vector<std::uint32_t> filtered;
    std::vector<std::uint64_t> filtered_off;
    std::vector<bool> served;
    std::uint32_t unserved;
  };

  void UploadRange(Iterator first, Iterator last);
  void Append(Resident& r, Iterator first, Iterator last);
  void UploadResident(const Resident& r);
  // position of `s` in the device set, or -1 when its words are not there
  std::int64_t ResidentPosition(const biosoup::NucleicAcid& s) const;
  BatchResults& Results(bool avoid_equal, bool avoid_symmetric, bool minhash,
                        bool want_filtered) const;

  rvn_ctx* ctx_;
  std::unique_ptr<std::mutex> mutex_;
  std::uint32_t occurrence_;
  Resident resident_;
  // results of the current index and threshold; cleared by Minimize, Filter
  // and Upload, and each set once all its reads have been served
  mutable std::vector<BatchResults> batches_;
  mutable MapCounters counters_;
  std::shared_ptr<thread_pool::ThreadPool> thread_pool_;
};

}  // namespace ram

#endif  // RAM_MINIMIZER_ENGINE_HPP_
