// raven-b200: drop-in `racon/polisher.hpp`.
//
// The reference includes this header from the un-vendored `racon` library
// (RavenLib/src/polish.cc:4) and uses exactly two members:
//   racon::Polisher::Create(thread_pool, q, e, w, trim, m, n, g,
//       cuda_poa_batches, cuda_banded_alignment, cuda_alignment_batches)
//                                                   RavenLib/src/polish.cc:43-48
//   polisher->Polish(targets, sequences, drop_unpolished)   polish.cc:51
// This class keeps those signatures. Mapping (ram) and the window consensus
// (POA) run on the GPU through the C ABI (rvn_minimize / rvn_map /
// rvn_align_breaking_points / rvn_polish_windows): the alignment paths, the window
// cuts, racon's layer rules and the window layers are built on the device. The cuda_* arguments of the
// reference select NVIDIA's cudapoa/cudaaligner inside upstream racon; here the
// GPU path is always on and they are accepted and ignored.
#ifndef RACON_POLISHER_HPP_
#define RACON_POLISHER_HPP_

#include <cstdint>
#include <memory>
#include <vector>

#include "biosoup/nucleic_acid.hpp"
#include "thread_pool/thread_pool.hpp"

struct rvn_ctx;

namespace racon {

class Polisher {
 public:
  ~Polisher();

  static std::unique_ptr<Polisher> Create(
      std::shared_ptr<thread_pool::ThreadPool> thread_pool = nullptr,
      double quality_threshold = 10.0, double error_threshold = 0.3,
      std::uint32_t window_len = 500, bool trim_consensus = true,
      std::int8_t match = 3, std::int8_t mismatch = -5, std::int8_t gap = -4,
      std::uint32_t cuda_poa_batches = 0, bool cuda_banded_alignment = false,
      std::uint32_t cuda_alignment_batches = 0);

  std::vector<std::unique_ptr<biosoup::NucleicAcid>> Polish(
      const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& targets,
      const std::vector<std::unique_ptr<biosoup::NucleicAcid>>& sequences,
      bool drop_unpolished_sequences);

  // counters of the last Polish() (POA windows/s accounting)
  std::uint64_t num_windows() const { return num_windows_; }
  std::uint64_t num_polished_windows() const { return num_polished_windows_; }
  // windows that ran on the wide (32-bit) consensus kernel: deeper than the 16-bit
  // kernels take (option "poa_wide" of include/raven_b200.h)
  std::uint64_t num_wide_windows() const { return num_wide_windows_; }
  // batches of windows the consensus ran in (option "poa_batch_bytes")
  std::uint64_t num_window_batches() const { return num_window_batches_; }
  // the layer rules, the packing and the consensus (rvn_polish_windows)
  double poa_seconds() const { return poa_seconds_; }
  // map (GPU), alignment paths + window cuts (GPU), window packing (GPU), consensus
  // (GPU), stitch, layer rules (GPU)
  const double* phase_seconds() const { return phase_seconds_; }

 private:
  Polisher(std::shared_ptr<thread_pool::ThreadPool> thread_pool, double q, double e,
           std::uint32_t w, bool trim, std::int8_t m, std::int8_t n, std::int8_t g);

  std::shared_ptr<thread_pool::ThreadPool> thread_pool_;
  double q_, e_;
  std::uint32_t w_;
  bool trim_;
  std::int8_t m_, n_, g_;
  rvn_ctx* ctx_;
  std::uint64_t num_windows_ = 0, num_polished_windows_ = 0, num_wide_windows_ = 0;
  std::uint64_t num_window_batches_ = 0;
  double poa_seconds_ = 0;
  double phase_seconds_[6] = {0, 0, 0, 0, 0, 0};
};

}  // namespace racon

#endif  // RACON_POLISHER_HPP_
