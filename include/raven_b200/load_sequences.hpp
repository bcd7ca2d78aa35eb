// raven-b200: the reads of raven's input loop (RavenExe/src/main.cc:258-299) parsed and packed
// on the GPU (rvn_reads_upload_files). Needs only biosoup and the C ABI, so a program that
// does not build RavenLib may include it alone; construct_b200.hpp includes it.
#ifndef RAVEN_B200_LOAD_SEQUENCES_HPP_
#define RAVEN_B200_LOAD_SEQUENCES_HPP_

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "biosoup/nucleic_acid.hpp"
#include "raven_b200.h"

namespace raven_b200 {

// main.cc's loop over raven::CreateParser(path)->Parse(-1) for every path in order (empty
// files skipped): the same biosoup::NucleicAcid objects field for field, ids taken from
// NucleicAcid::num_objects in order. Throws std::invalid_argument with the message the
// loop prints for the first failing record. Runs on a short-lived context of its own on
// `device`, so no engine's context changes.
inline std::vector<std::unique_ptr<biosoup::NucleicAcid>> LoadSequences(
    const std::vector<std::string>& paths, int device = 0) {
  rvn_ctx* ctx = nullptr;
  if (rvn_ctx_create(device, nullptr, &ctx) != RVN_OK) {
    throw std::runtime_error("[raven_b200::LoadSequences] error: no usable sm_90 device");
  }
  struct Close {
    rvn_ctx* c;
    ~Close() { rvn_ctx_destroy(c); }
  } close{ctx};
  auto check = [&](int rc) {
    if (rc == RVN_ERR_INVALID) throw std::invalid_argument(rvn_last_error(ctx));
    if (rc != RVN_OK) throw std::runtime_error(rvn_last_error(ctx));
  };
  std::vector<const char*> p;
  for (const auto& it : paths) p.push_back(it.c_str());
  std::uint64_t sizes[4] = {0, 0, 0, 0};
  check(rvn_set_option(ctx, "host_bases", 0));  // (the words only come back)
  check(rvn_reads_upload_files(ctx, p.data(), static_cast<std::uint32_t>(p.size()), sizes));
  std::vector<std::uint64_t> words(sizes[1]), word_off(sizes[0] + 1), bq_off(sizes[0] + 1),
      name_off(sizes[0] + 1);
  std::vector<std::uint32_t> lens(sizes[0]);
  std::vector<std::uint8_t> bq(sizes[2]);
  std::string names(sizes[3], '\0');
  check(rvn_reads_parsed(ctx, words.data(), word_off.data(), lens.data(), bq.data(),
                         bq_off.data(), &names[0], name_off.data()));
  std::vector<std::unique_ptr<biosoup::NucleicAcid>> dst;
  dst.reserve(sizes[0]);
  for (std::uint64_t i = 0; i < sizes[0]; ++i) {
    std::unique_ptr<biosoup::NucleicAcid> s(new biosoup::NucleicAcid());
    s->id = biosoup::NucleicAcid::num_objects++;
    s->name = names.substr(name_off[i], name_off[i + 1] - name_off[i]);
    s->deflated_data.assign(words.begin() + word_off[i], words.begin() + word_off[i + 1]);
    s->block_quality.assign(bq.begin() + bq_off[i], bq.begin() + bq_off[i + 1]);
    s->inflated_len = lens[i];
    s->is_reverse_complement = false;
    dst.emplace_back(std::move(s));
  }
  return dst;
}

}  // namespace raven_b200

#endif  // RAVEN_B200_LOAD_SEQUENCES_HPP_
