// Seeded temperature / top-k / top-p sampling beside the greedy ArgmaxSampler: the id is drawn on the device by
// the rule of kllm_sample_top_p_f32 (DESIGN.md "Sampling"), a pure function of the logits, the settings of a
// DrawConfig and the position.  Temperature 0 is the greedy argmax.  Before each sample() the caller sets the
// position of the logits and, when step 0 is on, the ids fed at positions 0 .. pos, from which sample() cuts the
// windows of sampling.cuh: H(pos), the last last_n of them (all for last_n 0), and C(pos), those at [from_pos, pos].
// With a repetition penalty other than 1, sample() first runs kllm_repetition_penalty_f32 over H(pos) (DESIGN.md
// 5.7); with a frequency or presence penalty or a logit bias, kllm_logit_penalties_f32 over H(pos) and C(pos)
// instead (DESIGN.md 5.9).  It draws from the adjusted logits.
#ifndef KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
#define KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

#include "sampler/argmax_sampler.h"
#include "sampler/draw_config.h"

namespace sampler {
class SeededSampler final : public Sampler {
 public:
  SeededSampler(base::DeviceType device_type, DrawConfig cfg) : Sampler(device_type), cfg_(std::move(cfg)) {}
  // fed[i]: the id fed at position i (ids outside the vocabulary are ignored); only fed[0 .. pos] are read
  void set_position(int32_t pos, const std::vector<int32_t>& fed = {}) {
    pos_ = pos;
    fed_.assign(fed.begin(), fed.begin() + std::min(fed.size(), static_cast<size_t>(pos) + 1));
  }
  size_t sample(const float* logits, size_t size, void* stream) override;

 private:
  const DrawConfig cfg_;
  int32_t pos_ = 0;
  std::vector<int32_t> fed_;
};
}  // namespace sampler
#endif  // KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
