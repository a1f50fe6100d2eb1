// Seeded temperature / top-k / top-p sampling beside the greedy ArgmaxSampler: the id is drawn on the device by
// the rule of kllm_sample_top_p_f32 (DESIGN.md "Sampling"), a pure function of the logits, the settings and the
// position.  top_p 1 (the default) is kllm_sample_f32's rule.  The model sets the position of the logits before
// each sample() (post_processing).  With a repetition penalty other than 1, sample() first runs
// kllm_repetition_penalty_f32 over the ids of set_history() (the window of fed ids, DESIGN.md 5.7) and draws from
// the penalised logits.  With a frequency or presence penalty or a logit bias (set_penalties), it runs
// kllm_logit_penalties_f32 instead, over set_history() and the ids of set_counted() (DESIGN.md 5.9).  Temperature 0
// is the greedy argmax of the adjusted logits.
#ifndef KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
#define KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
#include <cstdint>
#include <utility>
#include <vector>

#include "sampler/argmax_sampler.h"

namespace sampler {
class SeededSampler final : public Sampler {
 public:
  SeededSampler(base::DeviceType device_type, float temperature, int32_t top_k, uint64_t seed, float top_p = 1.f,
                float repetition_penalty = 1.f)
      : Sampler(device_type), temperature_(temperature), top_k_(top_k), seed_(seed), top_p_(top_p),
        penalty_(repetition_penalty) {}
  void set_position(int32_t pos) { pos_ = pos; }
  // the ids the penalty applies to at the next sample() (ids outside the vocabulary are ignored)
  void set_history(std::vector<int32_t> ids) { history_ = std::move(ids); }
  // step 0's frequency / presence penalties and logit bias, and the ids they count at the next sample()
  void set_penalties(float frequency, float presence, const std::vector<std::pair<int32_t, float>>& bias) {
    frequency_ = frequency, presence_ = presence;
    bias_ids_.clear(), bias_.clear();
    for (const auto& [id, b] : bias) bias_ids_.push_back(id), bias_.push_back(b);
  }
  void set_counted(std::vector<int32_t> ids) { counted_ = std::move(ids); }
  size_t sample(const float* logits, size_t size, void* stream) override;

 private:
  float temperature_;
  int32_t top_k_;
  uint64_t seed_;
  float top_p_;
  float penalty_;
  std::vector<int32_t> history_;
  float frequency_ = 0.f, presence_ = 0.f;
  std::vector<int32_t> bias_ids_;
  std::vector<float> bias_;
  std::vector<int32_t> counted_;
  int32_t pos_ = 0;
};
}  // namespace sampler
#endif  // KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
