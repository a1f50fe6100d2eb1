// Seeded temperature / top-k / top-p sampling beside the greedy ArgmaxSampler: the id is drawn on the device by
// the rule of kllm_sample_top_p_f32 (DESIGN.md "Sampling"), a pure function of the logits, the settings and the
// position.  top_p 1 (the default) is kllm_sample_f32's rule.  The model sets the position of the logits before
// each sample() (post_processing).  With a repetition penalty other than 1, sample() first runs
// kllm_repetition_penalty_f32 over the ids of set_history() (the window of fed ids, DESIGN.md 5.7) and draws from
// the penalised logits.
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
  size_t sample(const float* logits, size_t size, void* stream) override;

 private:
  float temperature_;
  int32_t top_k_;
  uint64_t seed_;
  float top_p_;
  float penalty_;
  std::vector<int32_t> history_;
  int32_t pos_ = 0;
};
}  // namespace sampler
#endif  // KLLM_KUIPER_SAMPLER_SEEDED_SAMPLER_H_
