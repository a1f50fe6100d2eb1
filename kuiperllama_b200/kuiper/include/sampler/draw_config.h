// sampler::DrawConfig -- every setting of how the C++ model draws an id (DESIGN.md "Sampling", 5.7 - 5.9), with
// where each comes from (fill_from_env), what is valid (validate) and how a fused decoder receives it
// (apply_to_decoder).  The defaults are the greedy argmax of the raw logits.
#ifndef KLLM_KUIPER_SAMPLER_DRAW_CONFIG_H_
#define KLLM_KUIPER_SAMPLER_DRAW_CONFIG_H_
#include <cstdint>
#include <utility>
#include <vector>

#include "base/base.h"

struct kllm_decoder;  // include/kllm_b200.h

namespace sampler {
struct DrawConfig {
  float temperature = 0.f;  // 0: greedy
  int32_t top_k = 0;
  uint64_t seed = 0;
  float top_p = 1.f;
  float penalty = 1.f;  // the repetition penalty over the ids fed at the last last_n positions (0: all)
  int32_t last_n = 0;
  float frequency = 0.f, presence = 0.f;  // over the ids fed at positions [from_pos, pos]
  int32_t from_pos = 0;
  std::vector<std::pair<int32_t, float>> logit_bias;
  int32_t logprobs_top_n = -1;  // -1: off

  // step 0 runs before the draw
  bool step0() const { return penalty != 1.f || step0_extras(); }
  // any of step 0's settings other than the repetition penalty is on
  bool step0_extras() const { return frequency != 0.f || presence != 0.f || !logit_bias.empty(); }
};

// The groups of settings a caller set explicitly; fill_from_env() leaves them alone.
struct DrawGroups {
  bool sampling = false;            // temperature, top_k, seed: KUIPER_TEMPERATURE / KUIPER_TOP_K / KUIPER_SEED
  bool top_p = false;               // KUIPER_TOP_P
  bool penalty = false;             // KUIPER_REPETITION_PENALTY / KUIPER_REPEAT_LAST_N
  bool frequency_presence = false;  // KUIPER_FREQUENCY_PENALTY / KUIPER_PRESENCE_PENALTY, from_pos 0
};

// Every group not in `set` from the environment (an unset variable is the default).
void fill_from_env(DrawConfig& cfg, const DrawGroups& set);
// InvalidArgument for the first setting out of range
base::Status validate(const DrawConfig& cfg);
// The settings that are on, through the kllm_decoder_set_* calls, each logged.
base::Status apply_to_decoder(const DrawConfig& cfg, kllm_decoder* dec);
}  // namespace sampler
#endif  // KLLM_KUIPER_SAMPLER_DRAW_CONFIG_H_
