#include "sampler/draw_config.h"

#include <kllm_b200.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <string>

namespace sampler {
namespace {
float env_float(const char* name, float unset) {
  const char* v = std::getenv(name);
  return v != nullptr ? std::strtof(v, nullptr) : unset;
}

int32_t env_int(const char* name) {
  const char* v = std::getenv(name);
  return v != nullptr ? static_cast<int32_t>(std::strtol(v, nullptr, 10)) : 0;
}
}  // namespace

void fill_from_env(DrawConfig& cfg, const DrawGroups& set) {
  if (!set.sampling) {
    const char* seed = std::getenv("KUIPER_SEED");
    cfg.temperature = env_float("KUIPER_TEMPERATURE", 0.f);
    cfg.top_k = env_int("KUIPER_TOP_K");
    cfg.seed = seed != nullptr ? std::strtoull(seed, nullptr, 10) : 0;
  }
  if (!set.top_p) cfg.top_p = env_float("KUIPER_TOP_P", 1.f);
  if (!set.penalty) {
    cfg.penalty = env_float("KUIPER_REPETITION_PENALTY", 1.f);
    cfg.last_n = env_int("KUIPER_REPEAT_LAST_N");
  }
  if (!set.frequency_presence) {
    cfg.frequency = env_float("KUIPER_FREQUENCY_PENALTY", 0.f);
    cfg.presence = env_float("KUIPER_PRESENCE_PENALTY", 0.f);
    cfg.from_pos = 0;
  }
}

base::Status validate(const DrawConfig& cfg) {
  using base::error::InvalidArgument;
  if (!std::isfinite(cfg.temperature) || cfg.temperature < 0.f)
    return InvalidArgument("sampling: the temperature must be finite and >= 0 (KUIPER_TEMPERATURE / set_sampling)");
  if (!(cfg.top_p > 0.f && cfg.top_p <= 1.f))
    return InvalidArgument("sampling: top_p must be in (0, 1] (KUIPER_TOP_P / set_top_p)");
  if (!std::isfinite(cfg.penalty) || !(cfg.penalty > 0.f) || cfg.last_n < 0)
    return InvalidArgument(
        "sampling: repetition_penalty must be finite and > 0, and its last_n >= 0 (KUIPER_REPETITION_PENALTY / "
        "KUIPER_REPEAT_LAST_N / set_repetition_penalty)");
  if (!std::isfinite(cfg.frequency) || !std::isfinite(cfg.presence) || cfg.from_pos < 0)
    return InvalidArgument(
        "sampling: frequency and presence penalties must be finite, and from_pos >= 0 (KUIPER_FREQUENCY_PENALTY / "
        "KUIPER_PRESENCE_PENALTY / set_frequency_presence)");
  std::vector<int32_t> ids;
  for (const auto& [id, b] : cfg.logit_bias) {
    if (id < 0 || !std::isfinite(b))
      return InvalidArgument("sampling: a logit bias needs ids >= 0 and finite values (set_logit_bias)");
    ids.push_back(id);
  }
  std::sort(ids.begin(), ids.end());
  if (std::adjacent_find(ids.begin(), ids.end()) != ids.end())
    return InvalidArgument("sampling: a logit bias lists an id twice (set_logit_bias)");
  if (cfg.logprobs_top_n < -1 || cfg.logprobs_top_n > KLLM_MAX_TOP_LOGPROBS)
    return InvalidArgument("logprobs: top_n must be in [-1, 20] (set_logprobs)");
  return base::error::Success();
}

base::Status apply_to_decoder(const DrawConfig& cfg, kllm_decoder* dec) {
  auto failed = [](const char* call, int rc) {
    return base::error::InternalError(std::string(call) + " failed: " + kllm_error_string(rc));
  };
  if (cfg.temperature > 0.f) {
    if (const int rc = kllm_decoder_set_sampling_top_p(dec, cfg.temperature, cfg.top_k, cfg.top_p, cfg.seed); rc != 0)
      return failed("kllm_decoder_set_sampling_top_p", rc);
    LOG(INFO) << "sampling: temperature " << cfg.temperature << ", top_k " << cfg.top_k << ", top_p " << cfg.top_p
              << ", seed " << cfg.seed;
  }
  if (cfg.penalty != 1.f) {
    if (const int rc = kllm_decoder_set_repetition_penalty(dec, cfg.penalty, cfg.last_n); rc != 0)
      return failed("kllm_decoder_set_repetition_penalty", rc);
    LOG(INFO) << "sampling: repetition_penalty " << cfg.penalty << ", last_n " << cfg.last_n;
  }
  if (cfg.frequency != 0.f || cfg.presence != 0.f) {
    if (const int rc = kllm_decoder_set_frequency_presence(dec, cfg.frequency, cfg.presence, cfg.from_pos); rc != 0)
      return failed("kllm_decoder_set_frequency_presence", rc);
    LOG(INFO) << "sampling: frequency_penalty " << cfg.frequency << ", presence_penalty " << cfg.presence
              << ", from_pos " << cfg.from_pos;
  }
  if (!cfg.logit_bias.empty()) {
    std::vector<int32_t> ids;
    std::vector<float> vals;
    for (const auto& [id, b] : cfg.logit_bias) ids.push_back(id), vals.push_back(b);
    if (const int rc = kllm_decoder_set_logit_bias(dec, ids.data(), vals.data(), static_cast<int32_t>(ids.size()));
        rc != 0)
      return base::error::InvalidArgument(std::string("sampling: kllm_decoder_set_logit_bias refused the map (an id "
                                                       "outside the vocabulary?): ") + kllm_error_string(rc));
    LOG(INFO) << "sampling: logit_bias of " << ids.size() << " id(s)";
  }
  if (cfg.logprobs_top_n >= 0) {
    if (const int rc = kllm_decoder_set_logprobs(dec, cfg.logprobs_top_n); rc != 0)
      return failed("kllm_decoder_set_logprobs", rc);
    LOG(INFO) << "logprobs: top_n " << cfg.logprobs_top_n;
  }
  return base::error::Success();
}
}  // namespace sampler
