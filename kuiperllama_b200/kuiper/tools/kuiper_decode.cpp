// kuiper_decode: drive model::LLama2Model / Qwen2Model with raw token ids, the way demo/main.cpp
// drives it with text (embedding -> fill_input -> predict per position).
//
//   kuiper_decode <checkpoint> <llama|qwen> <fp32|int8> <n_steps> <id0> [id1 ...]
//                 [--layers] [--copy-at K] [--logits out.f32] [--sampling T K SEED] [--top-p P]
//                 [--repetition-penalty P N] [--frequency-presence F P [FROM]] [--logit-bias ID:B,...]
//                 [--generate N [--stop ID]... [--then K]] [--logprobs N] [--score] [--kv-cache fp32|bf16]
//
// --generate N runs the prompt and LLama2Model::generate() for at most N ids instead (n_steps is then unused),
// stopping at the tokenizer's stop ids and every --stop ID, and prints the ids generate() returned, followed
// by the ids of K more predict() steps on the same sequence with --then K.
//
// ids are the prompt; after the prompt the model free-runs (greedily, or by the model's sampling
// settings: KUIPER_TEMPERATURE / KUIPER_TOP_K / KUIPER_TOP_P / KUIPER_SEED) until n_steps positions have been processed.  Prints the id chosen at every position (-1 for prompt steps before the
// last prompt token) on one line.  --layers uses Model::forward (layer-by-layer op registry path)
// instead of predict's fused decoder.  --copy-at K hands predict() a COPY of the embedding row at
// position K (so that step cannot be recognised and runs layer by layer in the middle of a sequence
// the fused decoder started).  --logits writes the last position's logits as raw fp32.  --sampling calls
// LLama2Model::set_sampling(T, K, SEED) before init() instead of leaving it to the environment, and --top-p
// LLama2Model::set_top_p(P) instead of KUIPER_TOP_P.  --repetition-penalty P N calls
// LLama2Model::set_repetition_penalty(P, N) instead of KUIPER_REPETITION_PENALTY / KUIPER_REPEAT_LAST_N; --layers
// applies the penalty itself, over the ids this tool fed, to the seeded draw and to its greedy argmax.
// --frequency-presence F P [FROM] calls LLama2Model::set_frequency_presence(F, P, FROM) (FROM, 0 when absent, is
// taken when the next argument is an integer: give the prompt ids first) and --logit-bias ID:B,...
// LLama2Model::set_logit_bias; with either on, --layers draws through SeededSampler (kllm_logit_penalties_f32 over
// the ids this tool fed), greedily at temperature 0.
// --logprobs N calls LLama2Model::set_logprobs(N) and, after the ids, prints one line per position that has a record
// entry: "lp <pos> <id> <lp>" followed by N pairs "<top id> <top lp>" (%.9g: the fp32 values round-trip).
// --score scores the given ids with LLama2Model::score() instead of decoding (n_steps is then unused): one line of
// the n - 1 log-probabilities, then "perplexity <exp(-mean)>".  The layer path has neither: --layers with either is
// refused.  --kv-cache bf16 calls LLama2Model::set_bf16_kv_cache(true) instead of leaving it to KUIPER_KV_CACHE (the
// fused decoder's bf16 KV cache needs KUIPER_NUMERICS=fast); --kv-cache fp32 turns it off.
#include <base/base.h>
#include <cuda_runtime_api.h>
#include <glog/logging.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "model/llama3.h"
#include "model/qwen2.h"

int main(int argc, char** argv) {
  if (argc < 6) {
    std::fprintf(stderr, "usage: %s <checkpoint> <llama|qwen> <fp32|int8> <n_steps> <id0> [id1 ...] "
                         "[--layers] [--copy-at K] [--logits out.f32] [--sampling T K SEED] [--top-p P] "
                         "[--repetition-penalty P N] [--frequency-presence F P [FROM]] [--logit-bias ID:B,...] "
                         "[--generate N [--stop ID]... [--then K]] [--kv-cache fp32|bf16]\n", argv[0]);
    return 2;
  }
  const std::string checkpoint = argv[1], family = argv[2], prec = argv[3];
  const int n_steps = std::atoi(argv[4]);
  std::vector<int> prompt;
  bool layers = false;
  int copy_at = -1;
  std::string logits_path;
  bool set_sampling = false;
  float temperature = 0.f;
  int32_t top_k = 0;
  uint64_t seed = 0;
  bool set_top_p = false;
  float top_p = 1.f;
  bool set_penalty = false;
  float penalty = 1.f;
  int32_t last_n = 0;
  bool set_fp = false;
  float frequency = 0.f, presence = 0.f;
  int32_t count_from = 0;
  std::vector<std::pair<int32_t, float>> logit_bias;
  int generate = 0, then = 0;
  std::vector<int32_t> stops;
  int32_t logprobs = -1;
  bool set_logprobs = false, score = false;
  int kv_cache = -1;  // -1: KUIPER_KV_CACHE decides, 0: fp32, 1: bf16
  for (int i = 5; i < argc; ++i) {
    if (!std::strcmp(argv[i], "--layers")) layers = true;
    else if (!std::strcmp(argv[i], "--sampling") && i + 3 < argc) {
      set_sampling = true;
      temperature = std::strtof(argv[++i], nullptr);
      top_k = static_cast<int32_t>(std::strtol(argv[++i], nullptr, 10));
      seed = std::strtoull(argv[++i], nullptr, 10);
    }
    else if (!std::strcmp(argv[i], "--top-p") && i + 1 < argc) {
      set_top_p = true;
      top_p = std::strtof(argv[++i], nullptr);
    }
    else if (!std::strcmp(argv[i], "--repetition-penalty") && i + 2 < argc) {
      set_penalty = true;
      penalty = std::strtof(argv[++i], nullptr);
      last_n = static_cast<int32_t>(std::strtol(argv[++i], nullptr, 10));
    }
    else if (!std::strcmp(argv[i], "--frequency-presence") && i + 2 < argc) {
      set_fp = true;
      frequency = std::strtof(argv[++i], nullptr);
      presence = std::strtof(argv[++i], nullptr);
      char* end = nullptr;
      if (i + 1 < argc) {
        const long from = std::strtol(argv[i + 1], &end, 10);
        if (end != argv[i + 1] && *end == '\0') {
          count_from = static_cast<int32_t>(from);
          ++i;
        }
      }
    }
    else if (!std::strcmp(argv[i], "--logit-bias") && i + 1 < argc) {
      for (char* tok = std::strtok(argv[++i], ","); tok != nullptr; tok = std::strtok(nullptr, ",")) {
        char* colon = std::strchr(tok, ':');
        if (colon == nullptr) return 2;
        logit_bias.emplace_back(static_cast<int32_t>(std::strtol(tok, nullptr, 10)), std::strtof(colon + 1, nullptr));
      }
    }
    else if (!std::strcmp(argv[i], "--generate") && i + 1 < argc) generate = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--stop") && i + 1 < argc) stops.push_back(std::atoi(argv[++i]));
    else if (!std::strcmp(argv[i], "--then") && i + 1 < argc) then = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--copy-at") && i + 1 < argc) copy_at = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--logprobs") && i + 1 < argc) {
      set_logprobs = true;
      logprobs = std::atoi(argv[++i]);
    }
    else if (!std::strcmp(argv[i], "--score")) score = true;
    else if (!std::strcmp(argv[i], "--kv-cache") && i + 1 < argc) {
      const std::string v = argv[++i];
      if (v != "fp32" && v != "bf16") return 2;
      kv_cache = v == "bf16" ? 1 : 0;
    }
    else if (!std::strcmp(argv[i], "--logits") && i + 1 < argc) logits_path = argv[++i];
    else prompt.push_back(std::atoi(argv[i]));
  }
  if (prompt.empty() || n_steps <= 0) return 2;
  if (layers && (set_logprobs || score)) {
    std::fprintf(stderr, "--layers has no log-probabilities: --logprobs and --score need the fused decoder\n");
    return 2;
  }
  const bool quant = prec == "int8";

  std::unique_ptr<model::LLama2Model> m;
  if (family == "qwen") {
    m = std::make_unique<model::Qwen2Model>(base::TokenizerType::kEncodeBpe, "<none>", checkpoint, quant);
  } else {
    m = std::make_unique<model::LLama2Model>(base::TokenizerType::kEncodeSpe, "<none>", checkpoint, quant);
  }
  if (set_sampling) m->set_sampling(temperature, top_k, seed);
  if (set_top_p) m->set_top_p(top_p);
  if (set_penalty) m->set_repetition_penalty(penalty, last_n);
  if (set_fp) m->set_frequency_presence(frequency, presence, count_from);
  if (!logit_bias.empty()) m->set_logit_bias(logit_bias);
  if (!stops.empty()) m->set_stop_ids(stops);
  if (set_logprobs) m->set_logprobs(logprobs);  // init() refuses a value outside [-1, 20]
  if (kv_cache >= 0) m->set_bf16_kv_cache(kv_cache == 1);
  base::Status st = m->init(base::DeviceType::kDeviceCUDA);
  if (!st) {
    std::fprintf(stderr, "init failed: %s\n", st.get_err_msg().c_str());
    return 1;
  }
  std::fprintf(stderr, "engine: %s%s\n", m->decoder_engine(), layers ? " (unused: --layers)" : "");

  // the record entries of positions [0, n): one line each where there is one
  auto print_logprobs = [&](int32_t n) {
    if (logprobs < 0) return true;
    std::vector<int32_t> ids, top_ids;
    std::vector<float> lp, top_lp;
    base::Status s = m->logprobs(0, n, ids, lp, top_ids, top_lp);
    if (!s) {
      std::fprintf(stderr, "logprobs failed: %s\n", s.get_err_msg().c_str());
      return false;
    }
    const int32_t k = std::max(logprobs, 0);
    for (int32_t p = 0; p < n; ++p) {
      if (ids[p] < 0) continue;
      std::printf("lp %d %d %.9g", p, ids[p], lp[p]);
      for (int32_t r = 0; r < k; ++r) std::printf(" %d %.9g", top_ids[p * k + r], top_lp[p * k + r]);
      std::printf("\n");
    }
    return true;
  };
  if (score) {
    std::vector<float> lp;
    st = m->score(std::vector<int32_t>(prompt.begin(), prompt.end()), lp);
    if (!st) {
      std::fprintf(stderr, "score failed: %s\n", st.get_err_msg().c_str());
      return 1;
    }
    double sum = 0.0;
    for (size_t i = 0; i < lp.size(); ++i) {
      std::printf("%s%.9g", i ? " " : "", lp[i]);
      sum += lp[i];
    }
    std::printf("\nperplexity %.9g\n", std::exp(-sum / static_cast<double>(lp.size())));
    return print_logprobs(static_cast<int32_t>(prompt.size())) ? 0 : 1;
  }

  tensor::Tensor pos_tensor = m->get_buffer(model::ModelBufferType::kInputPos);
  if (generate > 0) {
    // LLama2Model::generate(), then --then more predict() steps on the same sequence
    std::vector<int32_t> ids, streamed;
    st = m->generate(std::vector<int32_t>(prompt.begin(), prompt.end()), generate, ids,
                     [&streamed](const int32_t* t, int32_t k) { streamed.insert(streamed.end(), t, t + k); });
    if (!st) {
      std::fprintf(stderr, "generate failed: %s\n", st.get_err_msg().c_str());
      return 1;
    }
    if (streamed != ids) {
      std::fprintf(stderr, "generate: the streamed ids differ from the returned ones\n");
      return 1;
    }
    int next = ids.back();
    for (int k = 0; k < then; ++k) {
      const int32_t pos = static_cast<int32_t>(prompt.size() + ids.size()) - 1;
      pos_tensor.index<int32_t>(0) = pos;
      auto emb = m->embedding({next});
      STATUS_CHECK(m->predict(m->fill_input(pos_tensor, emb, false), pos_tensor, false, next));
      ids.push_back(next);
    }
    for (size_t i = 0; i < ids.size(); ++i) std::printf("%s%d", i ? " " : "", ids[i]);
    std::printf("\n");
    return print_logprobs(static_cast<int32_t>(prompt.size() + ids.size())) ? 0 : 1;
  }
  const int32_t prompt_len = static_cast<int32_t>(prompt.size());
  auto prompt_embedding = m->embedding(prompt);
  // --layers draws with the model's settings too (the layer path's SeededSampler)
  std::unique_ptr<sampler::SeededSampler> seeded;
  if (m->sampling_temperature() > 0.f || m->sampling_step0_extras()) {
    seeded = std::make_unique<sampler::SeededSampler>(base::DeviceType::kDeviceCUDA, m->sampling_temperature(),
                                                      m->sampling_top_k(), m->sampling_seed(),
                                                      m->sampling_top_p(), m->sampling_repetition_penalty());
    seeded->set_penalties(m->sampling_frequency_penalty(), m->sampling_presence_penalty(), m->sampling_logit_bias());
  }
  std::vector<float> host_logits;
  int next = -1;
  std::vector<int> chosen;
  // --layers: the id fed at each position, and the penalty's window of them at `pos` (DESIGN.md 5.7)
  const float theta = m->sampling_repetition_penalty();
  const size_t vocab = m->get_buffer(model::ModelBufferType::kForwardOutput).size();
  std::vector<int32_t> fed(static_cast<size_t>(n_steps), -1);
  auto window = [&](int32_t pos) {
    const int32_t n = m->sampling_repeat_last_n();
    const int32_t lo = n == 0 ? 0 : std::max(0, pos - n + 1);
    return std::vector<int32_t>(fed.begin() + lo, fed.begin() + pos + 1);
  };
  auto run = [&](const tensor::Tensor& input, bool is_prompt) {
    if (!layers) {
      if (pos_tensor.index<int32_t>(0) == copy_at) {
        // the row is a view into the model's embedding buffer: copy it into storage of its own
        tensor::Tensor copy(base::DataType::kDataTypeFp32, static_cast<int32_t>(input.size()), true,
                            base::CUDADeviceAllocatorFactory::get_instance());
        CHECK(cudaMemcpy(copy.ptr<float>(), input.ptr<float>(), input.byte_size(), cudaMemcpyDeviceToDevice) ==
              cudaSuccess);
        STATUS_CHECK(m->predict(copy, pos_tensor, is_prompt, next));
      } else {
        STATUS_CHECK(m->predict(input, pos_tensor, is_prompt, next));
      }
      return;
    }
    STATUS_CHECK(m->forward(input, pos_tensor, next));
    next = -1;
    if (!is_prompt && seeded) {
      const tensor::Tensor& lg = m->get_buffer(model::ModelBufferType::kForwardOutput);
      seeded->set_position(pos_tensor.index<int32_t>(0));
      seeded->set_history(window(pos_tensor.index<int32_t>(0)));
      // step 0's count window [from_pos, pos] of the ids fed (DESIGN.md 5.9)
      const int32_t at = pos_tensor.index<int32_t>(0), from = std::min(m->sampling_count_from(), at + 1);
      seeded->set_counted(std::vector<int32_t>(fed.begin() + from, fed.begin() + at + 1));
      next = static_cast<int>(seeded->sample(lg.ptr<float>(), lg.size(), nullptr));
    } else if (!is_prompt) {  // greedy argmax, lowest index on ties (argmax_sampler.cpp)
      tensor::Tensor lg = m->get_buffer(model::ModelBufferType::kForwardOutput).clone();
      lg.to_cpu();
      float* p = lg.ptr<float>();
      if (theta != 1.f) {  // step 0b on the host: one fp32 multiply or divide per distinct id of the window
        std::vector<int32_t> ids = window(pos_tensor.index<int32_t>(0));
        std::sort(ids.begin(), ids.end());
        ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
        for (int32_t id : ids)
          if (id >= 0 && static_cast<size_t>(id) < lg.size()) p[id] = p[id] < 0.f ? p[id] * theta : p[id] / theta;
      }
      size_t best = 0;
      for (size_t i = 1; i < lg.size(); ++i)
        if (p[i] > p[best]) best = i;
      next = static_cast<int>(best);
    }
  };
  for (int32_t pos = 0; pos < n_steps; ++pos) {
    pos_tensor.index<int32_t>(0) = pos;
    const int32_t id = pos < prompt_len ? prompt[pos] : next;
    fed[pos] = id >= 0 && static_cast<size_t>(id) < vocab ? id : -1;
    if (pos < prompt_len - 1) {
      run(m->fill_input(pos_tensor, prompt_embedding, true), true);
    } else if (pos == prompt_len - 1) {
      // the last prompt token already samples (demo/main.cpp:19-24 treats it as a prompt row but
      // is_prompt=false from pos == prompt_len-1 on)
      tensor::Tensor row = m->fill_input(pos_tensor, prompt_embedding, true);
      run(row, false);
    } else {
      auto emb = m->embedding({next});
      run(m->fill_input(pos_tensor, emb, false), false);
    }
    chosen.push_back(next);
  }
  for (size_t i = 0; i < chosen.size(); ++i) std::printf("%s%d", i ? " " : "", chosen[i]);
  std::printf("\n");
  if (!print_logprobs(n_steps)) return 1;
  if (!logits_path.empty() && m->tensor_parallel().rank == 0) {  // under kuiper_tp_launch every rank holds the same logits
    tensor::Tensor lg = m->get_buffer(model::ModelBufferType::kForwardOutput).clone();
    lg.to_cpu();
    FILE* f = std::fopen(logits_path.c_str(), "wb");
    if (!f) return 1;
    std::fwrite(lg.ptr<float>(), sizeof(float), lg.size(), f);
    std::fclose(f);
  }
  return 0;
}
