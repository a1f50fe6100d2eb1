// kuiper_decode: drive model::LLama2Model / Qwen2Model with raw token ids, the way demo/main.cpp
// drives it with text (embedding -> fill_input -> predict per position).
//
//   kuiper_decode <checkpoint> <llama|qwen> <fp32|int8> <n_steps> <id0> [id1 ...]
//                 [--layers] [--copy-at K] [--logits out.f32] [--sampling T K SEED] [--top-p P]
//                 [--repetition-penalty P N] [--frequency-presence F P [FROM]] [--logit-bias ID:B,...]
//                 [--generate N [--stop ID]... [--then K]] [--logprobs N] [--score] [--kv-cache fp32|bf16]
//                 [--weights fp32|bf16]
//
// --generate N runs the prompt and LLama2Model::generate() for at most N ids instead (n_steps is then unused),
// stopping at the tokenizer's stop ids and every --stop ID, and prints the ids generate() returned, followed
// by the ids of K more predict() steps on the same sequence with --then K.
//
// ids are the prompt; after the prompt the model free-runs (greedily, or by the model's draw settings, which the
// flags below set and the environment gives otherwise: sampler/draw_config.h) until n_steps positions have been
// processed.  Prints the id chosen at every position (-1 for prompt steps before the last prompt token) on one line.
// --layers uses Model::forward (layer-by-layer op registry path) instead of predict's fused decoder.  --copy-at K hands predict() a COPY of the embedding row at
// position K (so that step cannot be recognised and runs layer by layer in the middle of a sequence
// the fused decoder started).  --logits writes the last position's logits as raw fp32.  --sampling calls
// LLama2Model::set_sampling(T, K, SEED) before init() instead of leaving it to the environment, and --top-p
// LLama2Model::set_top_p(P).  --repetition-penalty P N calls LLama2Model::set_repetition_penalty(P, N).
// --frequency-presence F P [FROM] calls LLama2Model::set_frequency_presence(F, P, FROM) (FROM, 0 when absent, is
// taken when the next argument is an integer: give the prompt ids first) and --logit-bias ID:B,...
// LLama2Model::set_logit_bias.  --layers draws every id through a SeededSampler built from the model's settings,
// over the ids this tool fed (greedily at temperature 0).
// --logprobs N calls LLama2Model::set_logprobs(N) and, after the ids, prints one line per position that has a record
// entry: "lp <pos> <id> <lp>" followed by N pairs "<top id> <top lp>" (%.9g: the fp32 values round-trip).
// --score scores the given ids with LLama2Model::score() instead of decoding (n_steps is then unused): one line of
// the n - 1 log-probabilities, then "perplexity <exp(-mean)>".  The layer path has neither: --layers with either is
// refused.  --kv-cache bf16 calls LLama2Model::set_bf16_kv_cache(true) instead of leaving it to KUIPER_KV_CACHE (the
// fused decoder's bf16 KV cache needs KUIPER_NUMERICS=fast); --kv-cache fp8 calls set_fp8_kv_cache(true), unit scales
// (the same numerics); --kv-cache fp32 turns both off.  --weights bf16 / fp32 calls
// LLama2Model::set_bf16_weights instead of leaving it to KUIPER_WEIGHTS.  --speculative K calls
// LLama2Model::set_speculative(K) (0 off) instead of leaving it to KUIPER_SPECULATIVE: --generate then drafts by prompt
// lookup and verifies up to K drafts per pass, with the same ids.  After init() the tool reports on stderr the
// device memory init() took ("device bytes after init: N", from cudaMemGetInfo).
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
#include <utility>
#include <vector>

#include "model/llama3.h"
#include "model/qwen2.h"

int main(int argc, char** argv) {
  if (argc < 6) {
    std::fprintf(stderr, "usage: %s <checkpoint> <llama|qwen> <fp32|int8> <n_steps> <id0> [id1 ...] "
                         "[--layers] [--copy-at K] [--logits out.f32] [--sampling T K SEED] [--top-p P] "
                         "[--repetition-penalty P N] [--frequency-presence F P [FROM]] [--logit-bias ID:B,...] "
                         "[--generate N [--stop ID]... [--then K]] [--kv-cache fp32|bf16] [--weights fp32|bf16] [--speculative K]\n", argv[0]);
    return 2;
  }
  const std::string checkpoint = argv[1], family = argv[2], prec = argv[3];
  const int n_steps = std::atoi(argv[4]);
  const bool quant = prec == "int8";
  std::unique_ptr<model::LLama2Model> m;
  if (family == "qwen") {
    m = std::make_unique<model::Qwen2Model>(base::TokenizerType::kEncodeBpe, "<none>", checkpoint, quant);
  } else {
    m = std::make_unique<model::LLama2Model>(base::TokenizerType::kEncodeSpe, "<none>", checkpoint, quant);
  }
  std::vector<int> prompt;
  bool layers = false, score = false;
  int copy_at = -1;
  std::string logits_path;
  int generate = 0, then = 0;
  std::vector<int32_t> stops;
  for (int i = 5; i < argc; ++i) {
    if (!std::strcmp(argv[i], "--layers")) layers = true;
    else if (!std::strcmp(argv[i], "--sampling") && i + 3 < argc) {
      const float temperature = std::strtof(argv[++i], nullptr);
      const auto top_k = static_cast<int32_t>(std::strtol(argv[++i], nullptr, 10));
      m->set_sampling(temperature, top_k, std::strtoull(argv[++i], nullptr, 10));
    }
    else if (!std::strcmp(argv[i], "--top-p") && i + 1 < argc) m->set_top_p(std::strtof(argv[++i], nullptr));
    else if (!std::strcmp(argv[i], "--repetition-penalty") && i + 2 < argc) {
      const float penalty = std::strtof(argv[++i], nullptr);
      m->set_repetition_penalty(penalty, static_cast<int32_t>(std::strtol(argv[++i], nullptr, 10)));
    }
    else if (!std::strcmp(argv[i], "--frequency-presence") && i + 2 < argc) {
      const float frequency = std::strtof(argv[++i], nullptr);
      const float presence = std::strtof(argv[++i], nullptr);
      int32_t from_pos = 0;
      char* end = nullptr;
      if (i + 1 < argc) {
        const long from = std::strtol(argv[i + 1], &end, 10);
        if (end != argv[i + 1] && *end == '\0') {
          from_pos = static_cast<int32_t>(from);
          ++i;
        }
      }
      m->set_frequency_presence(frequency, presence, from_pos);
    }
    else if (!std::strcmp(argv[i], "--logit-bias") && i + 1 < argc) {
      auto bias = m->draw_config().logit_bias;
      for (char* tok = std::strtok(argv[++i], ","); tok != nullptr; tok = std::strtok(nullptr, ",")) {
        char* colon = std::strchr(tok, ':');
        if (colon == nullptr) return 2;
        bias.emplace_back(static_cast<int32_t>(std::strtol(tok, nullptr, 10)), std::strtof(colon + 1, nullptr));
      }
      m->set_logit_bias(std::move(bias));
    }
    else if (!std::strcmp(argv[i], "--generate") && i + 1 < argc) generate = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--stop") && i + 1 < argc) stops.push_back(std::atoi(argv[++i]));
    else if (!std::strcmp(argv[i], "--then") && i + 1 < argc) then = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--copy-at") && i + 1 < argc) copy_at = std::atoi(argv[++i]);
    // init() refuses a value outside [-1, 20]
    else if (!std::strcmp(argv[i], "--logprobs") && i + 1 < argc) m->set_logprobs(std::atoi(argv[++i]));
    else if (!std::strcmp(argv[i], "--score")) score = true;
    else if (!std::strcmp(argv[i], "--kv-cache") && i + 1 < argc) {
      const std::string v = argv[++i];
      if (v != "fp32" && v != "bf16" && v != "fp8") return 2;
      m->set_bf16_kv_cache(v == "bf16");
      m->set_fp8_kv_cache(v == "fp8");
    }
    else if (!std::strcmp(argv[i], "--weights") && i + 1 < argc) {
      const std::string v = argv[++i];
      if (v != "fp32" && v != "bf16") return 2;
      m->set_bf16_weights(v == "bf16");
    }
    else if (!std::strcmp(argv[i], "--speculative") && i + 1 < argc) m->set_speculative(std::atoi(argv[++i]));
    else if (!std::strcmp(argv[i], "--logits") && i + 1 < argc) logits_path = argv[++i];
    else prompt.push_back(std::atoi(argv[i]));
  }
  if (prompt.empty() || n_steps <= 0) return 2;
  const int32_t logprobs = m->logprobs_top_n();
  if (layers && (logprobs != -1 || score)) {
    std::fprintf(stderr, "--layers has no log-probabilities: --logprobs and --score need the fused decoder\n");
    return 2;
  }
  if (!stops.empty()) m->set_stop_ids(stops);
  size_t free_before = 0, free_after = 0, total = 0;
  const bool meminfo = cudaMemGetInfo(&free_before, &total) == cudaSuccess;
  base::Status st = m->init(base::DeviceType::kDeviceCUDA);
  if (st && meminfo && cudaMemGetInfo(&free_after, &total) == cudaSuccess)
    std::fprintf(stderr, "device bytes after init: %zu\n", free_before - free_after);
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
  // --layers draws with the model's settings too, over the id fed at each position
  sampler::SeededSampler seeded(base::DeviceType::kDeviceCUDA, m->draw_config());
  std::vector<int32_t> fed(static_cast<size_t>(n_steps), -1);
  int next = -1;
  std::vector<int> chosen;
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
    if (!is_prompt) {
      const tensor::Tensor& lg = m->get_buffer(model::ModelBufferType::kForwardOutput);
      seeded.set_position(pos_tensor.index<int32_t>(0), fed);
      next = static_cast<int>(seeded.sample(lg.ptr<float>(), lg.size(), nullptr));
    }
  };
  for (int32_t pos = 0; pos < n_steps; ++pos) {
    pos_tensor.index<int32_t>(0) = pos;
    fed[pos] = pos < prompt_len ? prompt[pos] : next;
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
