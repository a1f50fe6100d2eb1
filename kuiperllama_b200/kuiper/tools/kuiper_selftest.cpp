// kuiper_selftest: host-side semantics of the kuiper:: API mirror that need no GPU -- the CPU cases
// of the reference's own gtest programs (test/test_tensor/test_tensor.cpp: init1/init2/init3/
// assign1/clone_cpu; test/test_tensor/test_buffer.cpp: allocate/use_external) plus the Status,
// layer-check and checkpoint-header behaviour the model code relies on.  Plain asserts, no gtest.
//
//   kuiper_selftest [checkpoint.bin [llama|qwen fp32|int8]]      exit code 0 = all passed
#include <base/base.h>
#include <base/buffer.h>
#include <base/memory.h>
#include <glog/logging.h>
#include <op/add.h>
#include <op/matmul.h>
#include <op/rmsnorm.h>
#include <tensor/tensor.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "model/config.h"
#include "model/llama3.h"
#include "model/qwen2.h"
#include "model/raw_model_data.h"

namespace model {
// Runs the loading pipeline of a model (tokenizer stand-in -> mmap + header -> layers as views into
// the mapping) WITHOUT init(): no GPU involved, nothing uploaded.
struct ModelInspector {
  static base::Status load(LLama2Model& m) { return m.gen_model_from_file(); }
  static const TransformerConfig& config(const LLama2Model& m) { return *m.config_; }
  static const LLama2Layers& layers(const LLama2Model& m) { return *m.llama_layers_; }
  static const char* payload(const LLama2Model& m) { return static_cast<const char*>(m.raw_model_data_->weight_data); }
  static size_t file_size(const LLama2Model& m) { return m.raw_model_data_->file_size; }
  static int32_t group_size(const LLama2Model& m) { return m.group_size_; }
  // the draw settings init() goes on to validate
  static sampler::DrawConfig draw_from_env(const LLama2Model& m) {
    sampler::DrawConfig cfg = m.draw_;
    sampler::fill_from_env(cfg, m.draw_set_);
    return cfg;
  }
};
}  // namespace model

namespace {
int g_failed = 0, g_run = 0;
#define EXPECT(cond)                                                              \
  do {                                                                            \
    if (!(cond)) {                                                                \
      std::fprintf(stderr, "  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);     \
      ++g_failed;                                                                 \
    }                                                                             \
  } while (0)

void run(const char* name, const std::function<void()>& fn) {
  ++g_run;
  const int before = g_failed;
  fn();
  std::printf("[%s] %s\n", g_failed == before ? "  ok  " : "FAILED", name);
}
}  // namespace

// kuiper_selftest --bf16-round in.f32 out.u16: the host's fp32 -> bf16 rounding (base::fp32_to_bf16_rne, what the
// bf16-weight upload applies) over a raw fp32 file, written as raw bf16 bits.
static int bf16_round(const char* in_path, const char* out_path) {
  FILE* in = std::fopen(in_path, "rb");
  FILE* out = std::fopen(out_path, "wb");
  if (in == nullptr || out == nullptr) return 2;
  float f;
  while (std::fread(&f, sizeof(f), 1, in) == 1) {
    const uint16_t b = base::fp32_to_bf16_rne(f);
    if (std::fwrite(&b, sizeof(b), 1, out) != 1) return 2;
  }
  std::fclose(in);
  return std::fclose(out) == 0 ? 0 : 2;
}

int main(int argc, char** argv) {
  using namespace base;
  if (argc == 4 && !std::strcmp(argv[1], "--bf16-round")) return bf16_round(argv[2], argv[3]);
  auto cpu = CPUDeviceAllocatorFactory::get_instance();

  run("buffer.allocate", [&] {  // test_buffer.cpp:7-12
    Buffer buffer(32, cpu);
    EXPECT(buffer.ptr() != nullptr);
    EXPECT(buffer.byte_size() == 32);
    EXPECT(buffer.device_type() == DeviceType::kDeviceCPU);
    EXPECT(!buffer.is_external());
  });
  run("buffer.use_external", [&] {  // test_buffer.cpp:14-21
    float* ptr = new float[32];
    {
      Buffer buffer(32, nullptr, ptr, true);
      EXPECT(buffer.is_external());
      EXPECT(buffer.ptr() == ptr);
    }
    ptr[0] = 1.f;  // still ours: an external buffer never frees
    delete[] ptr;
  });
  run("buffer.copy_from cpu->cpu", [&] {
    Buffer a(64, cpu), b(64, cpu);
    for (int i = 0; i < 16; ++i) static_cast<float*>(a.ptr())[i] = float(i);
    b.copy_from(a);
    EXPECT(std::memcmp(a.ptr(), b.ptr(), 64) == 0);
  });

  run("tensor.init1 (1-D, need_alloc)", [&] {  // test_tensor.cpp:95-103
    tensor::Tensor t1(DataType::kDataTypeFp32, 32 * 151, true, cpu);
    EXPECT(!t1.is_empty());
    EXPECT(t1.size() == 32u * 151u && t1.byte_size() == 32u * 151u * 4u && t1.dims_size() == 1);
  });
  run("tensor.init2 (1-D, no alloc -> empty even with an allocator)", [&] {  // test_tensor.cpp:115-123
    tensor::Tensor t1(DataType::kDataTypeFp32, 32 * 151, false, cpu);
    EXPECT(t1.is_empty());
  });
  run("tensor.init3 (wraps external memory)", [&] {  // test_tensor.cpp:105-113
    float* ptr = new float[32];
    ptr[0] = 31;
    tensor::Tensor t1(DataType::kDataTypeFp32, 32, false, nullptr, ptr);
    EXPECT(!t1.is_empty());
    EXPECT(t1.ptr<float>() == ptr);
    EXPECT(*t1.ptr<float>() == 31);
    delete[] ptr;
  });
  run("tensor.assign1", [&] {  // test_tensor.cpp:125-143
    tensor::Tensor t(DataType::kDataTypeFp32, 32, 32, true, cpu);
    EXPECT(!t.is_empty());
    const int32_t size = 32 * 32;
    float* ptr = new float[size];
    for (int i = 0; i < size; ++i) ptr[i] = float(i);
    auto buffer = std::make_shared<Buffer>(size * sizeof(float), nullptr, ptr, true);
    buffer->set_device_type(DeviceType::kDeviceCPU);
    EXPECT(t.assign(buffer));
    EXPECT(!t.is_empty());
    EXPECT(t.ptr<float>() == ptr);
    EXPECT(t.index<float>(5) == 5.f);
    // a buffer that is too small is refused
    auto small = std::make_shared<Buffer>(16, nullptr, ptr, true);
    EXPECT(!t.assign(small));
    delete[] ptr;
  });
  run("tensor.clone_cpu", [&] {  // test_tensor.cpp:53-74
    tensor::Tensor t1(DataType::kDataTypeFp32, 32, 32, true, cpu);
    for (int i = 0; i < 32 * 32; ++i) t1.index<float>(i) = 1.f;
    tensor::Tensor t2 = t1.clone();
    EXPECT(t2.ptr<float>() != t1.ptr<float>());
    EXPECT(t2.size() == t1.size() && t2.data_type() == DataType::kDataTypeFp32);
    for (int i = 0; i < 32 * 32; ++i) EXPECT(t2.index<float>(i) == 1.f);
    t2.index<float>(0) = 7.f;
    EXPECT(t1.index<float>(0) == 1.f);  // deep copy
    tensor::Tensor t3 = t1;             // plain copy shares the buffer
    EXPECT(t3.ptr<float>() == t1.ptr<float>());
  });
  run("tensor.reshape / strides / dims", [&] {
    tensor::Tensor t(DataType::kDataTypeFp32, 4, 6, true, cpu);
    EXPECT(t.get_dim(0) == 4 && t.get_dim(1) == 6);
    const auto st = t.strides();
    EXPECT(st.size() == 2 && st[0] == 6 && st[1] == 1);
    for (int i = 0; i < 24; ++i) t.index<float>(i) = float(i);
    t.reshape({2, 12});  // same size: the data stays
    EXPECT(t.get_dim(0) == 2 && t.get_dim(1) == 12 && t.index<float>(23) == 23.f);
    t.reshape({8, 8});  // grows: reallocated, old contents carried over
    EXPECT(t.size() == 64 && t.index<float>(23) == 23.f);
    tensor::Tensor i8(DataType::kDataTypeInt8, 10, true, cpu);
    EXPECT(i8.byte_size() == 10);
    tensor::Tensor i32(DataType::kDataTypeInt32, 10, true, cpu);
    EXPECT(i32.byte_size() == 40);
  });

  run("status", [&] {
    Status ok = error::Success();
    EXPECT(bool(ok) && ok.get_err_code() == StatusCode::kSuccess);
    Status bad = error::InvalidArgument("nope");
    EXPECT(!bad && bad.get_err_code() == StatusCode::kInvalidArgument && bad.get_err_msg() == "nope");
    EXPECT(bad == StatusCode::kInvalidArgument && bad != StatusCode::kSuccess);
    EXPECT(error::PathNotValid().get_err_code() == StatusCode::kPathNotValid);
    EXPECT(error::ModelParseError().get_err_code() == StatusCode::kModelParseError);
    EXPECT(error::KeyHasExits().get_err_code() == StatusCode::kKeyValueHasExist);
    EXPECT(error::FunctionNotImplement().get_err_code() == StatusCode::kFunctionUnImplement);
  });

  run("layer.check rejects wrong shapes / devices before any kernel is looked up", [&] {
    op::VecAddLayer add(DeviceType::kDeviceCUDA);
    tensor::Tensor a(DataType::kDataTypeFp32, 8, true, cpu), b(DataType::kDataTypeFp32, 8, true, cpu),
        c(DataType::kDataTypeFp32, 8, true, cpu);
    add.set_input(0, a), add.set_input(1, b), add.set_output(0, c);
    EXPECT(!add.check());  // CPU tensors handed to a CUDA layer
    op::VecAddLayer empty(DeviceType::kDeviceCUDA);
    EXPECT(!empty.check());  // nothing bound
    op::RmsNormLayer norm(DeviceType::kDeviceCUDA, 16);
    EXPECT(norm.weight_size() == 1);
    float w[16] = {};
    EXPECT(bool(norm.set_weight(0, {16}, w, DeviceType::kDeviceCPU)));
    EXPECT(norm.get_weight(0).ptr<float>() == w);  // a view, not a copy (mmap'd checkpoint)
    tensor::Tensor x(DataType::kDataTypeFp32, 12, true, cpu);
    norm.set_input(0, x), norm.set_output(0, x);
    EXPECT(!norm.check());  // 12 != 16
    op::MatmulLayer mm(DeviceType::kDeviceCUDA, 4, 64, /*is_quant_layer=*/true);
    mm.set_group_size(64);
    std::vector<int8_t> blob(4 * 64 + 4 * sizeof(float));
    EXPECT(bool(mm.set_weight(0, {4, 64}, blob.data(), DeviceType::kDeviceCPU)));
    EXPECT(mm.get_scale_num() == 4);
    // export.py --version 3: the fp32 group scales sit right behind the int8 block
    EXPECT(static_cast<const void*>(mm.get_scales().ptr<float>()) == static_cast<const void*>(blob.data() + 4 * 64));
  });

  run("draw settings: each group from its setter, else from its KUIPER_* variables, else the default", [&] {
    const char* vars[][2] = {{"KUIPER_TEMPERATURE", "0.5"}, {"KUIPER_TOP_K", "7"}, {"KUIPER_SEED", "9"},
                             {"KUIPER_TOP_P", "0.5"}, {"KUIPER_REPETITION_PENALTY", "1.5"}, {"KUIPER_REPEAT_LAST_N", "4"},
                             {"KUIPER_FREQUENCY_PENALTY", "0.25"}, {"KUIPER_PRESENCE_PENALTY", "0.75"}};
    // the defaults, the values of `vars` and the values the setters below are given
    const sampler::DrawConfig unset, env{0.5f, 7, 9, 0.5f, 1.5f, 4, 0.25f, 0.75f, 0},
        set{0.875f, 3, 11, 0.625f, 1.25f, 2, 0.125f, 0.375f, 5};
    auto group = [](const sampler::DrawConfig& c, int g) {  // the fields of group g
      return std::vector<std::vector<double>>{{c.temperature, double(c.top_k), double(c.seed)}, {c.top_p},
                                              {c.penalty, double(c.last_n)},
                                              {c.frequency, c.presence, double(c.from_pos)}}[g];
    };
    // init()'s settings with or without the variables, after the setters of the groups in `mask`
    auto expect = [&](bool env_on, unsigned mask) {
      for (const auto& v : vars) env_on ? setenv(v[0], v[1], 1) : unsetenv(v[0]);
      model::LLama2Model m(TokenizerType::kEncodeSpe, "<none>", "<none>", false);
      if (mask & 1) m.set_sampling(set.temperature, set.top_k, set.seed);
      if (mask & 2) m.set_top_p(set.top_p);
      if (mask & 4) m.set_repetition_penalty(set.penalty, set.last_n);
      if (mask & 8) m.set_frequency_presence(set.frequency, set.presence, set.from_pos);
      const sampler::DrawConfig c = model::ModelInspector::draw_from_env(m);
      for (int g = 0; g < 4; ++g) EXPECT(group(c, g) == group(mask >> g & 1 ? set : env_on ? env : unset, g));
    };
    for (unsigned mask : {0u, 1u, 2u, 4u, 8u, 15u}) expect(true, mask);  // the environment only, one setter each, all
    expect(false, 15), expect(false, 0);                                   // the setters only; neither
  });

  if (argc > 1) {
    run("checkpoint header (model/config.h, export.py:91-92)", [&] {
      FILE* f = std::fopen(argv[1], "rb");
      EXPECT(f != nullptr);
      if (!f) return;
      model::ModelConfig cfg{};
      EXPECT(std::fread(&cfg, sizeof(cfg), 1, f) == 1);
      std::fclose(f);
      EXPECT(sizeof(cfg) == 28);
      EXPECT(cfg.dim > 0 && cfg.layer_num > 0 && cfg.head_num % cfg.kv_head_num == 0);
      std::printf("         dim %d hidden %d layers %d heads %d kv_heads %d vocab %d seq_len %d\n", cfg.dim,
                  cfg.hidden_dim, cfg.layer_num, cfg.head_num, cfg.kv_head_num, cfg.vocab_size, cfg.seq_len);
    });
  }

  // kuiper_selftest <ckpt> <llama|qwen> <fp32|int8>: the layers must be views at the offsets the
  // exporter's layout implies (tools/export.py / export_qwen2.py), computed here independently
  if (argc > 3) {
    const std::string family = argv[2];
    const bool quant = std::string(argv[3]) == "int8";
    run("model loading pipeline: header, config, every weight a view at its file offset", [&] {
      std::unique_ptr<model::LLama2Model> m;
      if (family == "qwen")
        m = std::make_unique<model::Qwen2Model>(TokenizerType::kEncodeBpe, "<none>", argv[1], quant);
      else
        m = std::make_unique<model::LLama2Model>(TokenizerType::kEncodeSpe, "<none>", argv[1], quant);
      using I = model::ModelInspector;
      const base::Status st = I::load(*m);
      EXPECT(bool(st));
      if (!st) return;
      const auto& c = I::config(*m);
      const auto& ly = I::layers(*m);
      const size_t dim = c.dim_, kvd = c.kv_dim_, hid = c.hidden_dim_, L = c.layer_num_, V = c.vocab_size_;
      EXPECT(c.head_size_ * c.head_num_ == c.dim_ && c.kv_mul_ * c.kv_head_num_ == c.head_num_);
      EXPECT(ly.wq_layers_.size() == L && ly.w2_layers_.size() == L && ly.rmsnorm_layers_.size() == 2 * L + 1);
      auto weight_at = [&](const std::shared_ptr<op::Layer>& l) {
        return reinterpret_cast<const char*>(std::static_pointer_cast<op::LayerParam>(l)->get_weight(0).ptr<int8_t>());
      };
      const char* base_ptr = I::payload(*m);
      const bool bias = family == "qwen" && !quant;
      if (!quant) {
        size_t off = 0;  // bytes
        EXPECT(weight_at(ly.embedding_layer_) == base_ptr + off);
        off += V * dim * 4;
        EXPECT(weight_at(ly.rmsnorm_layers_[0]) == base_ptr + off);
        off += L * dim * 4;
        const size_t q_stride = (dim * dim + (bias ? dim : 0)) * 4, kv_stride = (kvd * dim + (bias ? kvd : 0)) * 4;
        EXPECT(weight_at(ly.wq_layers_[L - 1]) == base_ptr + off + (L - 1) * q_stride);
        off += L * q_stride;
        EXPECT(weight_at(ly.wk_layers_[L - 1]) == base_ptr + off + (L - 1) * kv_stride);
        off += L * kv_stride;
        EXPECT(weight_at(ly.wv_layers_[0]) == base_ptr + off);
        off += L * kv_stride;
        EXPECT(weight_at(ly.wo_layers_[0]) == base_ptr + off);
        off += L * dim * dim * 4;
        EXPECT(weight_at(ly.rmsnorm_layers_[L]) == base_ptr + off);  // first ffn norm
        off += L * dim * 4;
        EXPECT(weight_at(ly.w1_layers_[0]) == base_ptr + off);
        off += L * hid * dim * 4;
        EXPECT(weight_at(ly.w2_layers_[0]) == base_ptr + off);
        off += L * dim * hid * 4;
        EXPECT(weight_at(ly.w3_layers_[L - 1]) == base_ptr + off + (L - 1) * hid * dim * 4);
        off += L * hid * dim * 4;
        EXPECT(weight_at(ly.rmsnorm_layers_[2 * L]) == base_ptr + off);  // final norm
        off += dim * 4 + static_cast<size_t>(c.seq_len_) * c.head_size_ * 4;  // + freqs_cos | freqs_sin
        if (c.is_shared_weight_) {
          EXPECT(weight_at(ly.cls_layer_) == weight_at(ly.embedding_layer_));
        } else {
          EXPECT(weight_at(ly.cls_layer_) == base_ptr + off);
          off += V * dim * 4;
        }
        EXPECT(off + 28 == I::file_size(*m));
        if (bias) {
          auto mm = std::static_pointer_cast<op::MatmulLayer>(ly.wq_layers_[0]);
          EXPECT(mm->has_bias());
          EXPECT(reinterpret_cast<const char*>(mm->get_bias(0).ptr<float>()) == weight_at(ly.wq_layers_[0]) + dim * dim * 4);
        }
      } else {
        const size_t g = static_cast<size_t>(I::group_size(*m));
        EXPECT(g == 64);
        auto blob = [&](size_t rows, size_t cols) { return rows * cols + rows * cols / g * 4; };
        size_t off = 0;
        EXPECT(weight_at(ly.wq_layers_[0]) == base_ptr + off);
        auto q0 = std::static_pointer_cast<op::LayerParam>(ly.wq_layers_[0]);
        EXPECT(reinterpret_cast<const char*>(q0->get_scales().ptr<float>()) == base_ptr + dim * dim);
        off += L * blob(dim, dim);
        EXPECT(weight_at(ly.wk_layers_[0]) == base_ptr + off);
        off += 2 * L * blob(kvd, dim);
        EXPECT(weight_at(ly.wo_layers_[0]) == base_ptr + off);
        off += L * blob(dim, dim);
        EXPECT(weight_at(ly.w1_layers_[0]) == base_ptr + off);
        off += L * blob(hid, dim);
        EXPECT(weight_at(ly.w2_layers_[L - 1]) == base_ptr + off + (L - 1) * blob(dim, hid));
        off += L * blob(dim, hid);
        EXPECT(weight_at(ly.w3_layers_[0]) == base_ptr + off);
        off += L * blob(hid, dim);
        EXPECT(weight_at(ly.cls_layer_) == base_ptr + off);
        off += blob(V, dim);
        EXPECT(weight_at(ly.embedding_layer_) == base_ptr + off);
        off += V * dim * 4;
        EXPECT(weight_at(ly.rmsnorm_layers_[0]) == base_ptr + off);
        EXPECT(weight_at(ly.rmsnorm_layers_[2 * L]) == base_ptr + off + 2 * L * dim * 4);
        off += (2 * L + 1) * dim * 4;
        EXPECT(off + 32 == I::file_size(*m));
      }
    });
  }

  std::printf("%d groups, %d failed expectation(s)\n", g_run, g_failed);
  return g_failed == 0 ? 0 : 1;
}
