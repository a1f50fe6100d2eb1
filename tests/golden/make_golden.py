"""Generate the golden fixtures in this directory by IMPORTING the reference's own PyTorch
model and exporters (tools/model.py, tools/export.py, tools/model_qwen2.py,
tools/export_qwen2.py) from a reference checkout:

    KUIPER_REFERENCE_DIR=/path/to/KuiperLLama python tests/golden/make_golden.py

Outputs (committed):
  tiny_llama2_fp32_shared.bin / .npz     legacy_export (v0), shared classifier
  tiny_llama2_fp32.bin        / .npz     legacy_export (v0), separate classifier
  tiny_llama2_int8.bin        / .npz     legacy_export_quant (v3, group 64)
  tiny_qwen2file_fp32.bin     / .npz     export_qwen2.legacy_export (bias after wq/wk/wv);
                                         NOTE tools/model_qwen2.py keeps Llama-2 arithmetic
                                         (interleaved RoPE, theta 1e4, eps 1e-5), so this pins
                                         the FILE LAYOUT + bias path, not the QWEN2_SUPPORT math.
Each .npz holds `tokens` [T] and `logits` [T, vocab]: PyTorch fp32 logits of the reference
Transformer at the last position of tokens[:t+1] for every t (teacher forced).  For int8 the
PyTorch model carries the DEQUANTISED weights q*scale of the exporter's own quantize_q80.
The reference's unit-test known answers (test_load.cpp, test_cu_matmul.cpp, ...) are written to
reference_known_answers.json by hand-transcription of the constants, with file:line.
"""
import copy
import os
import sys

import numpy as np
import torch

REF_TOOLS = os.path.join(os.environ["KUIPER_REFERENCE_DIR"], "tools")
sys.path.insert(0, REF_TOOLS)
HERE = os.path.dirname(os.path.abspath(__file__))


def randomise_norms(model, gen):
    for layer in model.layers:
        layer.attention_norm.weight.data.uniform_(0.5, 1.5, generator=gen)
        layer.ffn_norm.weight.data.uniform_(0.5, 1.5, generator=gen)
    model.norm.weight.data.uniform_(0.5, 1.5, generator=gen)


def logits_per_position(model, tokens):
    model.eval()
    out = []
    with torch.no_grad():
        for t in range(len(tokens)):
            lg = model(torch.tensor([tokens[: t + 1]], dtype=torch.long))
            out.append(lg[0, -1].float().numpy().copy())
    return np.stack(out).astype(np.float32)


def main():
    import export as ref_export
    import model as ref_model
    torch.manual_seed(20240923)
    gen = torch.Generator().manual_seed(7)
    args = dict(dim=64, n_layers=2, n_heads=4, n_kv_heads=2, vocab_size=128, hidden_dim=128,
                max_seq_len=32)
    tokens = [1, 5, 17, 99, 3, 64, 127, 0, 42, 42, 8, 120]

    # ---- shared classifier, fp32 v0 -------------------------------------------------
    m = ref_model.Transformer(ref_model.ModelArgs(**args))
    randomise_norms(m, gen)
    ref_export.legacy_export(m, os.path.join(HERE, "tiny_llama2_fp32_shared.bin"))
    m.params.vocab_size = abs(m.params.vocab_size)
    np.savez(os.path.join(HERE, "tiny_llama2_fp32_shared.npz"), tokens=np.array(tokens, np.int32),
             logits=logits_per_position(m, tokens))

    # ---- separate classifier, fp32 v0 ------------------------------------------------
    m2 = ref_model.Transformer(ref_model.ModelArgs(**args))
    randomise_norms(m2, gen)
    m2.tok_embeddings.weight = torch.nn.Parameter(m2.tok_embeddings.weight.detach().clone())
    m2.output.weight = torch.nn.Parameter(torch.empty(args["vocab_size"], args["dim"]).normal_(0, 0.02, generator=gen))
    assert not torch.equal(m2.tok_embeddings.weight, m2.output.weight)
    ref_export.legacy_export(m2, os.path.join(HERE, "tiny_llama2_fp32.bin"))
    m2.params.vocab_size = abs(m2.params.vocab_size)
    np.savez(os.path.join(HERE, "tiny_llama2_fp32.npz"), tokens=np.array(tokens, np.int32),
             logits=logits_per_position(m2, tokens))

    # ---- int8 v3 of the same separate-classifier model ----------------------------------
    ref_export.legacy_export_quant(m2, os.path.join(HERE, "tiny_llama2_int8.bin"))
    m2.params.vocab_size = abs(m2.params.vocab_size)
    mq = copy.deepcopy(m2)
    with torch.no_grad():
        def deq(p):
            q, s, _ = ref_export.quantize_q80(p, 64)
            return (q.float().view(-1, 64) * s.float()[:, None]).view(p.shape)
        for layer in mq.layers:
            for lin in (layer.attention.wq, layer.attention.wk, layer.attention.wv,
                        layer.attention.wo, layer.feed_forward.w1, layer.feed_forward.w2,
                        layer.feed_forward.w3):
                lin.weight.copy_(deq(lin.weight))
        mq.output.weight.copy_(deq(mq.output.weight))
    np.savez(os.path.join(HERE, "tiny_llama2_int8.npz"), tokens=np.array(tokens, np.int32),
             logits=logits_per_position(mq, tokens))

    # ---- Qwen2 file layout (bias) --------------------------------------------------------
    import export_qwen2 as ref_export_q
    import model_qwen2 as ref_model_q
    mqw = ref_model_q.Transformer(ref_model_q.ModelArgs(**args))
    randomise_norms(mqw, gen)
    with torch.no_grad():
        for layer in mqw.layers:
            for lin in (layer.attention.wq, layer.attention.wk, layer.attention.wv):
                lin.bias.normal_(0, 0.02, generator=gen)
    ref_export_q.legacy_export(mqw, os.path.join(HERE, "tiny_qwen2file_fp32.bin"))
    mqw.params.vocab_size = abs(mqw.params.vocab_size)
    np.savez(os.path.join(HERE, "tiny_qwen2file_fp32.npz"), tokens=np.array(tokens, np.int32),
             logits=logits_per_position(mqw, tokens))
    for f in sorted(os.listdir(HERE)):
        print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
