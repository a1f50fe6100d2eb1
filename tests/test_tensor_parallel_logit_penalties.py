"""-m gpu, >= 2 GPUs: the logit bias and the frequency and presence penalties under tensor parallelism.  Every rank
feeds the same ids, so every rank's history is the same and no exchange is needed: the persistent engine's gather
phase applies step 0 to its CTA's range of the assembled logits, the graph engine to the replicated classifier's.
Every rank draws the same ids, which follow the rule on each rank's logits and equal the single-GPU decoder's."""
import numpy as np
import pytest

from tp_util import spawn

pytestmark = pytest.mark.gpu

# (T, top_k, top_p, penalty, last_n, seed, frequency, presence, from_pos, bias)
SETTINGS = [(0.0, 0, 1.0, 1.0, 0, 0, 0.6, 1.5, 0, {}), (0.8, 0, 1.0, 1.2, 16, 5, 0.0, 1.0, 4, {3: 2.0, 9: -1.0}),
            (0.7, 20, 0.8, 1.05, 0, 2**40 + 3, 0.4, 0.4, 0, {7: 0.5})]
STEPS = 32
MARGIN = 1e-5


def _need_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _step0_rank(rank, world, key, backend, engine, out_dir):
    import os
    os.environ["KLLM_ENGINE"] = engine
    import torch
    from kuiperllama_b200 import SHAPES, sampling, synth_weights
    from kuiperllama_b200.tensor_parallel import Comm, comm_words, make_tp_decoder
    shape = SHAPES[key]
    full = synth_weights(shape, "cuda", 11)
    comm = Comm(comm_words(shape, world), backend)
    dec = make_tp_decoder(shape, full, comm)
    out = {}
    for i, (T, k, p, theta, last_n, seed, f, pr, from_pos, bias) in enumerate(SETTINGS):
        dec.set_sampling(T, k, seed, top_p=p)
        dec.set_repetition_penalty(theta, last_n)
        dec.set_frequency_presence(f, pr, from_pos)
        dec.set_logit_bias(bias)
        torch.distributed.barrier()  # the ranks' kernels wait for each other's partial sums: start together
        ids = dec.generate(1, 0, STEPS)
        tok, stepped, fed = 1, [], []
        for pos in range(STEPS):
            fed.append(tok)
            tok = dec.step(tok, pos)
            stepped.append(tok)
            pen = sampling.penalties(dec.logits(), bias=sampling.bias_table(bias, shape.vocab_size),
                                     rep_ids=sampling.history_window(fed, pos, last_n), penalty=theta,
                                     count_ids=sampling.count_window(fed, pos, from_pos), frequency=f, presence=pr)
            if sampling.margin(pen, T, k, seed, pos, top_p=p) >= MARGIN:
                assert tok == sampling.sample(pen, T, k, seed, pos, top_p=p), (rank, engine, i, pos)
        assert stepped == ids, (rank, engine, i)
        assert list(dec.history()[:STEPS]) == fed, (rank, engine, i)
        out[f"s{i}"] = np.array(ids)
    np.savez(f"{out_dir}/{backend}_{engine}_rank{rank}.npz", **out)
    dec.close()
    comm.close()


@pytest.mark.parametrize("key", ["small-tp", "small-qwen"])
def test_tp_ranks_draw_the_same_ids_with_bias_and_penalties(kllm_lib, tmp_path, key):
    _need_gpus(2)
    world = 2
    modes = [("peer", "persistent"), ("peer", "graph")]
    for backend, engine in modes:
        spawn(_step0_rank, world, "nccl", (key, backend, engine, str(tmp_path)))
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[key]
    dec = Decoder(shape, synth_weights(shape, "cuda", 11))
    want = {}
    for i, (T, k, p, theta, last_n, seed, f, pr, from_pos, bias) in enumerate(SETTINGS):
        dec.set_sampling(T, k, seed, top_p=p)
        dec.set_repetition_penalty(theta, last_n)
        dec.set_frequency_presence(f, pr, from_pos)
        dec.set_logit_bias(bias)
        want[f"s{i}"] = dec.generate(1, 0, STEPS)
    dec.close()
    for backend, engine in modes:
        for r in range(world):
            got = np.load(tmp_path / f"{backend}_{engine}_rank{r}.npz")
            for name, ids in want.items():
                assert list(got[name]) == ids, (backend, engine, r, name)
