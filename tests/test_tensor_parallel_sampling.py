"""-m gpu, >= 2 GPUs: seeded sampling under tensor parallelism.  Every rank draws the same ids, with the
classifier sharded by vocabulary (persistent engine: each rank computes vocab / world rows and the gather
phase assembles the logits and folds the perturbed partials) or replicated (graph engine); the ids follow
the rule on each rank's logits and equal the single-GPU decoder's."""
import numpy as np
import pytest

from tp_util import spawn

pytestmark = pytest.mark.gpu

SETTINGS = [(0.8, 0, 5), (0.9, 40, 2**40 + 3)]
STEPS = 32
MARGIN = 1e-5


def _need_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _sampled_rank(rank, world, key, backend, engine, out_dir):
    import os
    os.environ["KLLM_ENGINE"] = engine
    import torch
    from kuiperllama_b200 import SHAPES, KllmError, sampling, synth_weights
    from kuiperllama_b200.tensor_parallel import Comm, comm_words, make_tp_decoder
    shape = SHAPES[key]
    full = synth_weights(shape, "cuda", 11)
    comm = Comm(comm_words(shape, world), backend)
    try:
        dec = make_tp_decoder(shape, full, comm)
    except KllmError as e:
        assert engine == "persistent" and "unsupported shape" in str(e), e
        open(f"{out_dir}/{backend}_{engine}_rank{rank}.refused", "w").write(str(e))
        comm.close()
        return
    assert dec.classifier_rows == (shape.vocab_size // world if engine == "persistent" else shape.vocab_size)
    out = {}
    for T, k, seed in SETTINGS:
        dec.set_sampling(T, k, seed)
        torch.distributed.barrier()  # the ranks' kernels wait for each other's partial sums: start together
        ids = dec.generate(1, 0, STEPS)
        tok, stepped = 1, []
        for pos in range(STEPS):
            tok = dec.step(tok, pos)
            stepped.append(tok)
            lg = dec.logits()
            if sampling.margin(lg, T, k, seed, pos) >= MARGIN:
                assert tok == sampling.sample(lg, T, k, seed, pos), (rank, engine, T, k, pos)
        assert stepped == ids, (rank, engine, T, k)
        out[f"k{k}"] = np.array(ids)
    np.savez(f"{out_dir}/{backend}_{engine}_rank{rank}.npz", **out)
    dec.close()
    comm.close()


@pytest.mark.parametrize("key", ["small-tp", "small-qwen"])
def test_tp_ranks_draw_the_same_sampled_ids(kllm_lib, tmp_path, key):
    _need_gpus(2)
    world = 2
    modes = [("peer", "persistent"), ("peer", "graph")]
    for backend, engine in modes:
        spawn(_sampled_rank, world, "nccl", (key, backend, engine, str(tmp_path)))
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[key]
    dec = Decoder(shape, synth_weights(shape, "cuda", 11))
    want = {}
    for T, k, seed in SETTINGS:
        dec.set_sampling(T, k, seed)
        want[f"k{k}"] = dec.generate(1, 0, STEPS)
    dec.close()
    assert not (tmp_path / "peer_persistent_rank0.refused").exists(), "the persistent engine must take this shape"
    for backend, engine in modes:
        for r in range(world):
            got = np.load(tmp_path / f"{backend}_{engine}_rank{r}.npz")
            for name, ids in want.items():
                assert list(got[name]) == ids, (backend, engine, r, name)


@pytest.mark.parametrize("key,family,prec,variant", [("small-tp", "llama", "fp32", "llama2"),
                                                     ("small-qwen", "qwen", "fp32", "qwen2")])
def test_cpp_tensor_parallel_sampling_equals_single_gpu(kllm_lib, tmp_path, key, family, prec, variant):
    """kuiper_tp_launch 2 kuiper_decode with KUIPER_TEMPERATURE / KUIPER_TOP_K / KUIPER_SEED: both ranks read
    the same environment and draw the same ids (a rank that drew another id would feed the exchange a
    different token), and those are the single-GPU run's ids."""
    import os
    import subprocess
    from test_cpp_tensor_parallel import free_port, tool
    from kuiperllama_b200 import SHAPES
    from kuiperllama_b200.checkpoint import write_checkpoint
    from kuiperllama_b200.decoder import synth_weights
    _need_gpus(2)
    shape = SHAPES[key]
    path = tmp_path / "model.bin"
    write_checkpoint(str(path), shape, synth_weights(shape, device="cpu", seed=11))
    steps, prompt = 40, [1, 5, 9]
    decode = tool(variant, "kuiper_decode")
    args = [str(path), family, prec, str(steps), *map(str, prompt)]
    for T, k, seed in SETTINGS:
        env = dict(os.environ, KUIPER_TEMPERATURE=str(T), KUIPER_TOP_K=str(k), KUIPER_SEED=str(seed))
        one = subprocess.run([decode, *args], capture_output=True, text=True, timeout=300, env=env)
        assert one.returncode == 0, one.stderr
        many = subprocess.run([tool(variant, "kuiper_tp_launch"), "2", "--port", str(free_port()), "--", decode, *args],
                              capture_output=True, text=True, timeout=600, env=env)
        assert many.returncode == 0, many.stderr
        assert "persistent" in many.stderr
        assert one.stdout.split() == many.stdout.split(), (T, k)
