"""-m gpu, >= 2 GPUs: nucleus (top-p) sampling under tensor parallelism.  With top-p the persistent engine's
gather phase keeps the raw per-CTA maxima and every CTA of every rank draws the id from the assembled
logits; the graph engine replicates the classifier.  Every rank draws the same ids, which follow the rule
on each rank's logits and equal the single-GPU decoder's."""
import numpy as np
import pytest

from tp_util import spawn

pytestmark = pytest.mark.gpu

SETTINGS = [(0.8, 0, 0.9, 5), (0.7, 20, 0.8, 2**40 + 3)]
STEPS = 32
MARGIN = 1e-5


def _need_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _top_p_rank(rank, world, key, backend, engine, out_dir):
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
    for T, k, p, seed in SETTINGS:
        dec.set_sampling(T, k, seed, top_p=p)
        torch.distributed.barrier()  # the ranks' kernels wait for each other's partial sums: start together
        ids = dec.generate(1, 0, STEPS)
        tok, stepped = 1, []
        for pos in range(STEPS):
            tok = dec.step(tok, pos)
            stepped.append(tok)
            lg = dec.logits()
            if sampling.margin(lg, T, k, seed, pos, top_p=p) >= MARGIN:
                assert tok == sampling.sample(lg, T, k, seed, pos, top_p=p), (rank, engine, T, k, p, pos)
        assert stepped == ids, (rank, engine, T, k, p)
        out[f"k{k}"] = np.array(ids)
    np.savez(f"{out_dir}/{backend}_{engine}_rank{rank}.npz", **out)
    dec.close()
    comm.close()


@pytest.mark.parametrize("key", ["small-tp", "small-qwen"])
def test_tp_ranks_draw_the_same_top_p_ids(kllm_lib, tmp_path, key):
    _need_gpus(2)
    world = 2
    modes = [("peer", "persistent"), ("peer", "graph")]
    for backend, engine in modes:
        spawn(_top_p_rank, world, "nccl", (key, backend, engine, str(tmp_path)))
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[key]
    dec = Decoder(shape, synth_weights(shape, "cuda", 11))
    want = {}
    for T, k, p, seed in SETTINGS:
        dec.set_sampling(T, k, seed, top_p=p)
        want[f"k{k}"] = dec.generate(1, 0, STEPS)
    dec.close()
    for backend, engine in modes:
        for r in range(world):
            got = np.load(tmp_path / f"{backend}_{engine}_rank{r}.npz")
            for name, ids in want.items():
                assert list(got[name]) == ids, (backend, engine, r, name)
