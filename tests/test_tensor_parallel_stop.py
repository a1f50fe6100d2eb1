"""-m gpu, >= 2 GPUs: kllm_decoder_generate_until under tensor parallelism.  Every rank computes the same id, so
every rank stops on the same step without an exchange (persistent engine) or launches exactly the same steps
(graph engine, host-driven), on both transports; the ids are the single-GPU decoder's, and a generate that
follows finds the exchange tags and barrier counts where the stopped run left them."""
import numpy as np
import pytest

from tp_util import spawn

pytestmark = pytest.mark.gpu

STEPS = 48
MODES = [("peer", "persistent"), ("peer", "graph"), ("nccl", "graph")]


def _need_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _stop_rank(rank, world, key, backend, engine, stop_id, out_dir):
    import os
    os.environ["KLLM_ENGINE"] = engine
    import torch
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.tensor_parallel import Comm, comm_words, make_tp_decoder
    shape = SHAPES[key]
    comm = Comm(comm_words(shape, world), backend)
    dec = make_tp_decoder(shape, synth_weights(shape, "cuda", 11), comm)
    assert dec.engine == engine
    out = {}
    for name, stops in (("none", []), ("hit", [stop_id])):
        torch.distributed.barrier()  # the ranks' kernels wait for each other's partial sums: start together
        got = []
        ids = dec.generate_until(1, 0, STEPS, stops, on_tokens=got.extend)
        assert got == ids
        torch.distributed.barrier()
        rest = dec.generate(ids[-1], len(ids), 8) if len(ids) + 8 <= shape.seq_len else []
        out[name] = np.array(ids)
        out[name + "_rest"] = np.array(rest)
    np.savez(f"{out_dir}/{backend}_{engine}_rank{rank}.npz", **out)
    dec.close()
    comm.close()


@pytest.mark.parametrize("key", ["small-tp", "small-qwen"])
def test_tp_ranks_stop_on_the_same_step(kllm_lib, tmp_path, key):
    _need_gpus(2)
    world = 2
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[key]
    dec = Decoder(shape, synth_weights(shape, "cuda", 11))
    full = dec.generate(1, 0, STEPS + 8)
    j = next(j for j in range(STEPS // 3, STEPS) if full[j] not in full[:j])
    dec.close()
    for backend, engine in MODES:
        spawn(_stop_rank, world, "nccl", (key, backend, engine, full[j], str(tmp_path)))
    for backend, engine in MODES:
        for r in range(world):
            got = np.load(tmp_path / f"{backend}_{engine}_rank{r}.npz")
            assert list(got["none"]) == full[:STEPS], (backend, engine, r)
            assert list(got["none_rest"]) == full[STEPS:STEPS + 8], (backend, engine, r)
            assert list(got["hit"]) == full[:j + 1], (backend, engine, r)
            assert list(got["hit_rest"]) == full[j + 1:j + 9], (backend, engine, r)
