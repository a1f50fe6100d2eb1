"""-m gpu, >= 2 GPUs (skipped below that): log-probabilities under tensor parallelism.  The persistent engine's
gather phase gives every rank the whole logits vector and splits it between the CTAs identically on every rank, so
every rank's record -- each written by its own CTA 0 -- is the same bits; the graph engine's replicated classifier
likewise.  The records agree with the single-GPU decoder's within the bound of DESIGN.md 5.8 (top-N ids exactly)."""
import numpy as np
import pytest

from tp_util import spawn

pytestmark = pytest.mark.gpu

STEPS, TOP_N, GRID = 24, 20, 132


def _need_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs: the ranks' records cannot be compared on fewer")


def _logprob_rank(rank, world, key, backend, engine, out_dir):
    import os
    os.environ["KLLM_ENGINE"] = engine
    import torch
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.tensor_parallel import Comm, comm_words, make_tp_decoder
    shape = SHAPES[key]
    full = synth_weights(shape, "cuda", 11)
    comm = Comm(comm_words(shape, world), backend)
    dec = make_tp_decoder(shape, full, comm)
    dec.set_sampling(0.8, 0, 5)
    dec.set_logprobs(TOP_N)
    torch.distributed.barrier()  # the ranks' kernels wait for each other's partial sums: start together
    ids = dec.generate(1, 0, STEPS)
    rec = dec.logprobs(0, STEPS)
    tokens = [int(t) for t in np.random.default_rng(2).integers(0, shape.vocab_size, STEPS + 1)]
    torch.distributed.barrier()
    lp = dec.score(tokens)
    np.savez(f"{out_dir}/{backend}_{engine}_rank{rank}.npz", ids=np.array(ids), rid=rec[0], rlp=rec[1], rti=rec[2],
             rtl=rec[3], score=lp, engine=np.array(dec.engine))
    dec.close()
    comm.close()


@pytest.mark.parametrize("key", ["small-tp", "small-qwen"])
def test_tp_records_identical_on_every_rank(kllm_lib, tmp_path, key):
    _need_gpus(2)
    world = 2
    modes = [("peer", "persistent"), ("peer", "graph")]
    for backend, engine in modes:
        spawn(_logprob_rank, world, "nccl", (key, backend, engine, str(tmp_path)))
    from kuiperllama_b200 import SHAPES, Decoder, sampling, synth_weights
    shape = SHAPES[key]
    V = shape.vocab_size
    dec = Decoder(shape, synth_weights(shape, "cuda", 11))
    dec.set_sampling(0.8, 0, 5)
    dec.set_logprobs(TOP_N)
    want_ids = dec.generate(1, 0, STEPS)
    want = dec.logprobs(0, STEPS)
    tokens = [int(t) for t in np.random.default_rng(2).integers(0, V, STEPS + 1)]
    want_score = dec.score(tokens)
    k1 = sampling.chain_persistent(V, GRID) if dec.engine == "persistent" else sampling.chain_one_block(V)
    dec.close()
    k = k1 + max(sampling.chain_persistent(V, GRID), sampling.chain_one_block(V))
    for backend, engine in modes:
        got = [np.load(tmp_path / f"{backend}_{engine}_rank{r}.npz") for r in range(world)]
        for g in got[1:]:  # bit-identical on every rank
            for name in ("ids", "rid", "rti", "rlp", "rtl", "score"):
                assert (np.asarray(g[name]).view(np.uint32) == np.asarray(got[0][name]).view(np.uint32)).all(), (
                    backend, engine, name)
        g = got[0]
        assert list(g["ids"]) == want_ids and (g["rid"] == want[0]).all() and (g["rti"] == want[2]).all(), (backend, engine)
        for a, b in ((g["rlp"], want[1]), (g["rtl"], want[3]), (g["score"], want_score)):
            b = np.asarray(b, np.float64)
            assert np.all(np.abs(np.asarray(a, np.float64) - b) <= sampling.logprob_bound(b, k, V)), (backend, engine)
