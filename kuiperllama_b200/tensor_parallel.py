"""Tensor-parallel decode (SURVEY.md section 8e): heads and FFN columns sharded over N GPUs, one
process per GPU, exactly two all-reduces per layer (after o_proj, after down_proj).

The reference is single-GPU (llama3.cpp:118 pins device 0), so this file defines the sharding:

  column-parallel (split OUTPUT ROWS of the [out, in] matrices): wq by head, wk / wv by kv head,
      w1 / w3 by FFN row; each rank keeps only its kv heads' cache and runs RoPE + attention for
      its own heads;
  row-parallel (split INPUT COLUMNS, repacked contiguous): wo[:, my heads], w2[:, my FFN rows];
      each rank produces a full-length partial sum that meets in the all-reduce;
  replicated: embedding, norm weights, classifier; the residual stream x is bit-identical on
      every rank because every rank sums the partials in rank order.
  GQA models with fewer kv heads than ranks (TinyLlama: 4) replicate each kv head over the
      ranks that share it.

Sharding is plain indexing and works on numpy arrays and torch tensors alike (the world_size-2
gloo tests run it on CPU); rendezvous uses torch.distributed as plumbing; the exchange itself is
kllm_comm (csrc/tp_comm.cu).
"""
from __future__ import annotations

import ctypes
import os
from dataclasses import replace

from . import KllmError, check, load_library
from .decoder import Decoder, ModelShape

COMM_BACKENDS = {"peer": 0, "nccl": 1}


def kv_heads_of_rank(shape: ModelShape, tp: int, rank: int) -> range:
    """Global kv-head indices rank `rank` owns (a single, shared one when kv_head_num < tp)."""
    if shape.kv_head_num >= tp:
        n = shape.kv_head_num // tp
        return range(rank * n, (rank + 1) * n)
    first_q = rank * (shape.head_num // tp)
    kv = first_q // shape.kv_mul
    return range(kv, kv + 1)


# int8 FFN shards are cut in units of 256 columns: whole quantisation groups (64) AND 16-byte rows of
# group scales per shard, which is what the persistent engine's TMA ring can stage
INT8_FFN_UNIT = 256


def ffn_range(shape: ModelShape, tp: int, rank: int) -> range:
    """FFN rows (w1 / w3 output rows = w2 input columns) rank `rank` owns.  fp32: equal slices.
    int8: multiples of INT8_FFN_UNIT, spread as evenly as they go (Llama-2-7B: 11008 = 43 units ->
    5632 + 5376 at tp 2), so ranks may differ by one unit."""
    h = shape.hidden_dim
    if not shape.group_size:
        n = h // tp
        return range(rank * n, (rank + 1) * n)
    units = h // INT8_FFN_UNIT
    base, extra = divmod(units, tp)
    start = rank * base + min(rank, extra)
    return range(start * INT8_FFN_UNIT, (start + base + (1 if rank < extra else 0)) * INT8_FFN_UNIT)


def check_shardable(shape: ModelShape, tp: int) -> None:
    s = shape
    if tp < 1 or s.head_num % tp:
        raise KllmError(f"{s.name}: {s.head_num} heads do not split {tp} ways")
    if s.group_size:
        if s.hidden_dim % INT8_FFN_UNIT or s.hidden_dim // INT8_FFN_UNIT < tp:
            raise KllmError(f"{s.name}: int8 hidden_dim {s.hidden_dim} does not split {tp} ways in units of "
                            f"{INT8_FFN_UNIT} columns")
    elif s.hidden_dim % tp:
        raise KllmError(f"{s.name}: hidden {s.hidden_dim} does not split {tp} ways")
    if s.kv_head_num >= tp:
        if s.kv_head_num % tp:
            raise KllmError(f"{s.name}: {s.kv_head_num} kv heads do not split {tp} ways")
    elif tp % s.kv_head_num or (s.head_num // tp) > s.kv_mul or s.kv_mul % (s.head_num // tp):
        raise KllmError(f"{s.name}: cannot replicate {s.kv_head_num} kv heads over {tp} ranks")
    if not s.group_size and (s.hidden_dim // tp) % 4:
        raise KllmError(f"{s.name}: hidden_dim/{tp} must be a multiple of 4")
    if s.group_size and (s.head_num // tp * s.head_size) % s.group_size:
        raise KllmError(f"{s.name}: int8 groups of {s.group_size} straddle the {tp}-way split of the "
                        f"attention columns ({s.head_num // tp * s.head_size} per rank)")


def local_shape(shape: ModelShape, tp: int, rank: int = 0) -> ModelShape:
    """The LOCAL counts kllm_decoder_desc wants under tensor parallelism; `dim` stays the full
    model dim (include/kllm_b200.h, tp fields)."""
    check_shardable(shape, tp)
    return replace(shape, name=f"{shape.name}[tp{tp}]", head_num=shape.head_num // tp,
                   kv_head_num=len(kv_heads_of_rank(shape, tp, rank)), hidden_dim=len(ffn_range(shape, tp, rank)))


def comm_words(shape: ModelShape, world: int) -> int:
    """max_count for Comm / kllm_comm_create: the residual exchange needs `dim` words per rank; with
    room for vocab / world more, the persistent engine shards the classifier by vocabulary."""
    per_rank = -(-shape.vocab_size // max(world, 1))
    return max(shape.dim, per_rank if shape.vocab_size % max(world, 1) == 0 else 0)


def weight_bytes_per_token_per_gpu(shape: ModelShape, tp: int, rank: int = 0, classifier_rows: int | None = None) -> int:
    """ALGORITHMIC bytes ONE rank streams per decode step: its shard of every layer matmul
    (+ int8 scales), its classifier rows (`classifier_rows`: Decoder.classifier_rows; default all,
    i.e. replicated) plus what is replicated (norm vectors, one embedding row)."""
    if tp == 1:
        return shape.weight_bytes_per_token()
    s = shape
    d, L, V, hs = s.dim, s.layer_num, s.vocab_size, s.head_size
    if classifier_rows:
        V = classifier_rows
    kv_rows = len(kv_heads_of_rank(s, tp, rank)) * hs
    numel = L * (2 * d * d // tp + 2 * kv_rows * d + 3 * len(ffn_range(s, tp, rank)) * d) + V * d
    wbytes = numel * 4 if s.group_size == 0 else numel + numel // s.group_size * 4
    extra = (2 * L + 1) * d * 4 + d * 4
    if s.flavour == "qwen2" and s.group_size == 0:
        extra += L * (d // tp + 2 * kv_rows) * 4
    return wbytes + extra


def _contig(a):
    return a.contiguous() if hasattr(a, "contiguous") else __import__("numpy").ascontiguousarray(a)


def shard_weights(shape: ModelShape, w: dict, tp: int, rank: int) -> dict:
    """Rank `rank`'s shard of a full weight dict (keys of synth_weights / read_checkpoint)."""
    check_shardable(shape, tp)
    s = shape
    hs, g = s.head_size, s.group_size
    q0, q1 = rank * (s.head_num // tp) * hs, (rank + 1) * (s.head_num // tp) * hs
    kvh = kv_heads_of_rank(s, tp, rank)
    k0, k1 = kvh.start * hs, kvh.stop * hs
    ffn = ffn_range(s, tp, rank)
    f0, f1 = ffn.start, ffn.stop
    out = {k: w[k] for k in ("tok_emb", "attn_norm", "ffn_norm", "final_norm", "wcls") if k in w}
    rows = {"wq": (q0, q1), "wk": (k0, k1), "wv": (k0, k1), "w1": (f0, f1), "w3": (f0, f1)}
    cols = {"wo": (q0, q1), "w2": (f0, f1)}
    for name, (a, b) in rows.items():
        out[name] = _contig(w[name][:, a:b, :])
        if g:  # scales follow the flattened row-major order: [L, rows * in/g]
            sc = w["s" + name[1:]]
            per_row = w[name].shape[2] // g
            out["s" + name[1:]] = _contig(sc.reshape(s.layer_num, -1, per_row)[:, a:b, :].reshape(s.layer_num, -1))
    for name, (a, b) in cols.items():
        out[name] = _contig(w[name][:, :, a:b])
        if g:
            sc = w["s" + name[1:]]
            per_row = w[name].shape[2] // g
            out["s" + name[1:]] = _contig(
                sc.reshape(s.layer_num, w[name].shape[1], per_row)[:, :, a // g:b // g].reshape(s.layer_num, -1))
    if g:
        out["scls"] = w["scls"]
    for bias, (a, b) in (("bq", (q0, q1)), ("bk", (k0, k1)), ("bv", (k0, k1))):
        if bias in w:
            out[bias] = _contig(w[bias][:, a:b])
    return out


class Comm:
    """A kllm_comm plus its rendezvous over an initialised torch.distributed process group."""

    def __init__(self, max_count: int, backend: str | None = None, group=None):
        import torch
        import torch.distributed as dist
        self.lib = load_library()
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        backend = backend or os.environ.get("KLLM_TP_COMM", "peer")
        if backend not in COMM_BACKENDS:
            raise KllmError(f"KLLM_TP_COMM={backend!r}: expected one of {sorted(COMM_BACKENDS)}")
        self.backend, self.group, self._dist = backend, group, dist
        self.handle = ctypes.c_void_p()
        max_count = (max_count + 3) // 4 * 4
        if backend == "nccl":
            ident = [None]
            if self.rank == 0:
                buf = (ctypes.c_ubyte * 128)()
                check(self.lib.kllm_comm_unique_id(buf), "kllm_comm_unique_id")
                ident = [bytes(buf)]
            dist.broadcast_object_list(ident, src=0, group=group)
            check(self.lib.kllm_comm_create(self.world, self.rank, 1, max_count, ident[0],
                                            ctypes.byref(self.handle)), "kllm_comm_create(nccl)")
        else:
            check(self.lib.kllm_comm_create(self.world, self.rank, 0, max_count, None,
                                            ctypes.byref(self.handle)), "kllm_comm_create(peer)")
            mine = (ctypes.c_ubyte * 64)()
            if self.world > 1:
                check(self.lib.kllm_comm_ipc_handle(self.handle, mine), "kllm_comm_ipc_handle")
            handles = [None] * self.world
            dist.all_gather_object(handles, bytes(mine), group=group)
            check(self.lib.kllm_comm_connect(self.handle, b"".join(handles)), "kllm_comm_connect")
        torch.cuda.synchronize()
        dist.barrier(group=group)  # every rank has mapped every peer before the first exchange

    def allreduce_(self, t, residual=None, stream=None):
        """In-place test hook: t <- (residual or 0) + sum over ranks of t."""
        check(self.lib.kllm_comm_allreduce_residual(
            self.handle, t.data_ptr(), residual.data_ptr() if residual is not None else None,
            t.data_ptr(), t.numel(), stream), "kllm_comm_allreduce_residual")
        return t

    def close(self):
        if getattr(self, "handle", None):
            import torch
            torch.cuda.synchronize()
            self._dist.barrier(group=self.group)  # nobody frees while a peer may still push
            self.lib.kllm_comm_destroy(self.handle)
            self.handle = None


def make_tp_decoder(shape: ModelShape, full_weights: dict, comm: Comm, stream=None, numerics="exact",
                    kv_cache="fp32", weight_format="fp32") -> Decoder:
    """Decoder for this rank's shard of `full_weights` (every rank passes the same full dict,
    e.g. synth_weights with the same seed; the shard is cut here and the rest can be freed).
    A bf16 or fp8 KV cache and bf16 weights run on one GPU only (kllm_decoder_desc::kv_cache, ::weights)."""
    tp, rank = comm.world, comm.rank
    if tp == 1:
        return Decoder(shape, full_weights, stream=stream, numerics=numerics, kv_cache=kv_cache,
                       weight_format=weight_format)
    if kv_cache != "fp32":
        raise ValueError(f"kv_cache={kv_cache!r} is not supported under tensor parallelism (tp_size {tp})")
    if weight_format != "fp32":
        raise ValueError(f"weight_format={weight_format!r} is not supported under tensor parallelism (tp_size {tp})")
    shard = shard_weights(shape, full_weights, tp, rank)
    return Decoder(local_shape(shape, tp, rank), shard, stream=stream, tp_size=tp, tp_rank=rank,
                   comm=comm, full_dim=shape.dim, numerics=numerics)
