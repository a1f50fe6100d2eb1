"""A schedule-fuzzing model of the persistent megakernel's barrier-free hand-over protocol
(kuiperllama_b200/csrc/megakernel.cu; DESIGN.md section 5.2).

The kernel replaces grid barriers by tagged 64-bit words: a producer publishes {tag, value} with one
store, a consumer polls until the tag is the one it expects.  Which buffers may be single-slot, which
need two slots, and why the plain (untagged) residual-stream buffers can be double-buffered without any
barrier is an argument about ALL interleavings of 132 CTAs (x N ranks); a GPU test only ever sees a
few of them.  This test restates the protocol at the level of individual memory operations and runs it
under randomised, adversarial schedulers:

  * every CTA of every rank is a coroutine that yields before each load / store;
  * the scheduler picks who moves next (uniformly, or strongly favouring a few "fast" CTAs);
  * values are logical versions (token, layer, what), so a consumer can assert it read exactly the
    value the dataflow says it must -- a lost update, an early read or an overwritten slot fails.

Buffers, as in the kernel:  q|k|v, attention output, SwiGLU output h: single slot, tagged, local;
residual exchange (Wo / W2 partial sums): two slots alternating with the exchange index, tagged, written
into EVERY rank's area; residual stream x: two plain buffers alternating with the exchange index, each
CTA writes its slice after forming x = x_old + sum(partials); one grid barrier per token per rank.

Negative controls show the checker has teeth: a single-slot exchange and a single residual buffer must
both be caught.
"""
import random

import pytest


class ProtocolError(AssertionError):
    pass


def split(n_units, n_ctas, cta):
    """The kernel's contiguous split of a phase's units over the CTAs."""
    return range(cta * n_units // n_ctas, (cta + 1) * n_units // n_ctas)


class Rank:
    def __init__(self, cfg):
        c = cfg
        self.qkv = [(0, None)] * (c.heads * c.hq + 2 * c.kv_heads * c.hq)  # q | k | v, tagged, one slot
        self.attn = [(0, None)] * (c.heads * c.hq)
        self.h = [(0, None)] * c.ffn
        self.exch = [[[(0, None)] * c.dim for _ in range(c.world)] for _ in range(c.exch_slots)]
        self.x = [[None] * c.dim for _ in range(c.x_bufs)]
        self.barrier = 0


class Config:
    def __init__(self, world=1, ctas=4, heads=2, kv_heads=1, layers=2, tokens=3, exch_slots=2, x_bufs=2,
                 dim=None, ffn=None, cls_shard=False, prompt_tokens=0):
        self.world, self.ctas, self.heads, self.kv_heads = world, ctas, heads, kv_heads
        self.layers, self.tokens, self.exch_slots, self.x_bufs = layers, tokens, exch_slots, x_bufs
        # tensor parallel, classifier sharded by vocabulary: one more exchange per token (each rank
        # publishes its logits rows to every rank; a gather step polls them before the grid barrier),
        # which makes the number of exchanges per token ODD -- the slot parity flips from token to token
        self.cls_shard = cls_shard
        # the first `prompt_tokens` positions are prompt positions: the classifier is skipped (nobody
        # consumes the token's last W2 exchange), only the grid barrier that closes the token stays
        self.prompt_tokens = prompt_tokens
        self.exch_per_token = 2 * layers + (1 if cls_shard else 0)
        self.hq = 2  # elements per head
        # residual stream / FFN width; by default not a multiple of the CTA count on purpose.  Small
        # models have FEWER rows than the GPU has CTAs, so some CTAs own no rows of a phase at all.
        self.dim = dim or 2 * ctas + 1
        self.ffn = ffn or 3 * ctas - 1


def poll(buf, idx, tag, what):
    """Spin until buf[idx] carries `tag`; seeing a LATER tag means the value we need is gone."""
    while True:
        yield "load"
        t, v = buf[idx]
        if t == tag:
            return v
        if t > tag:
            raise ProtocolError(f"{what}[{idx}]: waiting for tag {tag}, slot already holds {t} (overwritten)")


def cta_program(cfg, ranks, r, c, stats):
    me = ranks[r]
    L, W, G = cfg.layers, cfg.world, cfg.ctas
    n_q = cfg.heads * cfg.hq
    n_kv = cfg.kv_heads * cfg.hq
    kv_mul = cfg.heads // cfg.kv_heads

    def x_version(tok, e):  # the residual stream after exchange e of token tok (e == -1: the embedding row)
        return ("x", tok, e)

    def stage_residual(tok, e):
        """Input staging of a phase that consumes the residual stream after exchange e (tp_in)."""
        tag = tok * cfg.exch_per_token + e + 1
        slot = tag % cfg.exch_slots
        mine = split(cfg.dim, G, c)
        for i in range(cfg.dim):
            if e >= 1:  # x_old is plain memory: no tag to wait for, the dataflow must already order it
                yield "load"
                old = me.x[(e - 1) % cfg.x_bufs][i]
                if old != x_version(tok, e - 1):
                    raise ProtocolError(f"rank {r} cta {c}: x_old[{i}] for exchange {e} of token {tok} is {old}")
            for src in range(W):
                v = yield from poll(me.exch[slot][src], i, tag, f"rank {r} exchange {e} from rank {src}")
                if v != ("partial", tok, e, src):
                    raise ProtocolError(f"rank {r} cta {c}: exchange {e} element {i} holds {v}")
            if i in mine:
                yield "store"
                me.x[e % cfg.x_bufs][i] = x_version(tok, e)
        stats["staged"] += 1

    def publish_exchange(tok, e):
        tag = tok * cfg.exch_per_token + e + 1
        slot = tag % cfg.exch_slots
        for i in split(cfg.dim, G, c):
            for k in range(1, W + 1):  # every rank's area, own last
                dst = ranks[(r + k) % W]
                yield "store"
                dst.exch[slot][r][i] = (tag, ("partial", tok, e, r))

    for tok in range(cfg.tokens):
        for l in range(L):
            hand = tok * 3 * L + 3 * l + 1  # tags of the three local hand-offs of this layer
            # ---- QKV: consumes x after the previous layer's W2 exchange, publishes q | k | v
            if l > 0:
                yield from stage_residual(tok, 2 * l - 1)
            for u in split(n_q + 2 * n_kv, G, c):
                yield "store"
                me.qkv[u] = (hand, ("qkv", tok, l, u))
            # ---- attention: one head per CTA, the others go straight on
            if c < cfg.heads:
                kvh = c // kv_mul
                need = list(range(c * cfg.hq, (c + 1) * cfg.hq))
                need += [n_q + kvh * cfg.hq + j for j in range(cfg.hq)]
                need += [n_q + n_kv + kvh * cfg.hq + j for j in range(cfg.hq)]
                for u in need:
                    v = yield from poll(me.qkv, u, hand, f"rank {r} q|k|v")
                    if v != ("qkv", tok, l, u):
                        raise ProtocolError(f"attention read {v}")
                for j in range(cfg.hq):
                    yield "store"
                    me.attn[c * cfg.hq + j] = (hand + 1, ("attn", tok, l))
            # ---- Wo: consumes the attention output, publishes exchange 2l
            for u in range(n_q):
                v = yield from poll(me.attn, u, hand + 1, f"rank {r} attention output")
                if v != ("attn", tok, l):
                    raise ProtocolError(f"Wo read {v}")
            yield from publish_exchange(tok, 2 * l)
            # ---- W1|W3: consumes x after exchange 2l, publishes h
            yield from stage_residual(tok, 2 * l)
            for u in split(cfg.ffn, G, c):
                yield "store"
                me.h[u] = (hand + 2, ("h", tok, l))
            # ---- W2: consumes h, publishes exchange 2l+1
            for u in range(cfg.ffn):
                v = yield from poll(me.h, u, hand + 2, f"rank {r} h")
                if v != ("h", tok, l):
                    raise ProtocolError(f"W2 read {v}")
            yield from publish_exchange(tok, 2 * l + 1)
        # ---- classifier: consumes x after the last exchange; then the one grid barrier of the token
        if tok >= cfg.prompt_tokens:
            yield from stage_residual(tok, 2 * L - 1)
        if cfg.cls_shard and tok >= cfg.prompt_tokens:
            # this rank's logits rows (the model reuses `dim` as the rows per rank) go to every rank as
            # exchange 2L; the gather splits the world x dim words of the local area over the CTAs
            yield from publish_exchange(tok, 2 * L)
            tag = tok * cfg.exch_per_token + 2 * L + 1
            slot = tag % cfg.exch_slots
            for i in split(W * cfg.dim, G, c):
                src, j = divmod(i, cfg.dim)
                v = yield from poll(me.exch[slot][src], j, tag, f"rank {r} logits of rank {src}")
                if v != ("partial", tok, 2 * L, src):
                    raise ProtocolError(f"rank {r} cta {c}: logit {i} holds {v}")
        yield "store"
        me.barrier += 1
        while me.barrier < (tok + 1) * G:
            yield "load"
    stats["finished"] += 1


def run(cfg, seed, fast_bias):
    rng = random.Random(seed)
    ranks = [Rank(cfg) for _ in range(cfg.world)]
    stats = {"staged": 0, "finished": 0}
    procs = [cta_program(cfg, ranks, r, c, stats) for r in range(cfg.world) for c in range(cfg.ctas)]
    alive = list(range(len(procs)))
    fast = set(rng.sample(alive, max(1, len(alive) // 3)))
    idle = 0
    while alive:
        if fast_bias and rng.random() < fast_bias:
            pool = [p for p in alive if p in fast] or alive
        else:
            pool = alive
        p = rng.choice(pool)
        try:
            op = next(procs[p])
        except StopIteration:
            alive.remove(p)
            idle = 0
            continue
        idle = 0 if op == "store" else idle + 1
        if idle > 20000 * len(procs):
            raise ProtocolError("no CTA has stored anything for a long time: deadlock")
    assert stats["finished"] == cfg.world * cfg.ctas
    return stats


CONFIGS = {
    "1 rank, every CTA a head": Config(world=1, ctas=2, heads=2, kv_heads=1),
    "1 rank, more CTAs than heads": Config(world=1, ctas=5, heads=2, kv_heads=1),
    "1 rank, grouped kv heads": Config(world=1, ctas=6, heads=4, kv_heads=2, layers=3),
    "2 ranks": Config(world=2, ctas=4, heads=2, kv_heads=2, tokens=3),
    "3 ranks, long run": Config(world=3, ctas=3, heads=2, kv_heads=1, layers=2, tokens=4),
    # tiny models on a big GPU: most CTAs own no q|k|v row, some no row of the residual stream either
    "1 rank, more CTAs than rows": Config(world=1, ctas=12, heads=2, kv_heads=1, dim=7, ffn=9),
    "2 ranks, more CTAs than rows": Config(world=2, ctas=9, heads=2, kv_heads=2, dim=5, ffn=11, tokens=2),
    # classifier sharded by vocabulary: an odd number of exchanges per token
    "2 ranks, sharded classifier": Config(world=2, ctas=4, heads=2, kv_heads=2, tokens=4, cls_shard=True),
    "3 ranks, sharded classifier, one layer": Config(world=3, ctas=3, heads=2, kv_heads=1, layers=1, tokens=4, cls_shard=True),
    "2 ranks, sharded classifier, more CTAs than rows": Config(world=2, ctas=9, heads=2, kv_heads=2, dim=5, ffn=11,
                                                               tokens=3, cls_shard=True),
    # a prompt in one launch: classifier skipped for its positions (kllm_decoder_prompt)
    "1 rank, prompt positions": Config(world=1, ctas=5, heads=2, kv_heads=1, tokens=5, prompt_tokens=3),
    "2 ranks, sharded classifier, prompt positions": Config(world=2, ctas=4, heads=2, kv_heads=2, tokens=5,
                                                            cls_shard=True, prompt_tokens=3),
    "2 ranks, sharded classifier, prompt positions, more CTAs than rows":
        Config(world=2, ctas=9, heads=2, kv_heads=2, dim=5, ffn=11, tokens=4, cls_shard=True, prompt_tokens=2),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_protocol_survives_random_and_adversarial_schedules(name):
    cfg = CONFIGS[name]
    for seed in range(12):
        for bias in (0.0, 0.9, 0.99):
            run(cfg, seed, bias)


def _must_fail(cfg, what):
    caught = 0
    for seed in range(24):
        for bias in (0.0, 0.9, 0.99):
            try:
                run(cfg, seed, bias)
            except ProtocolError:
                caught += 1
    assert caught > 0, f"the checker did not notice {what}"


def test_checker_catches_a_single_slot_exchange():
    """With ONE exchange slot a fast CTA's Wo partials of the next layer overwrite W2 partials that a
    slower CTA is still polling.  (That needs a CTA nobody waits for between the two exchanges: one
    that owns no q|k|v row -- the small-model case.  When every CTA owns q|k|v rows, attention already
    orders everybody, and the second slot is merely conservative.)"""
    _must_fail(Config(world=1, ctas=12, heads=2, kv_heads=1, dim=7, ffn=9, exch_slots=1), "a single-slot exchange")
    _must_fail(Config(world=2, ctas=9, heads=2, kv_heads=2, dim=5, ffn=11, tokens=2, exch_slots=1),
               "a single-slot exchange across ranks")
    _must_fail(Config(world=2, ctas=9, heads=2, kv_heads=2, dim=5, ffn=11, tokens=3, exch_slots=1, cls_shard=True),
               "a single-slot exchange with the sharded classifier")


def test_checker_catches_a_single_residual_buffer():
    """With ONE residual buffer a CTA that finished staging overwrites x_old under a slower one."""
    _must_fail(Config(world=1, ctas=5, heads=2, kv_heads=1, x_bufs=1), "a single residual buffer")


# ---- the graph engine's one-shot all-reduce (csrc/tp_comm.cu allreduce_oneshot_kernel) --------------------

def _oneshot_rank(world, r, mem, flags, calls, slots):
    """Call n: store my vector into every rank's slot (n % slots) row r, then publish flag n there
    (the kernel: plain stores, __threadfence_system, st.release.sys); wait for every rank's flag n in my
    own memory; read all rows.  No other synchronisation between calls."""
    for n in range(1, calls + 1):
        s = n % slots
        for k in range(1, world + 1):
            dst = (r + k) % world
            for i in range(3):
                yield "store"
                mem[dst][s][r][i] = (n, r, i)
            yield "store"
            flags[dst][s][r] = n
        for src in range(world):
            while True:
                yield "load"
                f = flags[r][s][src]
                if f == n:
                    break
                if f > n:
                    raise ProtocolError(f"rank {r}: flag of rank {src} is already {f} while waiting for call {n}")
        for src in range(world):
            for i in range(3):
                yield "load"
                if mem[r][s][src][i] != (n, src, i):
                    raise ProtocolError(f"rank {r} call {n}: row of rank {src} holds {mem[r][s][src][i]}")


def _run_oneshot(world, slots, seed, bias):
    rng = random.Random(seed)
    mem = [[[[None] * 3 for _ in range(world)] for _ in range(slots)] for _ in range(world)]
    flags = [[[0] * world for _ in range(slots)] for _ in range(world)]
    procs = {r: _oneshot_rank(world, r, mem, flags, 12, slots) for r in range(world)}
    fast = rng.randrange(world)
    steps = 0
    while procs:
        r = fast if (fast in procs and rng.random() < bias) else rng.choice(list(procs))
        try:
            next(procs[r])
        except StopIteration:
            del procs[r]
        steps += 1
        assert steps < 2_000_000, "deadlock"


@pytest.mark.parametrize("world", [2, 4])
def test_oneshot_allreduce_slots_and_flags(world):
    for seed in range(20):
        for bias in (0.0, 0.9, 0.99):
            _run_oneshot(world, 2, seed, bias)
    caught = 0
    for seed in range(20):
        for bias in (0.0, 0.9, 0.99):
            try:
                _run_oneshot(world, 1, seed, bias)  # one slot: the next call's stores land under a reader
            except ProtocolError:
                caught += 1
    assert caught > 0
