"""Schedule-fuzzing model of how a stoppable megakernel run ends (csrc/megakernel.cu, kllm_decoder_generate_until).

The producer warp streams ring stages on its own and runs ahead of the consumer warps, across the token
boundary.  A run that stops after token j therefore finds the producer somewhere in token j + 1 or later: it
may have issued stages nobody will read, it may be blocked on the `empty` barrier of a slot nobody will free,
or it may wait for the grid barrier of token j + 1, which nobody will reach.  The kernel's protocol:

* After the token's last grid barrier every consumer warp knows the same id, so all of them stop on the same
  token.  They set a CTA-local stop flag.
* The producer checks the flag while it waits on `empty` and while it waits for a grid barrier; once it sees it
  it issues nothing more and publishes its final ring position.
* Each consumer warp waits on `full` for every fill up to that position (the drain), then exits.  The bulk
  copies land in shared memory, so the CTA may not exit while one is in flight.

The model runs that protocol under random and adversarial schedules, with copies that land at random later
times, and fails on a warp that can wait forever, a stage refilled while it is still being read, or a CTA that
exits with a fill in flight.  Two negative controls -- consumers that exit without the drain, and a producer
that does not look at the flag while it waits -- must be caught.
"""
import random

import pytest


class ProtocolError(AssertionError):
    pass


class MBarrier:
    """Phase-counting barrier; waiters may only ask about the parity of the last completed phase."""

    def __init__(self, arrivals):
        self.arrivals, self.pending, self.completed = arrivals, arrivals, 0

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.completed += 1
            self.pending = self.arrivals

    def test_wait(self, parity):
        return ((self.completed - 1) & 1) == parity


class Cta:
    def __init__(self, W, S, schedule):
        self.W, self.S, self.schedule = W, S, schedule  # schedule[t] = list of stage kinds ("w" | "kv")
        self.full = [MBarrier(1) for _ in range(S)]
        self.empty = [MBarrier(W) for _ in range(S)]
        self.stage_data = [None] * S
        self.reading = [set() for _ in range(S)]
        self.in_flight = []  # (fill number, slot) issued, not landed
        self.barriers_passed = 0  # grid barriers (one per token in the model) every warp has passed
        self.at_barrier = 0
        self.stop = False
        self.prod_end = None  # (slot, parity) published by the producer when it is done


def advance(slot, parity, S):
    slot += 1
    if slot == S:
        return 0, parity ^ 1
    return slot, parity


def producer(c, check_flag):
    slot, parity, n = 0, 0, 0
    for t, stages in enumerate(c.schedule):
        for kind in stages:
            if kind == "kv" and t > 0:
                # KV rows of token t - 1 are final once that token's grid barrier is passed
                while c.barriers_passed < t:
                    if check_flag and c.stop:
                        c.prod_end = (slot, parity)
                        return
                    yield "wait"
            while not c.empty[slot].test_wait(parity ^ 1):
                if check_flag and c.stop:
                    c.prod_end = (slot, parity)
                    return
                yield "wait"
            if c.reading[slot]:
                raise ProtocolError(f"fill {n} issued into stage {slot} while warps {sorted(c.reading[slot])} read it")
            c.in_flight.append((n, slot))  # expect_tx + bulk copy: lands later (dma)
            yield "issue"
            n += 1
            slot, parity = advance(slot, parity, c.S)
    c.prod_end = (slot, parity)


def dma(c, rng):
    while True:
        if c.in_flight and rng.random() < 0.5:
            n, slot = c.in_flight.pop(rng.randrange(len(c.in_flight)) if rng.random() < 0.3 else 0)
            if c.reading[slot]:
                raise ProtocolError(f"fill {n} lands in stage {slot} while warps {sorted(c.reading[slot])} read it")
            c.stage_data[slot] = n
            c.full[slot].arrive()  # complete_tx
        yield "dma"


def consumer(c, w, stop_token, drain):
    slot, parity, n = 0, 0, 0
    for t, stages in enumerate(c.schedule):
        for _ in stages:
            while not c.full[slot].test_wait(parity):
                yield "wait"
            c.reading[slot].add(w)
            yield "read"
            if c.stage_data[slot] != n:
                raise ProtocolError(f"warp {w} expected fill {n} in stage {slot}, found {c.stage_data[slot]}")
            c.reading[slot].discard(w)
            c.empty[slot].arrive()
            n += 1
            slot, parity = advance(slot, parity, c.S)
        # the token's last grid barrier: every warp arrives, then the id is known
        c.at_barrier += 1
        while c.at_barrier < c.W * (t + 1):
            yield "wait"
        c.barriers_passed = t + 1
        if t == stop_token:
            c.stop = True
            if not drain:
                return
            while c.prod_end is None:
                yield "wait"
            while (slot, parity) != c.prod_end:
                while not c.full[slot].test_wait(parity):
                    yield "wait"
                slot, parity = advance(slot, parity, c.S)
            return


def progress_possible(procs, dma_proc, c):
    """A long run of waits under a biased schedule may just be starvation: land every copy in flight, then
    give every warp a few fair turns.  If none of them gets past a wait, none ever will."""
    while c.in_flight:
        next(dma_proc)
    for _ in range(4):
        for k in list(procs):
            try:
                if next(procs[k]) != "wait":
                    return True
            except StopIteration:
                del procs[k]
                return True
    return False


def run(W, S, schedule, stop_token, seed, bias, drain=True, check_flag=True):
    rng = random.Random(seed)
    c = Cta(W, S, schedule)
    procs = {"p": producer(c, check_flag)}
    for w in range(W):
        procs[w] = consumer(c, w, stop_token, drain)
    dma_proc = dma(c, rng)
    fast = rng.choice(list(procs))
    slow = rng.choice([k for k in procs if k != fast])
    idle = 0
    while procs:
        if rng.random() < 0.3:
            next(dma_proc)
        keys = list(procs)
        if rng.random() < bias and fast in procs:
            k = fast
        else:
            k = rng.choice([x for x in keys if x != slow] or keys) if rng.random() < bias else rng.choice(keys)
        try:
            op = next(procs[k])
        except StopIteration:
            del procs[k]
            idle = 0
            continue
        idle = idle + 1 if op == "wait" else 0
        if idle > 2000 and not progress_possible(procs, dma_proc, c):
            raise ProtocolError(f"warps {sorted(map(str, procs))} wait forever")
        if idle > 2000:
            idle = 0
    if c.in_flight:
        raise ProtocolError(f"the CTA exits with fills {c.in_flight} in flight")


def schedules(rng, n):
    """Token schedules: weight stages, and KV stages that wait for the previous token's barrier; tokens with
    fewer stages than the ring is deep let the producer run more than one token ahead."""
    out = []
    for _ in range(n):
        tokens = rng.randint(2, 6)
        sched = []
        for _ in range(tokens):
            k = rng.randint(1, 9)
            sched.append([rng.choice(["w", "w", "kv"]) for _ in range(k)])
        out.append(sched)
    return out


@pytest.mark.parametrize("W,S", [(8, 6), (8, 2), (4, 3), (3, 16), (2, 1)])
def test_stop_and_drain_is_safe(W, S):
    rng = random.Random(W * 100 + S)
    for i, sched in enumerate(schedules(rng, 12)):
        for stop_token in range(len(sched)):
            for bias in (0.0, 0.8, 0.97):
                run(W, S, sched, stop_token, seed=i * 31 + stop_token, bias=bias)


def test_a_run_without_a_stop_ends_cleanly():
    rng = random.Random(7)
    for i, sched in enumerate(schedules(rng, 20)):
        for bias in (0.0, 0.9):
            run(4, 3, sched, stop_token=None, seed=i, bias=bias)


def test_adversarial_producer_far_ahead():
    """The producer runs first until it blocks: it holds S issued stages of the next tokens, waits on a slot
    and on a barrier that never come."""
    sched = [["w"] * 3, ["w", "kv"], ["kv", "w"], ["w"] * 5]
    for stop_token in range(len(sched)):
        for seed in range(20):
            run(4, 4, sched, stop_token, seed=seed, bias=0.999)


def test_exit_without_drain_is_caught():
    caught = 0
    rng = random.Random(3)
    for i, sched in enumerate(schedules(rng, 20)):
        for bias in (0.0, 0.9, 0.999):
            try:
                run(4, 4, sched, stop_token=0, seed=i, bias=bias, drain=False)
            except ProtocolError as e:
                assert "in flight" in str(e) or "read" in str(e), e
                caught += 1
    assert caught > 0


def test_producer_that_ignores_the_flag_hangs():
    caught = 0
    sched = [["w"] * 2, ["w"] * 2, ["kv"] * 2, ["w"] * 6]
    for seed in range(10):
        try:
            run(4, 3, sched, stop_token=0, seed=seed, bias=0.9, check_flag=False)
        except ProtocolError as e:
            assert "forever" in str(e), e
            caught += 1
    assert caught == 10
