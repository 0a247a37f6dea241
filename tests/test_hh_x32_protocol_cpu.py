"""CPU model check of the synchronisation protocol of hk_update_R_x32 (fplll_b200/csrc/hh_api.cu): producer lanes, update
warps and the chain warp talk through mbarriers whose waits only see the PARITY of a phase, so a waiter that falls two
completions behind (or runs two ahead) of a barrier passes or blocks wrongly.  That is not a theoretical worry: a ring of 13
TMA stages with 4 product slots passed the small GPU parity tests and hung at n = 400.

The model below replays the kernel's three loops as coroutines over the same chunk sequence (XmIter), with the barrier
semantics of PTX (`mbarrier.try_wait.parity P` succeeds iff the phase in progress has the other parity; a count-1 barrier
advances one phase per arrive), under many random interleavings and TMA landing delays, and checks at every step that
  * an update warp only reads a stage that holds the chunk it is about to process,
  * a product slot is only overwritten after the chain warp has consumed its previous content,
  * the chain warp consumes the chunks in order and sees the products of the right chunk,
  * everybody terminates.
The ring sizes are read from the source, so a change of the constants is checked before it ever reaches a GPU."""
import os
import random
import re

import pytest

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fplll_b200", "csrc", "hh_api.cu")


def source_constants():
    text = open(SRC).read()
    get = lambda name: int(re.search(r"constexpr int %s\s*=\s*(\d+);" % name, text).group(1))
    return dict(NA=get("XM_NA"), S=get("XM_S"), PR=get("XM_PR"), K=get("X_K"))


def chunk_sequence(n, i, K):
    """XmIter: pass q = 0 loads R_i; pass q >= 1 is reflection j = q - 2, k0 from (max(j, 0) & ~(K-1)) in steps of K."""
    seq, q, k0 = [], 0, 0
    while q <= i + 1:
        seq.append((q, k0, k0 + K >= n))
        k0 += K
        if k0 >= n:
            q += 1
            k0 = max(q - 2, 0) & ~(K - 1)
    return seq


class Bar:
    """count-1 mbarrier: `phase` = index of the phase in progress"""

    def __init__(self):
        self.phase = 0

    def arrive(self):
        self.phase += 1

    def test(self, parity):
        return (self.phase & 1) != parity


class Violation(Exception):
    pass


def simulate(n, i, NA, S, PR, K, seed, max_steps=2_000_000):
    rng = random.Random(seed)
    seq = chunk_sequence(n, i, K)
    G = len(seq)
    full, empty = [Bar() for _ in range(S)], [Bar() for _ in range(S)]
    pready, pfree = [Bar() for _ in range(PR)], [Bar() for _ in range(PR)]
    state = dict(pass_done=0)
    stage = [None] * S   # chunk whose data the stage holds
    slot = [None] * PR   # chunk whose products the slot holds
    slot_consumed = [True] * PR
    landing = []         # (stage, chunk) issued, not landed yet

    def producer(p):
        g = p
        while g < G:
            while not empty[p].test(((g // S) & 1) ^ 1):
                yield
            landing.append((p, g))  # lands at some later step (land() below arrives on full[p])
            g += S
            yield

    def update(me):
        fq = 0
        for g in range(me, G, NA):
            q = seq[g][0]
            if q >= 1 and fq < q:
                while state["pass_done"] < q:
                    yield
                fq = q
            while not pfree[g % PR].test(((g // PR) & 1) ^ 1):
                yield
            while not full[g % S].test((g // S) & 1):
                yield
            if stage[g % S] != g:
                raise Violation("update warp %d: stage %d holds chunk %r, wanted %d" % (me, g % S, stage[g % S], g))
            yield  # ... computing ...
            if not slot_consumed[g % PR]:
                raise Violation("update warp %d overwrites product slot %d (chunk %r not consumed) with chunk %d"
                                % (me, g % PR, slot[g % PR], g))
            slot[g % PR], slot_consumed[g % PR] = g, False
            yield
            pready[g % PR].arrive()
            empty[g % S].arrive()
            yield

    def chain():
        for g in range(G):
            while not pready[g % PR].test((g // PR) & 1):
                yield
            if slot[g % PR] != g:
                raise Violation("chain warp: slot %d holds chunk %r, wanted %d" % (g % PR, slot[g % PR], g))
            slot_consumed[g % PR] = True
            yield
            pfree[g % PR].arrive()
            if seq[g][2]:
                state["pass_done"] = seq[g][0] + 1
            yield

    agents = [producer(p) for p in range(min(S, G))] + [update(w) for w in range(NA)] + [chain()]
    alive = list(range(len(agents)))
    asleep = {}  # agent -> step it wakes up at: warps are descheduled for long stretches on real hardware
    for step in range(max_steps):
        if not alive:
            return G
        # a pending TMA box lands (any order: different stages are independent copies)
        if landing and rng.random() < 0.3:
            st, g = landing.pop(rng.randrange(len(landing)))
            stage[st] = g
            full[st].arrive()
            continue
        awake = [a for a in alive if asleep.get(a, 0) <= step]
        if not awake:
            continue
        a = rng.choice(awake)
        if rng.random() < 0.01:
            asleep[a] = step + rng.randrange(50, 1500)
            continue
        try:
            next(agents[a])
        except StopIteration:
            alive.remove(a)
    raise Violation("no progress: deadlock or livelock with %d agents left" % len(alive))


@pytest.mark.parametrize("n,i", [(40, 39), (64, 20), (100, 99), (50, 33), (400, 10)])
def test_shipped_ring_sizes_are_safe(n, i):
    c = source_constants()
    assert c["NA"] <= c["PR"] <= c["S"], c  # the static_asserts of hh_api.cu
    for seed in range(25):
        assert simulate(n, i, c["NA"], c["S"], c["PR"], c["K"], seed) > 0


def test_the_model_finds_the_configuration_that_hung_on_the_gpu():
    """13 stages, 4 product slots, 6 update warps: a warp gets two rounds of a product slot ahead of the chain warp.  It
    takes passes longer than the lag (25 chunks at n = 400; the pass counter stops a warp at every pass boundary), which is
    why the small parity tests passed."""
    hits = 0
    for seed in range(40):
        try:
            simulate(400, 10, 6, 13, 4, 16, seed)
        except Violation:
            hits += 1
    assert hits > 0


@pytest.mark.parametrize("NA,S,PR", [(6, 12, 6), (4, 13, 4), (6, 8, 8)])
def test_deeper_rings_that_respect_the_constraint_are_safe(NA, S, PR):
    """more bytes in flight than the shipped ring, within XM_NA <= XM_PR <= XM_S"""
    for seed in range(15):
        assert simulate(400, 10, NA, S, PR, 16, seed) > 0
