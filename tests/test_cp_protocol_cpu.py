"""Properties of the context-parallel K/V exchange schedule (gen3c_b200/csrc/dit_engine.cu, default `p2p` mode), stated
on a pure-Python model of the two loops that define it:
  producer `me` pushes its slice to peers (me-1), (me-2), ... (mod N), each push followed by that peer's flag;
  consumer `c` (attn_wgmma.cu, TMA producer) visits KV chunks c, c+1, c+2, ... (mod N), the local one ungated.
The schedule is right when every consumer's k-th remote chunk is the k-th push of the rank that produces it, so that all
ranks can consume chunk k after k transfer slots."""
import pytest


def push_order(me: int, n: int):
    return [(me - i + n) % n for i in range(1, n)]


def visit_order(c: int, n: int):
    return [(c + j) % n for j in range(n)]


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_kth_remote_chunk_is_kth_push_of_its_producer(n):
    for c in range(n):
        remote = visit_order(c, n)[1:]  # first visited chunk is the local one
        for k, producer in enumerate(remote):
            assert push_order(producer, n)[k] == c


@pytest.mark.parametrize("n", [2, 4, 8])
def test_every_peer_is_served_exactly_once_and_never_self(n):
    for me in range(n):
        order = push_order(me, n)
        assert sorted(order) == [r for r in range(n) if r != me]


def test_two_buffer_sets_are_enough():
    """A rank can run at most one FA layer ahead of any peer (its attention of layer i needs every peer's flag of layer i,
    raised only after that peer finished attention i-1 in stream order), so a slot of set (i & 1) is rewritten by layer
    i+2 only after every reader of layer i is done.  Model: per-rank progress counters under that dependency."""
    n, layers = 4, 10
    done_attn = [0] * n  # number of attention layers each rank has completed
    pushed = [0] * n     # number of layers whose K/V each rank has pushed (needs its own attention of the layer before)
    import random
    rng = random.Random(0)
    for _ in range(10000):
        r = rng.randrange(n)
        if pushed[r] < layers and pushed[r] <= done_attn[r]:  # produce K/V of the next layer
            # writing set (pushed[r] & 1) on every peer: all peers must have finished reading layer pushed[r] - 2
            assert all(done_attn[p] >= pushed[r] - 1 for p in range(n)), "overwrite of a buffer still being read"
            pushed[r] += 1
        elif done_attn[r] < pushed[r] and all(pushed[p] > done_attn[r] for p in range(n)):
            done_attn[r] += 1
    assert min(done_attn) == layers
