"""Discrete-event model of the barrier protocol of the attention kernel (gen3c_b200/csrc/attn_wgmma.cu, k_attn_fwd):
one TMA producer filling a K ring and a V ring (ATT_STAGES stages each, full / empty mbarriers, asynchronous TMA
completion) and two consumer warpgroups, each with its own in-order wgmma pipe, software-pipelined with one S tile of
lookahead and alternating their MMA issue through a turn token (two mbarriers, turn[0] pre-arrived):

    prologue   wait K_0, [turn] S_0 [pass]; wait<0>; release K_0; softmax; pack P_0
    step j     wait K_j, V_{j-1}, [turn] S_j, commit, O += P_{j-1} V_{j-1}, commit [pass]; wait<1>; release K_j;
               softmax of S_j; wait<0>; release V_{j-1}; rescale O; pack P_j
    epilogue   wait V_{n-1}, [turn] O += P_{n-1} V_{n-1}, commit [pass]; wait<0>; release V_{n-1}; store; arrive `done`
    producer   K_j then V_j into stage j % ATT_STAGES after the matching empty barrier; finally waits on `done`

The roles run under random interleavings.  The model checks what the hardware tests can only show by not hanging:
  * no deadlock, for n_kv from 1 up and each ring depth the kernel may use;
  * a parity wait is never ambiguous: a barrier is never two phases ahead of its waiter;
  * a K or V stage is refilled only after every wgmma that reads it has retired;
  * P.V(j) reads P_j, and P_j is packed (over P_{j-1}) only after P.V(j-1) has retired;
  * O is rescaled only after P.V(j-1) has retired, and the softmax reads S_j only after S_j has retired;
  * MMAs are issued only while the warpgroup holds the turn, and the turn strictly alternates 0, 1, 0, 1, ...
mbarrier semantics: `wait(parity)` passes when the barrier's current phase parity differs from `parity`."""
import random

import pytest


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passed(self, parity):
        return (self.phase & 1) != parity


class Sim:
    def __init__(self, n_kv, stages, seed, early_v_release=False, skip_last_turn=None):
        self.n, self.S = n_kv, stages
        self.rng = random.Random(seed)
        self.early_v_release, self.skip_last_turn = early_v_release, skip_last_turn
        self.k_full = [Bar(1) for _ in range(stages)]
        self.v_full = [Bar(1) for _ in range(stages)]
        self.k_empty = [Bar(2) for _ in range(stages)]
        self.v_empty = [Bar(2) for _ in range(stages)]
        self.turn = [Bar(1), Bar(1)]
        self.turn[0].arrive()                      # consumer 0 holds the first turn
        self.done = Bar(2)
        self.k_stage = [None] * stages             # tile index currently in each stage
        self.v_stage = [None] * stages
        self.k_readers = [0] * stages              # issued, not yet retired wgmma reading the stage
        self.v_readers = [0] * stages
        self.tma = []                              # outstanding TMA loads: closures, complete in any order
        self.pipe = [[], []]                       # per consumer: committed wgmma groups (lists of ops), in order
        self.open = [[], []]                       # per consumer: ops issued since the last commit
        self.s_reg = [None, None]                  # step whose S the consumer's S registers hold (once retired)
        self.pa = [None, None]                     # step whose P the consumer's A fragments hold
        self.pv_done = [-1, -1]                    # last step whose P.V has retired
        self.holder = None
        self.turn_log = []

    def wait(self, bar, parity, expected_phase):
        while True:
            assert bar.phase <= expected_phase + 1, "parity wait is ambiguous: barrier ran two phases ahead of the waiter"
            if bar.passed(parity):
                assert bar.phase == expected_phase + 1
                return
            yield "spin"

    # ---- producer ----
    def producer(self):
        for j in range(self.n):
            st, use = j % self.S, j // self.S
            yield from self.wait(self.k_empty[st], (use & 1) ^ 1, use - 1)
            assert self.k_readers[st] == 0, "K stage refilled while a wgmma that reads it has not retired"
            self.tma.append(lambda st=st, j=j: (self.k_stage.__setitem__(st, j), self.k_full[st].arrive()))
            yield
            yield from self.wait(self.v_empty[st], (use & 1) ^ 1, use - 1)
            assert self.v_readers[st] == 0, "V stage refilled while a wgmma that reads it has not retired"
            self.tma.append(lambda st=st, j=j: (self.v_stage.__setitem__(st, j), self.v_full[st].arrive()))
            yield
        yield from self.wait(self.done, 0, 0)

    # ---- consumer helpers ----
    def take_turn(self, c, t):
        yield from self.wait(self.turn[c], t & 1, t)
        assert self.holder is None, "two warpgroups hold the turn"
        self.holder = c
        self.turn_log.append(c)

    def pass_turn(self, c):
        assert self.holder == c
        self.holder = None
        self.turn[c ^ 1].arrive()

    def issue_s(self, c, j):
        assert self.holder == c, "MMA issued outside this warpgroup's turn"
        st = j % self.S
        self.k_readers[st] += 1

        def op():
            assert self.k_stage[st] == j, "S reads a stage that does not hold K_j"
            self.k_readers[st] -= 1
            self.s_reg[c] = j
        self.open[c].append(op)

    def issue_pv(self, c, j):
        assert self.holder == c, "MMA issued outside this warpgroup's turn"
        st = j % self.S
        self.v_readers[st] += 1

        def op():
            assert self.v_stage[st] == j, "P.V reads a stage that does not hold V_j"
            assert self.pa[c] == j, "P.V(j) does not read P_j"
            self.v_readers[st] -= 1
            self.pv_done[c] = j
        self.open[c].append(op)

    def commit(self, c):
        self.pipe[c].append(self.open[c])
        self.open[c] = []

    def wgmma_wait(self, c, n):
        while len(self.pipe[c]) > n:
            yield "spin"

    def softmax(self, c, j):
        assert self.s_reg[c] == j, "softmax reads S before S_j has retired"

    def rescale_and_pack(self, c, j):
        assert self.pv_done[c] >= j - 1, "O rescaled / P_j packed while P.V(j-1) may still read P_{j-1}"
        self.pa[c] = j

    # ---- consumer ----
    def consumer(self, c):
        n, S = self.n, self.S
        # prologue
        yield from self.wait(self.k_full[0], 0, 0)
        yield from self.take_turn(c, 0)
        self.issue_s(c, 0)
        self.commit(c)
        self.pass_turn(c)
        yield
        yield from self.wgmma_wait(c, 0)
        self.k_empty[0].arrive()
        self.softmax(c, 0)
        self.rescale_and_pack(c, 0)
        yield
        for j in range(1, n):
            ks, vs = j % S, (j - 1) % S
            yield from self.wait(self.k_full[ks], (j // S) & 1, j // S)
            yield from self.wait(self.v_full[vs], ((j - 1) // S) & 1, (j - 1) // S)
            yield from self.take_turn(c, j)
            self.issue_s(c, j)
            self.commit(c)
            self.issue_pv(c, j - 1)
            self.commit(c)
            self.pass_turn(c)
            yield
            yield from self.wgmma_wait(c, 1)
            self.k_empty[ks].arrive()
            if self.early_v_release:
                self.v_empty[vs].arrive()
            self.softmax(c, j)
            yield
            yield from self.wgmma_wait(c, 0)
            if not self.early_v_release:
                self.v_empty[vs].arrive()
            self.rescale_and_pack(c, j)
            yield
        # epilogue
        vs = (n - 1) % S
        yield from self.wait(self.v_full[vs], ((n - 1) // S) & 1, (n - 1) // S)
        skip = self.skip_last_turn == c
        if not skip:
            yield from self.take_turn(c, n)
        else:
            self.holder = c                       # issues as if it held the turn, without waiting for it
        self.issue_pv(c, n - 1)
        self.commit(c)
        if not skip:
            self.pass_turn(c)
        else:
            self.holder = None
        yield
        yield from self.wgmma_wait(c, 0)
        self.v_empty[vs].arrive()
        assert self.pv_done[c] == n - 1, "store before the last P.V"
        self.done.arrive()

    def run(self):
        roles = [self.producer(), self.consumer(0), self.consumer(1)]
        live = list(range(len(roles)))
        idle = 0
        while live:
            choice = self.rng.random()
            busy = [c for c in (0, 1) if self.pipe[c]]
            if busy and choice < 0.35:
                c = self.rng.choice(busy)
                grp = self.pipe[c][0]
                if grp:
                    grp.pop(0)()
                if not grp:
                    self.pipe[c].pop(0)
                idle = 0
            elif self.tma and choice < 0.55:
                self.tma.pop(self.rng.randrange(len(self.tma)))()
                idle = 0
            else:
                r = self.rng.choice(live)
                try:
                    idle = idle + 1 if next(roles[r]) == "spin" else 0
                except StopIteration:
                    live.remove(r)
                    idle = 0
            stuck = not any(self.pipe) and not self.tma
            assert idle < 5000 * len(roles) or not stuck, "deadlock: every live role spins and nothing is in flight"
        assert not any(self.pipe) and not self.tma
        expect = [c for _ in range(self.n + 1) for c in (0, 1)]
        assert self.turn_log == expect, "the turn does not strictly alternate over n_kv + 1 turns per warpgroup"


@pytest.mark.parametrize("stages", [2, 3])
@pytest.mark.parametrize("n_kv", [1, 2, 3, 4, 5, 7, 8, 11])
def test_pingpong_protocol(n_kv, stages):
    for seed in range(8):
        Sim(n_kv, stages, seed=seed).run()


@pytest.mark.parametrize("stages", [2, 3])
def test_model_detects_early_v_release(stages):
    """Negative control: releasing V_{j-1} after wait<1> (S_j retired) instead of wait<0> lets the producer refill the
    V stage while P.V(j-1) still reads it."""
    failures = 0
    for seed in range(40):
        try:
            Sim(11, stages, seed=seed, early_v_release=True).run()
        except AssertionError as e:
            assert "V stage refilled" in str(e) or "does not hold V_j" in str(e), str(e)
            failures += 1
    assert failures > 0


@pytest.mark.parametrize("c", [0, 1])
def test_model_detects_a_skipped_last_turn(c):
    """Negative control: an epilogue in which one warpgroup issues its last P.V without taking (and passing) its turn."""
    with pytest.raises(AssertionError):
        Sim(5, 2, seed=3, skip_last_turn=c).run()
