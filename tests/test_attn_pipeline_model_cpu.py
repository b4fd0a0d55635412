"""Discrete-event model of a software-pipelined attention barrier protocol with S lookahead: one query tile per CTA, kBufs
S accumulator buffers, a ring of {K_{j+kBufs}, V_j} stages, S(j+kBufs) issued behind P.V(j) by a single MMA issuer.  The
attention kernel (gen3c_b200/csrc/attn_wgmma.cu) does not pipeline S yet (each consumer warpgroup runs S -> softmax -> P.V
in order, DESIGN.md §7); this model is the protocol that lookahead is to follow, and it is validated here before any
kernel relies on it.

The model restates the protocol's bookkeeping — ring slot / phase, per-buffer parity bits of the softmax warps (`sph`) and of the
issuer (`pph`), the prologue, the commits behind every P.V, the final waits, the second (exact) pass continuing with the same
parities — and runs the roles (loader, issuer, softmax warps, in-order tensor pipe, asynchronous TMA) under random
interleavings.  It checks what the hardware tests can only show by not hanging:
  * no deadlock for any n_kv (including n_kv < kBufs and n_kv % kBufs != 0), one or two passes;
  * a parity wait is never ambiguous: the barrier is never more than one phase ahead of what the waiter waits for;
  * S(j) is only overwritten after P.V has consumed the P stored in the same buffer, P.V(j) only runs on P(j) of every warp,
    a softmax warp only reads S(j) of its step, a ring stage is only refilled after the MMAs that read it have completed;
  * a rescale of O at step j (exact tiles) only runs when P.V(j-1) has completed.
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
    def __init__(self, n_kv, bufs, stages, warps, passes, rescale_steps, seed):
        self.n, self.B, self.S, self.W, self.passes = n_kv, bufs, stages, warps, passes
        self.rescale_steps = rescale_steps
        self.rng = random.Random(seed)
        self.st_full = [Bar(1) for _ in range(stages)]
        self.st_empty = [Bar(1) for _ in range(stages)]
        self.s_full = [Bar(1) for _ in range(bufs)]
        self.p_full = [Bar(warps) for _ in range(bufs)]
        self.pass_bar = [0, 0]                 # roles that finished pass 0 (stands for the __syncthreads + cluster sync)
        self.pipe = []                         # in-order tensor pipe: closures
        self.tma = []                          # outstanding TMA loads: closures, complete in any order
        self.buf = [None] * bufs               # ("S", g) / ("P", g): content of the S buffer, g = global step index
        self.pwritten = [[None] * warps for _ in range(bufs)]
        self.stage = [None] * stages           # (k index or None, v index or None) currently loaded
        self.stage_busy = [False] * stages     # MMAs reading it are issued but not complete
        self.pv_done = -1                      # last global step whose P.V has executed
        self.waits = 0

    # every wait records the absolute phase it waits for: the barrier may be at most one phase ahead (else parity aliases)
    def wait(self, bar, parity, expected_phase):
        while True:
            assert bar.phase <= expected_phase + 1, "parity wait is ambiguous: barrier ran two phases ahead of the waiter"
            if bar.passed(parity):
                assert bar.phase == expected_phase + 1
                return
            yield "spin"

    def loader(self):
        slot = phase = 0
        fills = 0
        for ps in range(self.passes):
            seq = [(j, None) for j in range(min(self.B, self.n))]
            seq += [(j + self.B if j + self.B < self.n else None, j) for j in range(self.n)]
            for (jk, jv) in seq:
                # producer-side wait on st_empty with phase ^ 1: expected absolute phase = uses of this slot so far - 1
                yield from self.wait(self.st_empty[slot], phase ^ 1, fills // self.S - 1)
                assert not self.stage_busy[slot], "ring stage refilled while MMAs still read it"
                sl, tag = slot, (None if jk is None else (ps, jk), None if jv is None else (ps, jv))

                def land(sl=sl, tag=tag):
                    self.stage[sl] = tag
                    self.st_full[sl].arrive()
                self.tma.append(land)
                fills += 1
                slot += 1
                if slot == self.S:
                    slot, phase = 0, phase ^ 1
                yield
            yield from self.end_of_pass(ps)

    def issuer(self):
        slot = phase = 0
        uses = 0                                # stages consumed so far
        pph = 0
        p_uses = [0] * self.B
        for ps in range(self.passes):
            g0 = ps * self.n
            for j in range(min(self.B, self.n)):
                yield from self.wait(self.st_full[slot], phase, uses // self.S)
                self.issue_s(ps, j, j, slot, release=True)
                uses += 1
                slot += 1
                if slot == self.S:
                    slot, phase = 0, phase ^ 1
            b = 0
            for j in range(self.n):
                yield from self.wait(self.st_full[slot], phase, uses // self.S)
                yield from self.wait(self.p_full[b], (pph >> b) & 1, p_uses[b])
                pph ^= 1 << b
                p_uses[b] += 1
                self.stage_busy[slot] = True
                sl = slot

                def pv(b=b, g=g0 + j, sl=sl, ps=ps, j=j):
                    assert self.stage[sl][1] == (ps, j), "P.V reads a stage that does not hold V_j"
                    assert self.buf[b] == ("S", g) and all(w == g for w in self.pwritten[b]), "P.V before P of every warp"
                    self.buf[b] = ("P-consumed", g)
                    self.pv_done = g
                self.pipe.append(pv)
                if j + self.B < self.n:
                    self.issue_s(ps, j + self.B, b, slot, release=False)
                if j + self.B < self.n or not getattr(self, "drop_tail_commits", False):
                    self.pipe.append(lambda b=b: self.s_full[b].arrive())       # commit s_full[b]

                def rel(sl=sl):
                    self.stage_busy[sl] = False
                    self.st_empty[sl].arrive()
                self.pipe.append(rel)                                            # commit st_empty[stage]
                uses += 1
                slot += 1
                if slot == self.S:
                    slot, phase = 0, phase ^ 1
                b = 0 if b == self.B - 1 else b + 1
                yield
            yield from self.end_of_pass(ps)

    def issue_s(self, ps, j, b, sl, release):
        g = ps * self.n + j
        self.stage_busy[sl] = True

        def s_mma():
            assert self.stage[sl][0] == (ps, j), "S MMA reads a stage that does not hold K_j"
            assert self.buf[b] is None or self.buf[b][0] == "P-consumed", "S overwrites a buffer whose P was not consumed"
            self.buf[b] = ("S", g)
        self.pipe.append(s_mma)
        if release:
            self.pipe.append(lambda: self.s_full[b].arrive())

            def rel():
                self.stage_busy[sl] = False
                self.st_empty[sl].arrive()
            self.pipe.append(rel)

    def softmax(self, w):
        sph = 0
        s_uses = [0] * self.B
        for ps in range(self.passes):
            g0 = ps * self.n
            b = 0
            for j in range(self.n):
                yield from self.wait(self.s_full[b], (sph >> b) & 1, s_uses[b])
                sph ^= 1 << b
                s_uses[b] += 1
                assert self.buf[b] == ("S", g0 + j), "softmax reads a buffer that does not hold S of its step"
                yield
                if j >= 1 and (ps, j) in self.rescale_steps:
                    bp = self.B - 1 if b == 0 else b - 1
                    # wait for the NEXT completion of s_full[bp] without consuming it
                    yield from self.wait(self.s_full[bp], (sph >> bp) & 1, s_uses[bp])
                    assert self.pv_done >= g0 + j - 1, "O rescaled while P.V(j-1) may still be running"
                assert self.buf[b] == ("S", g0 + j)
                self.pwritten[b][w] = g0 + j
                self.p_full[b].arrive()
                b = 0 if b == self.B - 1 else b + 1
                yield
            for j in range(max(0, self.n - self.B), self.n):
                bb = j % self.B
                yield from self.wait(self.s_full[bb], (sph >> bb) & 1, s_uses[bb])
                sph ^= 1 << bb
                s_uses[bb] += 1
            assert self.pv_done == g0 + self.n - 1, "epilogue before the last P.V"
            yield from self.end_of_pass(ps)

    def end_of_pass(self, ps):
        self.pass_bar[ps] += 1
        while self.pass_bar[ps] < 2 + self.W:
            yield "spin"

    def run(self):
        roles = [self.loader(), self.issuer()] + [self.softmax(w) for w in range(self.W)]
        live = list(range(len(roles)))
        idle = 0
        while live:
            choice = self.rng.random()
            if self.pipe and choice < 0.35:
                self.pipe.pop(0)()
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
            assert idle < 5000 * len(roles) or self.pipe or self.tma, "deadlock: every live role spins and nothing is in flight"
        assert not self.pipe and not self.tma


@pytest.mark.parametrize("bufs,stages", [(3, 5), (2, 6)])
@pytest.mark.parametrize("n_kv", [1, 2, 3, 4, 5, 7, 9, 10, 11, 16, 23])
def test_pipeline_protocol_one_pass(n_kv, bufs, stages):
    for seed in range(6):
        Sim(n_kv, bufs, stages, warps=4, passes=1, rescale_steps=set(), seed=seed).run()


@pytest.mark.parametrize("bufs,stages", [(3, 5), (2, 6)])
@pytest.mark.parametrize("n_kv", [1, 2, 3, 4, 8, 9, 10, 11])
def test_pipeline_protocol_second_exact_pass_with_rescales(n_kv, bufs, stages):
    """The redo path: the sweep is repeated in the exact mode with the barrier parities of every role simply continuing;
    exact tiles may rescale O at any step >= 1 (here: every step of pass 1, and some of pass 0)."""
    rescale = {(1, j) for j in range(1, n_kv)} | {(0, j) for j in range(1, n_kv, 3)}
    for seed in range(6):
        Sim(n_kv, bufs, stages, warps=4, passes=2, rescale_steps=rescale, seed=100 + seed).run()


def test_model_detects_a_missing_commit():
    """Negative control: without the commit of s_full behind a P.V that has no new S MMA in front of it (the last kBufs
    steps), the epilogue waits forever — the model must report the deadlock."""
    sim = Sim(7, 3, 5, warps=2, passes=1, rescale_steps=set(), seed=1)
    sim.drop_tail_commits = True
    with pytest.raises(AssertionError, match="deadlock"):
        sim.run()


def test_model_detects_too_few_buffers_for_the_lookahead():
    """Negative control: issuing S(j + kBufs + 1) into the buffer of step j + 1 (a look-ahead one larger than the number of
    buffers) must trip the 'S overwrites a buffer whose P was not consumed' / wrong-step checks."""
    class Broken(Sim):
        def issue_s(self, ps, j, b, sl, release):
            super().issue_s(ps, j, (b + 1) % self.B if not release else b, sl, release)

    with pytest.raises(AssertionError):
        Broken(9, 3, 5, warps=2, passes=1, rescale_steps=set(), seed=2).run()
