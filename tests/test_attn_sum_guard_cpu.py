"""CPU models of the sum-guarded softmax of the attention kernel's steady-state KV tiles (gen3c_b200/csrc/attn_wgmma.cu,
exp_tile and the fallback in `step`).

Numerics: a float32 model of one consumer warpgroup's rule, with P rounded to bf16 for the P.V product.  Tile 0 runs
the exact softmax_tile (row max, per-warp lazy rule: m moves when some row of the warp's 16 exceeds it by more than 8).
Every later tile is exponentiated against the current m; each quad thread sums its 32 columns (8 i + 2 (lane % 4) +
{0, 1}) of each row into t; the tile is accepted when every thread of the warpgroup (64 rows) has t < 2^24, and then
l += t.  Otherwise the whole warpgroup recomputes S and runs softmax_tile.  The model must stay within the float64
bound of tests/attn_ref64.py, and three wrong variants must not: no guard (P overflows), l updated before the decision
(a fallback tile counted twice), and a per-warp decision (the fallback's wgmma issued by only some warps of the
warpgroup, modelled as a wrong S for them).

Protocol: the ping-pong model of tests/test_attn_pingpong_model_cpu.py with the later K release (after the guard
decision) and the fallback's second S wgmma over K_j, issued outside the turn.  A consumer's arrive on k_empty promises
that none of its wgmma still reads the stage; the model checks that promise when it is made, and the negative control
releases K_j before the decision."""
import math

import numpy as np
import pytest
import torch

from tests import attn_ref64
from tests.test_attn_pingpong_model_cpu import Sim

TILE, WARP_ROWS, WG_ROWS, LAZY = 128, 16, 64, 8.0
GUARD = np.float32(2.0 ** 24)
LN2 = math.log(2.0)


def bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def ex2(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.exp2(x.astype(np.float32)).astype(np.float32)


def thread_sums(p):
    """[rows, 4]: each quad thread's sum of its 32 columns of each row (float32, in column order)"""
    t = np.zeros((p.shape[0], 4), np.float32)
    for i in range(16):
        for q in range(4):
            t[:, q] += p[:, 8 * i + 2 * q] + p[:, 8 * i + 2 * q + 1]
    return t


def softmax_tile(s, m, l, O):
    """The exact per-tile rule on rows whose group fell back: returns (p, m, l, O) with m moved per warp."""
    mx = s.max(axis=1)
    with np.errstate(invalid="ignore"):
        move = ~(mx - m <= LAZY)
    move = np.repeat(move.reshape(-1, WARP_ROWS).any(axis=1), WARP_ROWS)
    nm = np.where(move, np.fmax(m, mx), m).astype(np.float32)
    alpha = np.where(move, ex2(m - nm), np.float32(1.0)).astype(np.float32)
    p = ex2(s - nm[:, None])
    with np.errstate(invalid="ignore"):
        return p, nm, l * alpha + p.sum(axis=1, dtype=np.float32), O * alpha[:, None]


def model(q, k, v, guard=True, l_before=False, per_warp=False):
    """O = softmax(q k^T) v of one head by the kernel's rule; q [Lq, 128] (Lq a multiple of 64), k, v [Lk, 128]
    (Lk a multiple of 128), scores in log2 units (scale = ln 2)."""
    S = (q.astype(np.float32) @ k.astype(np.float32).T).astype(np.float32)
    rows = S.shape[0]
    m = np.full(rows, -np.inf, np.float32)
    l = np.zeros(rows, np.float32)
    O = np.zeros((rows, v.shape[1]), np.float32)
    for j in range(S.shape[1] // TILE):
        s = S[:, j * TILE:(j + 1) * TILE]
        vj = v[j * TILE:(j + 1) * TILE]
        if j == 0:
            p, m, l, O = softmax_tile(s, m, l, O)
        else:
            p = ex2(s - m[:, None])
            t = thread_sums(p)
            fail = ~np.all(t < GUARD, axis=1) if guard else np.zeros(rows, bool)
            group = WARP_ROWS if per_warp else WG_ROWS
            redo = np.repeat(fail.reshape(-1, group).any(axis=1), group)
            counted = np.ones(rows, bool) if l_before else ~redo
            l = l + np.where(counted, t.sum(axis=1, dtype=np.float32), np.float32(0))
            if redo.any():
                s2 = s.copy()
                if per_warp:  # a warp that issues the wgmma without the rest of its warpgroup gets no valid S
                    alone = redo & ~np.repeat(redo.reshape(-1, WG_ROWS).all(axis=1), WG_ROWS)
                    s2[alone] = 0.0
                p2, m2, l2, O2 = softmax_tile(s2[redo], m[redo], l[redo], O[redo])
                p[redo], m[redo], l[redo], O[redo] = p2, m2, l2, O2
        with np.errstate(over="ignore", invalid="ignore"):
            O = O + bf16(p) @ vj
    with np.errstate(over="ignore", invalid="ignore"):
        return O / l[:, None]


def operands(name, rng):
    """Scores built as in tests/test_attn_sum_guard_gpu.py: dimension 0 of every query is 1, dimension 0 of key n its
    score offset, dimensions 2.. a small random term."""
    Lq, n_kv = 128, 8
    if name in ("staircase", "large_v"):
        n_kv = 55
    Lk = n_kv * TILE
    q = rng.standard_normal((Lq, 128)) * 0.1
    k = rng.standard_normal((Lk, 128)) * 0.1
    v = rng.standard_normal((Lk, 128))
    q[:, 0], q[:, 1] = 1.0, 0.0
    tile = np.arange(Lk) // TILE
    k[:, 1] = 0.0
    k[:, 0] = -1.0

    def spike(keys, value, dim=0):
        k[keys] = 0.0
        k[keys, dim] = value

    if name == "random":
        q, k = rng.standard_normal((Lq, 128)) * 0.3, rng.standard_normal((Lk, 128)) * 0.3
    elif name == "drift":  # +4 per tile: the reference trails by up to 24 and moves every sixth tile
        k[:, 0] = 4.0 * tile - 1.0
    elif name == "staircase":  # +30 per tile: every tile falls back
        k[:, 0] = 30.0 * tile - 1.0
        spike(np.arange(n_kv) * TILE + 77, 30.0 * np.arange(n_kv))
    elif name.startswith("jump"):  # 16 keys of tile 3 in one quad thread's columns, `value` above m = 0
        spike([5], 0.0)
        cols = [8 * i + 2 + e for i in range(8) for e in (0, 1)]
        spike([3 * TILE + c for c in cols], float(name[4:]))
    elif name == "one_warp":  # only query 93 jumps by 150 in tile 2
        q[93, 1] = 1.0
        spike([2 * TILE + 9], 150.0, dim=1)
    elif name == "large_v":  # every later tile accepted at P = 2^18.875 against m = 0, |v| ~ 2^90
        k[:, 0] = np.where(tile == 0, 0.0, 18.875)
        k[:, 2:] = 0.0
        v = v * 2.0 ** 90
    return (torch.from_numpy(bf16(x)) for x in (q, k, v))


CASES = ["random", "drift", "staircase", "jump19.875", "jump20", "jump150", "one_warp", "large_v"]


@pytest.mark.parametrize("name", CASES)
def test_model_within_ref64_bound(name):
    q, k, v = operands(name, np.random.default_rng(3))
    out = torch.from_numpy(bf16(model(q.numpy(), k.numpy(), v.numpy())))
    attn_ref64.check(out, q, k, v, 1, LN2, label=name)


@pytest.mark.parametrize("variant,name", [("no_guard", "staircase"), ("no_guard", "jump150"),
                                          ("l_before", "jump20"), ("l_before", "one_warp"),
                                          ("per_warp", "one_warp")])
def test_wrong_variants_fail(variant, name):
    """Negative controls: without the guard P = 2^150 overflows; adding t to l before the decision counts a fallback
    tile twice; a per-warp decision leaves the other three warps of query 93's warpgroup out of the fallback's wgmma."""
    q, k, v = operands(name, np.random.default_rng(3))
    out = model(q.numpy(), k.numpy(), v.numpy(), guard=variant != "no_guard", l_before=variant == "l_before",
                per_warp=variant == "per_warp")
    if not np.isfinite(out).all():
        return
    e, s, _ = attn_ref64.Reference(q, k, v, 1, LN2).ratios(torch.from_numpy(bf16(out)))
    assert e > 1.0 or s > 1.0, (e, s)


# ---- protocol ----
class GuardSim(Sim):
    """Sim with the kernel's step: guard decision before the K release; on a fallback (the tiles in `redo`) a second S
    wgmma over K_j, issued outside the turn, then wait<0>."""

    def __init__(self, n_kv, stages, seed, redo=(), early_k_release=False):
        super().__init__(n_kv, stages, seed)
        self.redo, self.early_k_release = set(redo), early_k_release
        self.own_k = [[0] * stages, [0] * stages]  # per consumer: its issued, unretired wgmma reading each K stage
        self.k_released = [set(), set()]           # per consumer: the K tiles it has released

    def issue_s(self, c, j, in_turn=True):
        if in_turn:
            assert self.holder == c, "MMA issued outside this warpgroup's turn"
        assert j not in self.k_released[c], "S wgmma issued over K_j after this warpgroup released it"
        st = j % self.S
        self.k_readers[st] += 1
        self.own_k[c][st] += 1

        def op():
            assert self.k_stage[st] == j, "S reads a stage that does not hold K_j"
            self.k_readers[st] -= 1
            self.own_k[c][st] -= 1
            self.s_reg[c] = j
        self.open[c].append(op)

    def release_k(self, c, j):
        st = j % self.S
        assert self.own_k[c][st] == 0, "K stage released while this warpgroup's wgmma still reads it"
        self.k_released[c].add(j)
        self.k_empty[st].arrive()

    def consumer(self, c):
        n, S = self.n, self.S
        yield from self.wait(self.k_full[0], 0, 0)
        yield from self.take_turn(c, 0)
        self.issue_s(c, 0)
        self.commit(c)
        self.pass_turn(c)
        yield
        yield from self.wgmma_wait(c, 0)
        self.release_k(c, 0)
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
            self.softmax(c, j)  # guarded exponentials of S_j
            if self.early_k_release:
                self.release_k(c, j)
            yield
            if j in self.redo:  # the vote failed: S_j again from K_j
                self.issue_s(c, j, in_turn=False)
                self.commit(c)
                yield
                yield from self.wgmma_wait(c, 0)
            if not self.early_k_release:
                self.release_k(c, j)
            if j in self.redo:
                self.softmax(c, j)
            yield
            yield from self.wgmma_wait(c, 0)
            self.v_empty[vs].arrive()
            self.rescale_and_pack(c, j)
            yield
        vs = (n - 1) % S
        yield from self.wait(self.v_full[vs], ((n - 1) // S) & 1, (n - 1) // S)
        yield from self.take_turn(c, n)
        self.issue_pv(c, n - 1)
        self.commit(c)
        self.pass_turn(c)
        yield
        yield from self.wgmma_wait(c, 0)
        self.v_empty[vs].arrive()
        assert self.pv_done[c] == n - 1, "store before the last P.V"
        self.done.arrive()


REDO = {"none": (), "all": range(1, 64), "odd": range(1, 64, 2), "even": range(2, 64, 2), "one": (3,)}


@pytest.mark.parametrize("redo", list(REDO))
@pytest.mark.parametrize("stages", [2, 3])
@pytest.mark.parametrize("n_kv", [1, 2, 3, 5, 8, 11])
def test_guard_protocol(n_kv, stages, redo):
    for seed in range(6):
        GuardSim(n_kv, stages, seed, redo=REDO[redo]).run()


@pytest.mark.parametrize("stages", [2, 3])
def test_model_detects_early_k_release(stages):
    """Negative control: releasing K_j right after wait<1>, before the guard decision, promises the stage free while the
    fallback's second S wgmma has yet to read it."""
    with pytest.raises(AssertionError, match="after this warpgroup released it"):
        GuardSim(8, stages, seed=1, redo=REDO["all"], early_k_release=True).run()


class FakeSet(set):
    def __contains__(self, _):
        return False


@pytest.mark.parametrize("stages", [2, 3])
def test_fallback_reread_finds_k_j(stages):
    """The producer cannot overwrite K_j before the fallback has read it even at the moment K_j is released early: its
    next load into that K stage follows its load of V_{j+stages-1}, which waits for this consumer's release of V_{j-1}
    after its wait<0>, and that wait retires the second S.  The model shows it: with only the refill-time checks, the
    early release never lets a fallback read the wrong tile."""
    for seed in range(20):
        sim = GuardSim(11, stages, seed, redo=REDO["all"], early_k_release=True)
        sim.k_released = [FakeSet(), FakeSet()]  # refill-time checks only
        sim.run()
