"""Calibration of tests/attn_ref64.py on the CPU: a torch-fp32 emulation of the attention kernel's arithmetic (128-key
tiles visited in the kernel's order, the lazy rescale with its warp vote, bf16 P in the numerator, fp32 row sums) must
stay within both checks of attn_ref64 with a factor 2 to spare over a few hundred seeds and shapes, and each negative
control (a plausible kernel bug, emulated) must miss the check it targets by at least 3x on the case built for it."""
import math

import numpy as np
import pytest
import torch

from tests import attn_ref64

TILE, WARP_ROWS, THRESHOLD = 128, 16, 8.0
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634


def emulate(q, k, v, heads, scale, chunk_len=0, first=0, token_major=False, control=None):
    """The kernel's arithmetic in torch fp32.  q [Lq, heads*128], k and v [Lk, heads*128] bf16 (token-major V; the V^T
    build reads the same values).  V^T build: Lk % 128 == 0, chunks of chunk_len keys (0: one) visited from `first`;
    token-major build: any Lk, the keys past Lk in the last tile masked.  Query rows past Lq are the TMA's zeros and take
    part in their warp's vote.  `control` emulates one bug:
      drop_tile      the middle KV tile is skipped
      k_rotated_only K tiles follow the rotated chunk order, V^T tiles the unrotated one
      swap_cols      head dims 8..15 and 40..47 of head 0 exchanged at the store
      swap_rows      query rows 19 and 27 (rows a and a + 8 of one thread of warp 1) exchanged at the store
      log2e_twice    the scale multiplied by log2(e) a second time
      tail_zero      the zero-filled keys past Lk enter the softmax with score 0"""
    Lq, Lk = q.shape[0], k.shape[0]
    D = heads * 128
    sl2 = attn_ref64.scale_log2(scale)
    if control == "log2e_twice":
        sl2 = float(np.float32(np.float32(sl2) * np.float32(LOG2E)))
    n_kv = (Lk + TILE - 1) // TILE if token_major else Lk // TILE
    cl = Lk if (token_major or chunk_len <= 0) else chunk_len
    tpc, n_chunks = cl // TILE, Lk // cl
    rows = (Lq + TILE - 1) // TILE * TILE
    qp = torch.zeros(rows, D)
    qp[:Lq] = q.float()
    kp, vp = torch.zeros(n_kv * TILE, D), torch.zeros(n_kv * TILE, D)
    kp[:Lk], vp[:Lk] = k.float(), v.float()
    tiles = []  # (first key of the K tile, first key of the V tile, valid keys)
    for j in range(n_kv):
        if control == "drop_tile" and j == n_kv // 2:
            continue
        if token_major:
            tiles.append((j * TILE, j * TILE, min(TILE, Lk - j * TILE)))
            continue
        chunk = (first + j // tpc) % n_chunks
        vchunk = j // tpc if control == "k_rotated_only" else chunk
        within = j % tpc
        tiles.append((chunk * cl + within * TILE, vchunk * cl + within * TILE, TILE))
    out = torch.empty(rows, D)
    for h in range(heads):
        hs = slice(h * 128, (h + 1) * 128)
        Q = qp[:, hs]
        m = torch.full((rows,), -math.inf)
        l = torch.zeros(rows)
        O = torch.zeros(rows, 128)
        for k0, v0, valid in tiles:
            s = Q @ kp[k0:k0 + TILE, hs].T
            if valid < TILE and control != "tail_zero":
                s[:, valid:] = -math.inf
            mx = s.amax(1) * sl2
            stay = (mx - m <= THRESHOLD).reshape(-1, WARP_ROWS).all(1)
            move = (~stay).repeat_interleave(WARP_ROWS)
            nm = torch.where(move, torch.maximum(m, mx), m)
            alpha = torch.where(move, torch.exp2(m - nm), torch.ones_like(m))
            m = nm
            l = l * alpha
            O = O * alpha[:, None]
            p = torch.exp2((s.double() * sl2 - m.double()[:, None]).float())  # fma: one rounding
            p = torch.where(p < 2.0 ** -126, torch.zeros_like(p), p)          # ex2.approx.ftz
            l = l + p.sum(1)
            O = O + p.bfloat16().float() @ vp[v0:v0 + TILE, hs]
        out[:, hs] = O * (1.0 / l)[:, None]
    o = out[:Lq].bfloat16()
    if control == "swap_cols":
        o[:, 8:16], o[:, 40:48] = o[:, 40:48].clone(), o[:, 8:16].clone()
    if control == "swap_rows":
        o[[19, 27]] = o[[27, 19]]
    return o


def operands(Lq, Lk, heads, seed, gain=1.0, log2_units=False, v_mean=0.0):
    """q, k, v bf16 with N(0, gain^2) queries and keys; scale 1/sqrt(128), or ln 2 with Q pre-scaled by 1/sqrt(128) *
    log2(e) (the DiT engine's convention)."""
    g = torch.Generator().manual_seed(seed)
    D = heads * 128
    q = torch.randn(Lq, D, generator=g) * gain
    k = torch.randn(Lk, D, generator=g) * gain
    v = torch.randn(Lk, D, generator=g) + v_mean
    scale = 128 ** -0.5
    if log2_units:
        q, scale = q * (scale * LOG2E), LN2
    return q.bfloat16(), k.bfloat16(), v.bfloat16(), scale


def sweep_case(i):
    """Case i of the sweep: a random layout (V^T with rotated chunks, or token-major with any Lk), shape, score spread,
    scale convention, and now and then a block of keys far above the rest or a staircase of row maxima."""
    rng = np.random.default_rng(1000 + i)
    heads = int(rng.integers(1, 3))
    Lq = int(rng.integers(1, 300))
    token_major = bool(rng.integers(0, 2))
    kw = dict(token_major=token_major)
    if token_major:
        Lk = int(rng.integers(1, 2200))
    else:
        tpc = int(rng.choice([1, 2, 3, 7]))
        chunks = int(rng.integers(1, 5))
        Lk = tpc * chunks * TILE
        kw.update(chunk_len=tpc * TILE, first=int(rng.integers(0, chunks)))
    gain = float(rng.choice([0.3, 1.0, 2.0, 3.0]))
    q, k, v, scale = operands(Lq, Lk, heads, seed=i, gain=gain, log2_units=bool(rng.integers(0, 2)),
                              v_mean=float(rng.choice([0.0, 0.0, 2.0])))
    kind = rng.integers(0, 4)
    if kind == 1 and Lk > 40:  # a block of keys far above the others (the rescale of O and l at that tile)
        a = int(rng.integers(0, Lk - 32))
        k[a:a + 32, :128] = float(rng.choice([2.0, 4.0]))
        q[:, :128] = q[:, :128].abs()
    elif kind == 2 and Lk >= 4 * TILE:  # the row max rises by ~4 (log2) per tile: stale references, P up to 2^8
        t = torch.arange(Lk) // TILE
        k[:, 0] = (4.0 * t / max(float(q[:, 0].float().abs().max()), 1e-3) / scale * LN2).bfloat16()
        q[:, 0] = q[:, 0].abs()
    return q, k, v, heads, scale, kw


N_SWEEP = 300


def test_emulation_within_both_checks():
    worst_e = worst_s = 0.0
    for i in range(N_SWEEP):
        q, k, v, heads, scale, kw = sweep_case(i)
        o = emulate(q, k, v, heads, scale, **kw)
        e, s, _ = attn_ref64.Reference(q, k, v, heads, scale).ratios(o)
        assert e <= 0.5 and s <= 0.5, (i, e, s, q.shape[0], k.shape[0], heads, kw)
        worst_e, worst_s = max(worst_e, e), max(worst_s, s)
    print(f"emulation over {N_SWEEP} cases: largest element/bound {worst_e:.3g}, norm/(6 sigma) {worst_s:.3g}")


@pytest.mark.parametrize("Lq,n_kv,gain", [(256, 55, 1.0), (128, 55, 0.3), (64, 440, 1.0)])
def test_emulation_diffuse_long_rows(Lq, n_kv, gain):
    """The self-attention regime: thousands of keys of similar weight (up to the benchmark's 440 tiles), where the
    statistical check carries the weight."""
    q, k, v, scale = operands(Lq, n_kv * TILE, 2, seed=n_kv, gain=gain, log2_units=True)
    o = emulate(q, k, v, 2, scale)
    e, s, _ = attn_ref64.Reference(q, k, v, 2, scale).ratios(o)
    print(f"Lq={Lq} n_kv={n_kv} gain={gain}: element/bound {e:.3g}, norm/(6 sigma) {s:.3g}")
    assert e <= 0.5 and s <= 0.5, (e, s)


def control_case(name):
    """(q, k, v, heads, scale, emulate kwargs, index of the targeted check: 0 per element, 1 statistical)"""
    if name == "drop_tile":
        return (*operands(64, 55 * TILE, 1, seed=5), {}, 1)
    if name == "k_rotated_only":
        return (*operands(64, 4 * 512, 1, seed=6), dict(chunk_len=512, first=1), 1)
    if name in ("swap_cols", "swap_rows", "log2e_twice"):
        return (*operands(64, 8 * TILE, 1, seed=7, gain=2.0), {}, 0)
    if name == "tail_zero":  # valid keys score ~ -14 against every query: the zero keys (score 0) would dominate
        Lk = 1000
        g = torch.Generator().manual_seed(8)
        q = torch.ones(200, 128)
        k = -1.0 - 0.5 * torch.rand(Lk, 128, generator=g)
        v = torch.randn(Lk, 128, generator=g)
        return q.bfloat16(), k.bfloat16(), v.bfloat16(), 128 ** -0.5, dict(token_major=True), 0
    raise ValueError(name)


@pytest.mark.parametrize("name", ["drop_tile", "k_rotated_only", "swap_cols", "swap_rows", "log2e_twice", "tail_zero"])
def test_negative_control(name):
    q, k, v, scale, kw, target = control_case(name)
    ref = attn_ref64.Reference(q, k, v, 1, scale)
    good = ref.ratios(emulate(q, k, v, 1, scale, **kw))
    bad = ref.ratios(emulate(q, k, v, 1, scale, control=name, **kw))
    print(f"{name}: correct emulation {good[0]:.3g} / {good[1]:.3g}; control misses check {target} by {bad[target]:.3g}x")
    assert good[0] <= 0.5 and good[1] <= 0.5, good
    assert bad[target] >= 3.0, bad
