"""The sum guard of the attention kernel's steady-state KV tiles (gen3c_b200/csrc/attn_wgmma.cu, exp_tile and the
fallback in `step`): a tile is exponentiated against the current reference m without a row max and accepted when every
thread of the warpgroup holds partial row sums (its 32 columns of each of its two rows) below 2^24; otherwise the whole
warpgroup recomputes S from K_j and runs the exact softmax_tile, which moves m.  Each case builds scores whose values
are known exactly (scale = ln 2: S is in log2 units; see tests/test_attn_lazy_rescale_gpu.py for the operand layout),
runs both V layouts and checks them against the float64 bound and 6-sigma bar of tests/attn_ref64.py; with Lk a
multiple of 128 the two layouts must also agree bit for bit."""
import math

import pytest
import torch

from tests import attn_ref64
from tests.test_attn_chunk_gate_gpu import SEQ, chunked_vt, gated, rotated, ungated
from tests.test_attn_lazy_rescale_gpu import operands, ref64, rel, run_both, spike

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)
TOL = 5e-3


def check(q, k, v, heads=1, rows=None):
    """Both layouts against fp64 and attn_ref64 (rows `rows` only when given); returns the token-major output."""
    want = ref64(q, k, v, heads)
    o_vt, o_tok = run_both(q, k, v, heads)
    for o in (o_vt, o_tok):
        if o is None:
            continue
        sel = slice(None) if rows is None else rows
        assert torch.isfinite(o[sel].float()).all()
        assert rel(o[sel], want[sel]) < TOL, rel(o[sel], want[sel])
        attn_ref64.check(o, q, k, v, heads, LN2, rows=rows)
    if o_vt is not None:
        assert torch.equal(o_vt.nan_to_num(), o_tok.nan_to_num())
    return o_tok


def thread_columns(q_lane, n):
    """The first n columns of a 128-key tile held by quad thread q_lane (lane % 4): 8 i + 2 q_lane + {0, 1}"""
    cols = [8 * i + 2 * q_lane + e for i in range(16) for e in (0, 1)]
    return cols[:n]


@pytest.mark.parametrize("value,spread", [(19.875, False), (20.0, False), (21.875, True), (22.0, True)])
def test_guard_edges(value, spread):
    """Tile 0 sets m = 0 (one key at 0 over a background at -1).  Tile 3 holds 16 keys at `value` above it: all in the
    columns of quad thread 1 (its partial sum 16 * 2^value: 2^23.875 is accepted, 2^24 falls back) or spread 4 per quad
    thread (4 * 2^value: 2^23.875 accepted, 2^24 falls back).  An accepted tile keeps P up to 2^21.875 against the
    stale m; a fallback moves m.  Tile 5 holds one more key 30 above the first block, which always falls back."""
    Lq, Lk = 256, 1024
    q, k, v = operands(Lq, Lk, seed=11, background=-1.0)
    spike(k, [5], 0.0)
    if spread:
        cols = [c for ql in range(4) for c in thread_columns(ql, 4)]
    else:
        cols = thread_columns(1, 16)
    spike(k, [3 * 128 + c for c in cols], value)
    spike(k, [5 * 128 + 100], value + 30.0)
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


def test_staircase_falls_back_every_tile():
    """Every key of tile j scores 30 j - 1 (one at 30 j): the row max rises by 30 per tile over 55 tiles, so every
    steady-state tile, in both ring stages, fails the guard (its partial sums reach 2^34) and is redone exactly."""
    Lq, Lk = 256, 55 * 128
    tile = torch.arange(Lk, device="cuda") // 128
    q, k, v = operands(Lq, Lk, seed=12, background=(30.0 * tile - 1.0))
    spike(k, torch.arange(55, device="cuda") * 128 + 77, 30.0 * torch.arange(55, device="cuda", dtype=torch.float32))
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


@pytest.mark.parametrize("Lk", [677, 1061])
def test_fallback_in_masked_tail(Lk):
    """Token-major V, ragged Lk: the partial last tile holds a key 35 above a background at -30, so it falls back, and
    the redone S must be masked past Lk again: the zero-filled keys there score 0, 2^30 above the reference."""
    Lq = 200
    n_full = Lk // 128
    q, k, v = operands(Lq, Lk, seed=13, background=-30.0)
    spike(k, [n_full * 128 + 20], 5.0)
    q, k, v = (t.to(torch.bfloat16) for t in (q, k, v))
    want = ref64(q, k, v, 1)
    _, o = run_both(q, k, v, 1)
    assert torch.isfinite(o.float()).all()
    assert rel(o, want) < TOL, rel(o, want)
    attn_ref64.check(o, q, k, v, 1, LN2)


@pytest.mark.parametrize("row,jump", [(0, 30.0), (93, 150.0), (127, 30.0), (70, 150.0)])
def test_fallback_in_one_warp(row, jump):
    """Only query `row` scores one key of tile 2 `jump` above its reference: one thread of one warp fails the guard, the
    other three warps of its warpgroup pass, and the warpgroup vote must take all four into the fallback (its wgmma
    needs them all).  Rows 0, 70, 93 and 127 sit in different warps of both consumer warpgroups."""
    Lq, Lk = 128, 640
    q, k, v = operands(Lq, Lk, seed=14, background=-1.0)
    q[row, 1] = 1.0
    spike(k, [2 * 128 + 9], jump, dim=1)
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


def test_nan_row():
    """A NaN in one query makes its whole score row NaN: that row's guard fails on every tile and its output is NaN,
    as before the guard; every other row, including the other rows of its warpgroup, stays exact."""
    Lq, Lk, row = 128, 768, 37
    q, k, v = operands(Lq, Lk, seed=15, background=-1.0)
    q, k, v = (t.to(torch.bfloat16) for t in (q, k, v))
    q[row, 2] = float("nan")
    others = torch.tensor([r for r in range(Lq) if r != row], device="cuda")
    o = check(q, k, v, rows=others)
    assert torch.isnan(o[row].float()).all()


def test_large_v_near_fp32_range():
    """No noise in the scores: tile 0 scores 0 and every later key 18.875, so each thread's partial sums are 32 *
    2^18.875 = 2^23.875 and every tile is accepted with P = 2^18.875 against m = 0.  With |v| ~ 2^90 the fp32
    accumulator O reaches about 2^120 over 55 tiles, within 2^8 of the fp32 range, and must stay finite and exact."""
    Lq, Lk = 128, 55 * 128
    tile = torch.arange(Lk, device="cuda") // 128
    q, k, v = operands(Lq, Lk, seed=16, background=torch.where(tile == 0, 0.0, 18.875))
    k[:, 2:] = 0.0
    v = v * 2.0 ** 90
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


@pytest.mark.parametrize("heads,Lq,Lk", [(2, 1000, 1024), (4, 256, 55 * 128)])
def test_ordinary_inputs(heads, Lq, Lk):
    """Random q, k, v at the default scale: no steady-state tile comes near the guard, and the outputs meet the same
    element bound and 6-sigma bar as any other input."""
    from gen3c_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(17)
    q, k, v = (torch.randn(n, heads * 128, device="cuda", generator=g).to(torch.bfloat16) for n in (Lq, Lk, Lk))
    o = ops.attention(q, k, v.T.contiguous(), heads)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5)


@pytest.mark.parametrize("chunks,cl", [(2, 384), (4, 256)])
def test_gated_fallbacks_match_rotated(chunks, cl):
    """The context-parallel gate with fallbacks: keys rise by 30 per tile, so every steady-state tile falls back, and a
    gated launch from each first chunk must be bitwise the ungated kernel on chunks rotated to start there."""
    Lq, Lk = 256, chunks * cl
    tile = torch.arange(Lk, device="cuda") // 128
    q, k, v = operands(Lq, Lk, seed=18, background=(30.0 * tile - 1.0))
    q, k, v = (t.to(torch.bfloat16) for t in (q, k, v))
    vt = chunked_vt(v, chunks)
    flags = torch.full((chunks,), SEQ, device="cuda", dtype=torch.int32)
    for first in range(chunks):
        o, wait = gated(q, k, vt, 1, first, flags, scale=LN2)
        assert wait == 0
        kr, vtr = rotated(k, vt, first)
        assert torch.equal(o, ungated(q, kr, vtr, 1, scale=LN2)), first
        attn_ref64.check(o, q, k, v, 1, LN2, label=f"chunks={chunks} first={first}")
