"""The lazy rescale of the attention kernel's online softmax (gen3c_b200/csrc/attn_wgmma.cu, softmax_tile): the reference
row max m moves, and O and the row sums are rescaled, only when some row of a warp's 16 exceeds m by more than 8 in
log2 units; otherwise the tile is exponentiated against the stale m, so P <= 2^8.  Each test builds scores whose row
maxima are known exactly (scale = ln 2: S is in log2 units), runs both V layouts (V^T through g3c_attn_fwd,
token-major V through g3c_attn_fwd_sbhd) and compares with an fp64 softmax.  With Lk a multiple of 128 the two layouts
must also agree bit for bit.  Both outputs also pass the float64 checks of tests/attn_ref64.py."""
import math

import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)
TOL = 5e-3


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def ref64(q, k, v, heads):
    """fp64 softmax(q k^T) v per head, scores in log2 units."""
    Lq, Lk = q.shape[0], k.shape[0]
    qh, kh, vh = (t.double().view(t.shape[0], heads, 128).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(1, 2)
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    o = (p @ vh) / p.sum(-1, keepdim=True)
    return o.transpose(0, 1).reshape(Lq, heads * 128)


def run_both(q, k, v, heads):
    """(o with V^T or None when Lk % 128 != 0, o with token-major V), both [Lq, heads*128]"""
    from gen3c_b200 import ops

    Lq, Lk = q.shape[0], k.shape[0]
    o_vt = ops.attention(q, k, v.T.contiguous(), heads, scale=LN2) if Lk % 128 == 0 else None
    o_tok = ops.attention_sbhd(q.view(Lq, 1, heads, 128), k.view(Lk, 1, heads, 128), v.view(Lk, 1, heads, 128),
                               scale=LN2).view(Lq, heads * 128)
    return o_vt, o_tok


def check(q, k, v, heads=1):
    want = ref64(q, k, v, heads)
    o_vt, o_tok = run_both(q, k, v, heads)
    for o in (o_vt, o_tok):
        if o is None:
            continue
        assert torch.isfinite(o.float()).all()
        assert rel(o, want) < TOL, rel(o, want)
        attn_ref64.check(o, q, k, v, heads, LN2)
    if o_vt is not None:
        assert torch.equal(o_vt, o_tok)


def operands(Lq, Lk, seed, background):
    """Q and K whose scores are offset(key) + a small random term: dimension 0 of every query is 1 and dimension 0 of
    key n is `background[n]`; dimensions 2.. carry noise of std ~0.1 in the score.  Keys set later with k[n] = 0 except
    k[n, 0] (or k[n, 1] against q[r, 1]) score exactly that value."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(Lq, 128, device="cuda", generator=g) * 0.1
    k = torch.randn(Lk, 128, device="cuda", generator=g) * 0.1
    q[:, 0], q[:, 1] = 1.0, 0.0
    k[:, 0], k[:, 1] = background, 0.0
    v = torch.randn(Lk, 128, device="cuda", generator=g)
    return q, k, v


def spike(k, keys, value, dim=0):
    k[keys] = 0.0
    k[keys, dim] = value


@pytest.mark.parametrize("rise", [7.9, 8.0, 8.1])
def test_threshold_edges(rise):
    """Tile 0 sets m = 0 (a key scoring exactly 0 above a background near -1); tile 3 holds 16 keys scoring `rise`
    above it (bf16: 7.906, 8.0, 8.125) — stale at 7.9 and at exactly 8 (P = 2^8), rescaled at 8.1 — and tile 5 a
    second block another `rise` above, against whichever reference the first left."""
    Lq, Lk = 256, 1024
    q, k, v = operands(Lq, Lk, seed=1, background=-1.0)
    spike(k, [5], 0.0)
    spike(k, slice(3 * 128 + 40, 3 * 128 + 56), rise)
    spike(k, slice(5 * 128 + 100, 5 * 128 + 104), 2 * rise)
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


def test_staircase_drift():
    """The row max rises by 4 per tile over 55 tiles (to 216): no single step exceeds the threshold, but the growth
    since the reference does every third tile.  A rule comparing each tile's max with the previous tile's would never
    rescale and P = 2^216 would overflow."""
    Lq, Lk = 256, 55 * 128
    tile = torch.arange(Lk, device="cuda") // 128
    q, k, v = operands(Lq, Lk, seed=2, background=(4.0 * tile - 1.0))
    spike(k, torch.arange(55, device="cuda") * 128 + 77, 4.0 * torch.arange(55, device="cuda", dtype=torch.float32))
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


@pytest.mark.parametrize("row", [0, 93, 127])
def test_divergent_row_in_warp(row):
    """Only query `row` scores one key of tile 2 at 150 above its reference (through q[row, 1] = 1); the other 15 rows
    of its warp stay flat.  The warp must rescale for that one row: a decision that misses any row of the warp leaves
    it at P = 2^150, beyond bf16 and fp32.  Rows 0, 93 and 127 sit at different lanes of warps 0, 5 and 7."""
    Lq, Lk = 128, 640
    q, k, v = operands(Lq, Lk, seed=3, background=-1.0)
    q[row, 1] = 1.0
    spike(k, [2 * 128 + 9], 150.0, dim=1)
    check(*(t.to(torch.bfloat16) for t in (q, k, v)))


@pytest.mark.parametrize("Lk", [677, 1061])
def test_masked_tail_with_jump(Lk):
    """Token-major V, ragged Lk: the scores of the partial last tile are masked past Lk and the tile holds a jump of 35
    over a background at -30.  The rescale must take the masked keys' -inf in its stride; if the zero-filled keys past
    Lk (score 0) leaked in, each would weigh 2^-5 against the jump."""
    Lq = 200
    n_full = Lk // 128
    q, k, v = operands(Lq, Lk, seed=4, background=-30.0)
    spike(k, [n_full * 128 + 20], 5.0)
    q, k, v = (t.to(torch.bfloat16) for t in (q, k, v))
    want = ref64(q, k, v, 1)
    _, o = run_both(q, k, v, 1)
    assert torch.isfinite(o.float()).all()
    assert rel(o, want) < TOL, rel(o, want)
    attn_ref64.check(o, q, k, v, 1, LN2)
