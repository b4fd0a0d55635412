"""The DiT engine's single-GPU forward, replayed bit for bit from the per-operator entry points of gen3c_b200.ops.

The engine's other correctness tests compare against oracles with rel-L2 bars (5e-3 per forward), and the whole fp8
Linear mode moves the output by only about 5e-4 against bf16.  A forward that ran one Linear in the wrong precision, or
dropped a quantisation pass, could therefore still pass them.  This file rebuilds g3c_dit_forward from the same kernels
in the engine's order and with its arguments, and requires torch.equal: the kernels use no split-K and no atomics, so
the same launches give the same bits.  A mismatch means the replay has an order or an argument wrong, or the engine
changed.  It also pins the engine's launches per profiling category.

Inputs the engine derives itself are read back (the adaLN vectors through g3c_dit_read_modulation, the RoPE and abs-pos
tables through g3c_dit_read_tables) or rebuilt exactly: the query gain, the padded patch weight, patchify and
unpatchify.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gen3c_b200 import _lib, ops
from oracle import cases, dit_oracle
from tests.test_engine_signal_gpu import WIDER, build_net

pytestmark = pytest.mark.gpu

bf = torch.bfloat16
LN2 = 0.6931471805599453  # the attention scale: 1/sqrt(128) * log2(e) is folded into the query gain
# that factor as the engine computes it: a product of two fp32 constants, rounded to fp32
Q_SCALE = np.float32(0.08838834764831845) * np.float32(1.4426950408889634)
CATEGORIES = ("gemm", "attn_self", "attn_cross", "eltwise", "comm", "vector")


def engine_forward(net, x, mask, pose, pad, timestep, ctx):
    """g3c_dit_forward with profiling on: (output [16, T, H, W] bf16, launches per category)."""
    lib, h = _lib.load(), net._engine()
    out = torch.empty_like(x)
    _lib.check(lib.g3c_dit_profile(h, 1), "g3c_dit_profile")
    _lib.check(lib.g3c_dit_forward(h, _lib.ptr(x), _lib.ptr(mask), _lib.ptr(pose), _lib.ptr(pad), timestep,
                                   _lib.ptr(ctx), out.data_ptr(), _lib.stream_ptr()), "g3c_dit_forward")
    ms, n = (C.c_float * 6)(), (C.c_int * 6)()
    _lib.check(lib.g3c_dit_profile_read(h, ms, n, 6), "g3c_dit_profile_read")
    _lib.check(lib.g3c_dit_profile(h, 0), "g3c_dit_profile")
    assert net.last_launch_count() == sum(n)
    return out, dict(zip(CATEGORIES, n))


def engine_derived(net, timestep, L, D):
    """The engine's adaLN vectors at `timestep` and its forward's RoPE / abs-pos tables (first frame 0)."""
    lib, h = _lib.load(), net._engine()
    mods = torch.empty((net.num_blocks * 3, 3 * D), device="cuda")
    modf = torch.empty(2 * D, device="cuda")
    rope = torch.empty((L, 128), device="cuda")
    pos = torch.empty((L, D), device="cuda", dtype=bf)
    _lib.check(lib.g3c_dit_read_modulation(h, timestep, _lib.ptr(mods), _lib.ptr(modf), _lib.stream_ptr()),
               "g3c_dit_read_modulation")
    _lib.check(lib.g3c_dit_read_tables(h, 0, _lib.ptr(rope), _lib.ptr(pos), _lib.stream_ptr()), "g3c_dit_read_tables")
    return mods, modf, rope, pos


def replay(sd, cfg, x_in, mask, pose, pad, ctx, mods, modf, rope, pos, fp8):
    """g3c_dit_forward restated with gen3c_b200.ops.  In fp8 mode the eight large Linears of a block (self-attention
    q / k / v / out, cross-attention q / out, MLP layer1 / layer2) take e4m3 codes of their weight and their activation
    rows: xn straight from the fused LN-modulate, att and hid from a separate quantisation pass."""
    D, heads, Co = cfg.model_channels, cfg.num_heads, cfg.out_channels
    _, T, H, W = x_in.shape
    Hp, Wp = H // 2, W // 2
    L, M = T * Hp * Wp, ctx.shape[0]
    gated = dict(epilogue=ops.EPI_GATED_RESIDUAL_F32)

    def linear(a, w, **kw):  # a . w^T; a is bf16 rows, or (codes, scales) in fp8 mode
        return ops.gemm_fp8(*a, *ops.quantize_rows_fp8(w), **kw) if fp8 else ops.gemm(a, w, **kw)

    def linear_vt(a, w):  # (a . w^T)^T = w . a^T, the operands swapped
        return ops.gemm_fp8(*ops.quantize_rows_fp8(w), *a) if fp8 else ops.gemm(w, a)

    def norm_rope(a, w, gamma, cs):
        if fp8:
            return ops.gemm_norm_rope_fp8(*a, *ops.quantize_rows_fp8(w), gamma, cs)
        return ops.gemm_norm_rope(a, w, gamma, cs)

    def rows(t):  # a bf16 activation that feeds an fp8 Linear is quantised in a pass of its own
        return ops.quantize_rows_fp8(t) if fp8 else t

    def ln_mod(m, p=None):  # x += p in place, then LN(x) * (1 + scale) + shift
        return (ops.ln_modulate_fp8 if fp8 else ops.ln_modulate)(x, m[:D], m[D:2 * D], pos=p)

    # patch embedding: column c*4 + m*2 + n of token (t, h, w) is channel c at (2h + m, 2w + n); zero-padded columns
    if pose is None:
        pose = torch.zeros((cfg.in_channels - 17, T, H, W), device="cuda", dtype=bf)
    src = torch.cat([x_in, mask, pose, pad.expand(1, T, H, W)])
    tok = src.reshape(-1, T, Hp, 2, Wp, 2).permute(1, 2, 4, 0, 3, 5).reshape(L, -1)
    w_patch = sd["x_embedder.proj.1.weight"]
    kpad = (w_patch.shape[1] + 63) // 64 * 64
    tok = F.pad(tok, (0, kpad - tok.shape[1])).contiguous()
    x = ops.gemm(tok, F.pad(w_patch, (0, kpad - w_patch.shape[1])).contiguous(), ops.EPI_F32)

    q_scale = torch.tensor(float(Q_SCALE), dtype=torch.float32, device="cuda")
    for i in range(cfg.num_blocks):
        p = f"blocks.block{i}.blocks."
        for j, cs in ((0, rope), (1, None)):
            a = f"{p}{j}.block.attn."
            m = mods[3 * i + j]
            gq = sd[a + "to_q.1.weight"].float() * q_scale
            gk = sd[a + "to_k.1.weight"].float()
            if j == 0:  # self-attention, the abs-pos table added to x first
                xn = ln_mod(m, pos)
                k = norm_rope(xn, sd[a + "to_k.0.weight"], gk, cs)
                vt = linear_vt(xn, sd[a + "to_v.0.weight"])
            else:  # cross-attention to the text context, whose K / V^T stay bf16
                xn = ln_mod(m)
                k = ops.gemm_norm_rope(ctx, sd[a + "to_k.0.weight"], gk, None)
                vt = ops.gemm(sd[a + "to_v.0.weight"], ctx)
            q = norm_rope(xn, sd[a + "to_q.0.weight"], gq, cs)
            att = ops.attention(q, k, vt, heads, scale=LN2, vt_chunk_len=L if j == 0 else M)
            linear(rows(att), sd[a + "to_out.0.weight"], out=x, gate=m[2 * D:], **gated)
        m = mods[3 * i + 2]
        hid = linear(ln_mod(m), sd[p + "2.block.layer1.weight"], epilogue=ops.EPI_GELU_BF16)
        linear(rows(hid), sd[p + "2.block.layer2.weight"], out=x, gate=m[2 * D:], **gated)

    xn = ops.ln_modulate(x, modf[:D], modf[D:])
    y = ops.gemm(xn, sd["final_layer.linear.weight"], ops.EPI_F32, block_n=64)
    # unpatchify: column (p1*2 + p2)*C + c of token (t, h, w) -> channel c at (2h + p1, 2w + p2)
    return y.reshape(T, Hp, Wp, 2, 2, Co).permute(5, 0, 1, 3, 2, 4).reshape(Co, T, H, W).to(bf)


REPLAY_CASES = {
    "tiny": (cases.TINY, cases.TINY_SHAPE),  # L = 128: one query and one KV tile
    "wider_3tiles": (WIDER, dict(T=3, H=16, W=32, ctx_len=256)),  # L = 384 on a non-square grid, 2 context tiles
}


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("case", list(REPLAY_CASES))
@torch.no_grad()
def test_engine_forward_equals_operator_replay(case, fp8):
    """Two forwards at one timestep (cond: pose given; uncond: no pose, the other context), each torch.equal to its
    replay; launches per category of each; and, in fp8 mode, the bf16 replay must differ from the engine output."""
    cfg, shp = REPLAY_CASES[case]
    T, H, W, M = shp["T"], shp["H"], shp["W"], shp["ctx_len"]
    B, D, L = cfg.num_blocks, cfg.model_channels, T * (H // 2) * (W // 2)
    sd = dit_oracle.random_state_dict(cfg, seed=2)
    inp = cases.dit_inputs(cfg, **shp, seed=4)
    g = torch.Generator().manual_seed(5)
    inp["padding"] = (torch.rand(H, W, generator=g) < 0.3).float()  # the padding-mask channel is not all zero
    d = lambda t: t.to(bf).cuda().contiguous()  # noqa: E731
    x, mask, pose, pad = d(inp["x"]), d(inp["cond_mask"]), d(inp["pose"]), d(inp["padding"])
    ctx_c, ctx_u, ts = d(inp["ctx_c"]), d(inp["ctx_u"]), inp["timestep"]

    net = build_net(cfg, sd, fp8)
    net._sync_weights()
    net._set_shape(T, H, W, M, 24.0)
    out_c, n_first = engine_forward(net, x, mask, pose, pad, ts, ctx_c)
    out_u, n_second = engine_forward(net, x, mask, None, pad, ts, ctx_u)

    eltwise = 3 * B + 3 + (3 * B if fp8 else 0)
    want = dict(gemm=10 * B + 2, attn_self=B, attn_cross=B, eltwise=eltwise, comm=0, vector=6 * B + 5)
    assert n_first == want
    assert n_second == dict(want, vector=0)  # the adaLN vectors of this timestep are reused

    derived = engine_derived(net, ts, L, D)
    wsd = {k: v for k, v in net.state_dict().items() if k != "pos_embedder.seq"}
    for out, p, ctx in ((out_c, pose, ctx_c), (out_u, None, ctx_u)):
        ref = replay(wsd, cfg, x, mask, p, pad, ctx, *derived, fp8)
        torch.cuda.synchronize()
        assert torch.equal(out, ref), float((out.float() - ref.float()).abs().max())
    assert not torch.equal(out_c, out_u)
    if fp8:
        assert not torch.equal(out_c, replay(wsd, cfg, x, mask, pose, pad, ctx_c, *derived, False))
