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
import pytest
import torch

from oracle import cases, dit_oracle
from tests.engine_replay import engine_forward, launches, read_modulation, read_tables, replay
from tests.test_engine_signal_gpu import WIDER, build_net

pytestmark = pytest.mark.gpu

bf = torch.bfloat16


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
    B, L = cfg.num_blocks, T * (H // 2) * (W // 2)
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
    out_c, n_first, _ = engine_forward(net, x, mask, pose, pad, ts, ctx_c)
    out_u, n_second, _ = engine_forward(net, x, mask, None, pad, ts, ctx_u)

    assert n_first == launches(B, fp8)
    assert n_second == launches(B, fp8, vectors=False)  # the adaLN vectors of this timestep are reused

    mods, modf = read_modulation(net, ts)
    rope, pos = read_tables(net, 0, L)
    wsd = {k: v for k, v in net.state_dict().items() if k != "pos_embedder.seq"}

    def ref(p, ctx, fp8):
        return replay(wsd, cfg, [(x, mask, p, pad, rope, pos)], ctx, mods, modf, fp8)[0][0]

    for out, p, ctx in ((out_c, pose, ctx_c), (out_u, None, ctx_u)):
        want = ref(p, ctx, fp8)
        torch.cuda.synchronize()
        assert torch.equal(out, want), float((out.float() - want.float()).abs().max())
    assert not torch.equal(out_c, out_u)
    if fp8:
        assert not torch.equal(out_c, ref(pose, ctx_c, False))
