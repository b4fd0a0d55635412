"""DiT engine tests that can see the attention, RoPE and timestep paths.

With the weights of `random_state_dict` (std 0.02, q/k RMSNorm gains near 1) the gated attention branches move the
residual stream by about 1e-3, so an end-to-end rel-L2 bar of 5e-3 cannot tell a forward without self-attention,
cross-attention or RoPE from a correct one.  This file

1. runs the engine on test nets whose attention carries signal (q/k gains x2.5, to_v / to_out x6 in both attention
   sub-blocks) against the fp32 oracle, with the bar of test_fullsize_parity_gpu.py (no farther from fp32 than the
   oracle graph run in bf16) and oracle variants as negative controls: the engine output must be at least 3x farther
   from each broken graph than from the correct one, and each broken graph must miss the bar by 3x;
2. reads back the engine's RoPE / abs-pos tables and adaLN modulation vectors (g3c_dit_read_tables,
   g3c_dit_read_modulation) and checks them element by element against float64 restatements of the oracle.
"""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import cases, dit_oracle
from tests import fp8_oracle

pytestmark = pytest.mark.gpu

bf = torch.bfloat16
QK_GAIN, VO_SCALE = 2.5, 6.0

WIDER = dit_oracle.DitCfg(model_channels=512, num_blocks=3, num_heads=4, ffn_dim=2048, context_dim=128,
                          adaln_lora_dim=64, max_frames=8, max_h=16, max_w=16)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def signal_state_dict(cfg, seed):
    """random_state_dict with the q/k RMSNorm gains x QK_GAIN and to_v / to_out x VO_SCALE in the self- and the
    cross-attention of every block, rounded to bf16 again: the softmax is no longer near uniform and the attention
    branches move the residual stream by O(1e-1) instead of O(1e-3)."""
    sd = dit_oracle.random_state_dict(cfg, seed=seed)
    for i in range(cfg.num_blocks):
        for j in (0, 1):
            p = f"blocks.block{i}.blocks.{j}.block.attn."
            for k, f in (("to_q.1.weight", QK_GAIN), ("to_k.1.weight", QK_GAIN), ("to_v.0.weight", VO_SCALE),
                         ("to_out.0.weight", VO_SCALE)):
                sd[p + k] = (sd[p + k] * f).to(bf).float()
    return sd


@contextlib.contextmanager
def oracle_variant(name):
    """Patch dit_oracle (which tests/fp8_oracle.py also calls) into a broken graph:
    no_rope       every RoPE angle 0
    hw_swapped    the h columns of the angle table take the w position and the w columns the h position
    scale_log2e   softmax scale multiplied by log2(e)
    uniform_self  self-attention weights uniform over the keys
    ca_zeroed     cross-attention output 0
    The forward calls attention() for the self-attention, then for the cross-attention, block after block."""
    rope_angles, attention = dit_oracle.rope_angles, dit_oracle.attention
    calls = [0]

    def rope(cfg, T, Hp, Wp, fps, t0=0, device=None):
        a = rope_angles(cfg, T, Hp, Wp, fps, t0, device)
        if name == "no_rope":
            return torch.zeros_like(a)
        if name == "hw_swapped":
            n = max(Hp, Wp)
            sq = rope_angles(cfg, T, n, n, fps, t0, device).reshape(T, n, n, 128)
            tok = torch.arange(T * Hp * Wp)
            t, h, w = tok // (Hp * Wp), (tok // Wp) % Hp, tok % Wp
            return sq[t, w, h].reshape(-1, 128)
        return a

    def attn(q, k, v, heads):
        is_self = calls[0] % 2 == 0
        calls[0] += 1
        if name == "scale_log2e":
            return attention(q * math.log2(math.e), k, v, heads)
        if name == "uniform_self" and is_self:
            return v.mean(0, keepdim=True).expand(q.shape[0], -1).to(q.dtype)
        if name == "ca_zeroed" and not is_self:
            return torch.zeros_like(q)
        return attention(q, k, v, heads)

    dit_oracle.rope_angles, dit_oracle.attention = rope, attn
    try:
        yield
    finally:
        dit_oracle.rope_angles, dit_oracle.attention = rope_angles, attention


GRAPH_VARIANTS = ("no_rope", "hw_swapped", "scale_log2e", "uniform_self", "ca_zeroed")


def build_net(cfg, sd, fp8=False):
    from gen3c_b200.dit import VideoExtendGeneralDIT

    net = VideoExtendGeneralDIT(max_img_h=cfg.max_h * 2, max_img_w=cfg.max_w * 2, max_frames=cfg.max_frames,
                                in_channels=cfg.in_channels, out_channels=cfg.out_channels,
                                model_channels=cfg.model_channels, num_blocks=cfg.num_blocks, num_heads=cfg.num_heads,
                                crossattn_emb_channels=cfg.context_dim, adaln_lora_dim=cfg.adaln_lora_dim,
                                rope_h_extrapolation_ratio=cfg.rope_h_ratio, rope_w_extrapolation_ratio=cfg.rope_w_ratio,
                                rope_t_extrapolation_ratio=cfg.rope_t_ratio, base_fps=cfg.base_fps)
    net.load_state_dict({k: v.to(bf) for k, v in sd.items()}, strict=True)
    if fp8:
        net.enable_fp8_linear()
    return net


def engine_forward(net, inp, fps):
    d = lambda t: t.cuda().to(bf)  # noqa: E731
    T = inp["x"].shape[1]
    out = net(x=d(inp["x"])[None], timesteps=torch.tensor([inp["timestep"]], device="cuda", dtype=bf),
              crossattn_emb=d(inp["ctx_c"])[None], fps=torch.tensor([fps], device="cuda"),
              padding_mask=d(inp["padding"])[None, None], condition_video_input_mask=d(inp["cond_mask"])[None],
              condition_video_indicator=torch.zeros(1, 1, T, 1, 1, device="cuda", dtype=bf),
              condition_video_pose=d(inp["pose"])[None])
    return out[0].float().cpu()


def oracle_forward(cfg, sd, inp, fps, ctx="ctx_c", fp8=False, dtype=torch.float32):
    fwd = fp8_oracle.forward if fp8 else dit_oracle.forward
    return fwd(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp[ctx], fps=fps,
               compute_dtype=dtype).float()


# name: (config, weight seed, shape, input seed, fps, fp8 Linear mode, absolute cap on the engine's rel-L2)
SIGNAL_CASES = {
    "tiny_nonsquare": (cases.TINY, 0, dict(T=2, H=16, W=32, ctx_len=128), 1, 24.0, False, 1e-2),
    "wider_3kv_tiles": (WIDER, 7, dict(T=3, H=16, W=32, ctx_len=256), 11, 24.0, False, 2.5e-2),
    "wider_fps30": (WIDER, 7, dict(T=3, H=16, W=32, ctx_len=256), 11, 30.0, False, 2.5e-2),
    "tiny_nonsquare_fp8": (cases.TINY, 0, dict(T=2, H=16, W=32, ctx_len=128), 1, 24.0, True, 3e-2),
}


@pytest.mark.parametrize("case", list(SIGNAL_CASES))
@torch.no_grad()
def test_engine_forward_carries_attention_signal(case):
    """Engine vs the fp32 oracle (fp8 mode: vs tests/fp8_oracle.py) on a net whose attention matters.  Bar: no farther
    than the same graph run in bf16, and under an absolute cap.  Controls: every broken graph of oracle_variant, the
    uncond text context in place of the cond one, and (at fps 30) the fps-24 position table."""
    cfg, seed, shp, iseed, fps, fp8, cap = SIGNAL_CASES[case]
    sd = signal_state_dict(cfg, seed)
    inp = cases.dit_inputs(cfg, **shp, seed=iseed)
    want = oracle_forward(cfg, sd, inp, fps, fp8=fp8)
    floor = rel(oracle_forward(cfg, sd, inp, fps, fp8=fp8, dtype=torch.bfloat16), want)
    got = engine_forward(build_net(cfg, sd, fp8), inp, fps)
    err = rel(got, want)
    bad = {}
    # the fp8 graph's own bf16-storage spread is 2.2x below the scale error; the scale fold is the same in both modes
    for v in (v for v in GRAPH_VARIANTS if not (fp8 and v == "scale_log2e")):
        with oracle_variant(v):
            bad[v] = oracle_forward(cfg, sd, inp, fps, fp8=fp8)
    bad["ctx_swapped"] = oracle_forward(cfg, sd, inp, fps, ctx="ctx_u", fp8=fp8)
    if fps != 24.0:
        bad["fps_24"] = oracle_forward(cfg, sd, inp, 24.0, fp8=fp8)
    print(f"{case}: engine vs oracle rel-L2 {err:.3e}, bf16 graph {floor:.3e}; controls: "
          + ", ".join(f"{k} {rel(b, want):.2e} (engine {rel(got, b):.2e})" for k, b in bad.items()))
    assert err <= floor and err < cap, (err, floor)
    for k, b in bad.items():
        assert rel(b, want) >= 3 * floor, (k, rel(b, want), floor)
        assert rel(got, b) >= 3 * err, (k, rel(got, b), err)


@torch.no_grad()
def test_denoise_step_guidance_through_cross_attention():
    """One g3c_denoise_step whose cond and uncond branches differ only in the text context (same input mask, no pose
    in either), so the guidance term g * (cond - uncond) exists only through the cross-attention.  The CFG-combined
    network output and x_{t-1} are held to the bf16-graph bar; a step whose branches swap contexts, or whose
    cross-attention is zeroed (guidance term 0), misses by 3x."""
    from gen3c_b200 import sampler

    cfg = cases.TINY
    shp = dict(T=2, H=16, W=32, ctx_len=128)
    T, H, W = shp["T"], shp["H"], shp["W"]
    sd = signal_state_dict(cfg, 0)
    sig = dit_oracle.karras_sigmas(35)
    sigma, sigma_next, guidance = float(sig[20]), float(sig[21]), 1.5
    inp = cases.dit_inputs(cfg, **shp, x_scale=math.sqrt(sigma ** 2 + 0.25))
    noise = torch.from_numpy(dit_oracle.arch_invariant_rand((16, T, H, W), 1))
    ind = torch.zeros(T)
    ind[0] = 1.0

    def step(dtype=torch.float32, swap=False):
        def onet(x_in, t, cond):
            c = cond != swap
            return dit_oracle.forward(sd, cfg, x_in, inp["cond_mask"], None, inp["padding"], t,
                                      inp["ctx_c"] if c else inp["ctx_u"], compute_dtype=dtype).float()

        return dit_oracle.denoise_step(onet, inp["x"], inp["gt"], noise, ind, sigma, sigma_next, guidance,
                                       return_net_output=True)

    want_x, want_o = step()
    floor_x, floor_o = (rel(a, b) for a, b in zip(step(torch.bfloat16), (want_x, want_o)))
    net = build_net(cfg, sd)
    c = lambda t: t.cuda().to(bf)  # noqa: E731
    net_o = torch.empty((16, T, H, W), device="cuda", dtype=bf)
    got_x = sampler.denoise_step(net, c(inp["x"]), c(inp["gt"]), noise.cuda(), ind.cuda(), c(inp["cond_mask"]), None,
                                 c(inp["padding"]), c(inp["ctx_c"]), c(inp["ctx_u"]), sigma, sigma_next,
                                 guidance, net_output=net_o).float().cpu()
    got_o = net_o.float().cpu()
    e_x, e_o = rel(got_x, want_x), rel(got_o, want_o)
    bad = {"ctx_swapped": step(swap=True)}
    with oracle_variant("ca_zeroed"):
        bad["ca_zeroed"] = step()
    print(f"denoise step: net_output {e_o:.3e} (bf16 graph {floor_o:.3e}), x_next {e_x:.3e} (bf16 graph {floor_x:.3e}); "
          + ", ".join(f"{k} net_output {rel(b[1], want_o):.2e} x_next {rel(b[0], want_x):.2e}" for k, b in bad.items()))
    assert e_o <= floor_o and e_o < 2e-2, (e_o, floor_o)
    assert e_x <= floor_x and e_x < 5e-3, (e_x, floor_x)
    for k, (bx, bo) in bad.items():
        assert rel(bo, want_o) >= 3 * floor_o and rel(got_o, bo) >= 3 * e_o, k
        assert rel(bx, want_x) >= 3 * floor_x and rel(got_x, bx) >= 3 * e_x, k


# ---------------------------------------------------------------------------------------------------------------------
# read-back of the position tables and the modulation vectors
# ---------------------------------------------------------------------------------------------------------------------
def table_cfg(ratios=(1.0, 1.0, 2.0)):
    # the benchmark's 44 x 80 patch grid fits; D = 256 keeps the weights small
    return dit_oracle.DitCfg(model_channels=256, num_blocks=1, num_heads=2, ffn_dim=1024, context_dim=64,
                             adaln_lora_dim=32, max_frames=16, max_h=48, max_w=88, rope_h_ratio=ratios[0],
                             rope_w_ratio=ratios[1], rope_t_ratio=ratios[2])


def engine_handle(cfg, sd, T, Hp, Wp, fps, ctx_len=128):
    net = build_net(cfg, sd)
    net._sync_weights()
    net._set_shape(T, 2 * Hp, 2 * Wp, ctx_len, fps)
    return net


def read_tables(net, t0):
    from gen3c_b200 import _lib

    T, H, W = net._shape_key[:3]
    L, D = T * (H // 2) * (W // 2), net.model_channels
    rope = torch.full((L, 128), float("nan"), device="cuda")
    pos = torch.full((L, D), float("nan"), device="cuda", dtype=bf)
    rc = _lib.load().g3c_dit_read_tables(net._engine(), t0, _lib.ptr(rope), _lib.ptr(pos), _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc, rope.cpu(), pos.cpu()


def rope_angles64(cfg, T, Hp, Wp, fps, t0):
    """dit_oracle.rope_angles in float64: [T*Hp*Wp, 128] angles, columns t | h | w (22 | 21 | 21) twice."""
    dim = 128
    dim_h = dim // 6 * 2
    dim_t = dim - 2 * dim_h

    def freqs(ratio, d):
        theta = 10000.0 * ratio ** (d / (d - 2))
        return 1.0 / theta ** (np.arange(0, d, 2)[: d // 2] / d)

    ft, fh, fw = freqs(cfg.rope_t_ratio, dim_t), freqs(cfg.rope_h_ratio, dim_h), freqs(cfg.rope_w_ratio, dim_h)
    t = (t0 + np.arange(T)) / fps * cfg.base_fps
    a = np.concatenate([
        np.broadcast_to(np.outer(t, ft)[:, None, None], (T, Hp, Wp, ft.size)),
        np.broadcast_to(np.outer(np.arange(Hp), fh)[None, :, None], (T, Hp, Wp, fh.size)),
        np.broadcast_to(np.outer(np.arange(Wp), fw)[None, None, :], (T, Hp, Wp, fw.size)),
    ], axis=-1).reshape(-1, 64)
    return np.concatenate([a, a], axis=1)


def rope_bound(ang):
    """|engine - float64| allowed per element of the cos|sin table.  The engine takes fp32 frequencies
    1 / theta^(2j/d): the fp32 exponent's rounding is multiplied by ln(theta) ~ 10, which puts the angle up to ~8 ulp
    from the exact one; sincosf adds about one ulp of a value <= 1."""
    return 16 * np.spacing(np.abs(ang).astype(np.float32)).astype(np.float64) + 2.0 ** -22


def abs_pos64(sd, cfg, T, Hp, Wp, t0):
    """dit_oracle.abs_pos_emb in float64: v = pos_t + pos_h + pos_w, v / (1e-6 + ||v|| / sqrt(D))."""
    et = sd["extra_pos_embedder.pos_emb_t"].double()[t0:t0 + T]
    eh = sd["extra_pos_embedder.pos_emb_h"].double()[:Hp]
    ew = sd["extra_pos_embedder.pos_emb_w"].double()[:Wp]
    v = (et[:, None, None] + eh[None, :, None] + ew[None, None, :]).reshape(T * Hp * Wp, -1)
    return v / (1e-6 + v.norm(dim=-1, keepdim=True) / math.sqrt(v.shape[1]))


def bf16_ulp(x):
    """spacing of bf16 at |x| (the larger one at a power of two)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize("ratios", [(1.0, 1.0, 2.0), (1.5, 2.0, 3.0)])
@pytest.mark.parametrize("T,Hp,Wp", [(2, 44, 80), (3, 8, 16), (3, 16, 8)])
@pytest.mark.parametrize("fps", [24.0, 30.0, 12.5])
def test_position_tables_match_float64(ratios, T, Hp, Wp, fps):
    """The RoPE cos|sin table per element within 16 ulp of the angle + 2^-22, layout checked exactly; the abs-pos
    table within one bf16 ulp of float64 rounded to bf16; for first frames t0 = 0, 5 and max_frames - T.  The tables
    of t0 +- 1 must miss both bounds; t0 + T > max_frames is G3C_EINVAL and writes nothing."""
    cfg = table_cfg(ratios)
    sd = dit_oracle.random_state_dict(cfg, seed=3)
    net = engine_handle(cfg, sd, T, Hp, Wp, fps)
    # the float64 restatements are the oracle's own arithmetic
    assert np.allclose(rope_angles64(cfg, T, Hp, Wp, fps, 5), dit_oracle.rope_angles(cfg, T, Hp, Wp, fps, 5).numpy(),
                       rtol=1e-5, atol=1e-6)
    assert rel(abs_pos64(sd, cfg, T, Hp, Wp, 5), dit_oracle.abs_pos_emb(sd, cfg, T, Hp, Wp, 5)) < 1e-6

    def rope_ok(cs, t0):
        ang = rope_angles64(cfg, T, Hp, Wp, fps, t0)
        ref = np.concatenate([np.cos(ang[:, :64]), np.sin(ang[:, 64:])], axis=1)
        ratio = np.abs(cs.double().numpy() - ref) / rope_bound(ang)
        return float(ratio.max())

    def pos_ok(pos, t0):
        ref = abs_pos64(sd, cfg, T, Hp, Wp, t0)
        return float(((pos.double() - ref.to(bf).double()).abs() / bf16_ulp(ref)).max())

    last = cfg.max_frames - T
    for t0 in (0, 5, last):
        rc, cs, pos = read_tables(net, t0)
        assert rc == 0
        r_rope, r_pos = rope_ok(cs, t0), pos_ok(pos, t0)
        print(f"t0 {t0}: rope error / bound {r_rope:.3f}, abs-pos error / bf16 ulp {r_pos:.3f}")
        assert r_rope <= 1.0 and r_pos <= 1.0, (t0, r_rope, r_pos)
        # layout: t columns depend on the frame only, h columns on the row only, w columns on the column only
        g = cs.reshape(T, Hp, Wp, 2, 64)
        assert torch.equal(g[..., :22], g[:, :1, :1, :, :22].expand_as(g[..., :22]))
        assert torch.equal(g[..., 22:43], g[:1, :, :1, :, 22:43].expand_as(g[..., 22:43]))
        assert torch.equal(g[..., 43:], g[:1, :1, :, :, 43:].expand_as(g[..., 43:]))
        for t_other in (t0 - 1, t0 + 1):
            if 0 <= t_other <= last:
                assert rope_ok(cs, t_other) > 10 and pos_ok(pos, t_other) > 10, t_other
    for t0 in (last + 1, -1):
        rc, cs, pos = read_tables(net, t0)
        assert rc == -1  # G3C_EINVAL
        assert torch.isnan(cs).all() and torch.isnan(pos.float()).all()


def modulation64(sd, cfg, timestep):
    """The adaLN vectors of dit_oracle.forward in float64 on the bf16 weights: mods [num_blocks*3, 3D], modf [2D]."""
    D = cfg.model_channels
    dev = sd["t_embedder.1.linear_1.weight"].device
    half = D // 2
    e = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64, device=dev) / half)
    s = torch.cat([torch.cos(timestep * e), torch.sin(timestep * e)])
    w = lambda k: sd[k].to(torch.float64)  # noqa: E731
    h1 = w("t_embedder.1.linear_1.weight") @ s
    lora = w("t_embedder.1.linear_2.weight") @ torch.nn.functional.silu(h1)
    emb = s * torch.rsqrt(s.pow(2).mean() + 1e-6) * w("affline_norm.weight")

    def mod(prefix, n):
        a = w(prefix + "adaLN_modulation.1.weight") @ torch.nn.functional.silu(emb)
        return w(prefix + "adaLN_modulation.2.weight") @ a + lora[: n * D]

    mods = torch.stack([mod(f"blocks.block{i}.blocks.{j}.", 3) for i in range(cfg.num_blocks) for j in range(3)])
    return mods, mod("final_layer.", 2)


def read_modulation(net, timestep):
    from gen3c_b200 import _lib

    D = net.model_channels
    mods = torch.full((net.num_blocks * 3, 3 * D), float("nan"), device="cuda")
    modf = torch.full((2 * D,), float("nan"), device="cuda")
    _lib.check(_lib.load().g3c_dit_read_modulation(net._engine(), timestep, _lib.ptr(mods), _lib.ptr(modf),
                                                   _lib.stream_ptr()), "g3c_dit_read_modulation")
    torch.cuda.synchronize()
    return mods, modf


def modulation_errors(got, want, D):
    """largest rel-L2 over the shift / scale / gate vectors of every sub-block and the final layer's shift / scale."""
    (gm, gf), (wm, wf) = got, want
    vecs = [(gm[r, c * D:(c + 1) * D], wm[r, c * D:(c + 1) * D]) for r in range(gm.shape[0]) for c in range(3)]
    vecs += [(gf[c * D:(c + 1) * D], wf[c * D:(c + 1) * D]) for c in range(2)]
    return max(rel(a, b) for a, b in vecs)


MOD_CASES = {
    # D = 256 with a LoRA width of 40: K tails of the D x R and 3D x R products
    "d256": dict(model_channels=256, num_blocks=2, num_heads=2, ffn_dim=1024, context_dim=64, adaln_lora_dim=40,
                 max_frames=8, max_h=8, max_w=8),
    # the 7B net's vector widths (D = 4096, R = 256) on one block
    "d4096": dict(model_channels=4096, num_blocks=1, num_heads=32, ffn_dim=16384, context_dim=1024,
                  adaln_lora_dim=256, max_frames=8, max_h=8, max_w=8),
}


@pytest.mark.parametrize("case", list(MOD_CASES))
@torch.no_grad()
def test_modulation_vectors_match_float64(case):
    """Every adaLN vector (per sub-block shift / scale / gate, final shift / scale) within rel 1e-5 of float64 at three
    timesteps.  The per-timestep cache: reading at t1, a forward at t1, then a read at t2 equals a fresh handle's read
    at t2; a forward after a read at the same t reuses the vectors bit for bit.  After g3c_dit_load of one
    adaLN_modulation weight the vectors follow the new weight."""
    cfg = dit_oracle.DitCfg(**MOD_CASES[case])
    D = cfg.model_channels
    sd = dit_oracle.random_state_dict_on(cfg, torch.device("cuda"), seed=5)
    shp = dict(T=2, H=16, W=16, ctx_len=128)
    net = build_net(cfg, sd)
    net._sync_weights()
    net._set_shape(shp["T"], shp["H"], shp["W"], shp["ctx_len"], 24.0)
    t1, t2, t3 = 0.734375, -1.25, 3.0
    worst = 0.0
    for t in (t1, t2, t3):
        e = modulation_errors(read_modulation(net, t), modulation64(sd, cfg, t), D)
        worst = max(worst, e)
        assert e <= 1e-5, (t, e)
    # a different timestep must be visible in the vectors (the check above is not comparing constants)
    assert modulation_errors(read_modulation(net, t1), modulation64(sd, cfg, t2), D) > 1e-2
    print(f"{case}: largest per-vector rel error {worst:.2e}")

    inp = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in cases.dit_inputs(cfg, **shp, seed=6).items()}
    inp["timestep"] = t1
    fresh = build_net(cfg, sd)
    a1 = read_modulation(net, t1)
    out_a = engine_forward(net, inp, 24.0)
    n_cached = net.last_launch_count()
    out_b = engine_forward(fresh, inp, 24.0)
    assert torch.equal(out_a, out_b)
    assert n_cached == fresh.last_launch_count() - (3 + 3 * 2 * cfg.num_blocks + 2)  # the vector launches were skipped
    a2 = read_modulation(net, t2)
    f2 = read_modulation(fresh, t2)
    assert torch.equal(a2[0], f2[0]) and torch.equal(a2[1], f2[1])
    assert torch.equal(read_modulation(net, t1)[0], a1[0])

    key = "blocks.block0.blocks.1.adaLN_modulation.2.weight"
    new = (sd[key] * -1.5 + 0.01).to(bf).float()
    sd2 = dict(sd, **{key: new})
    wt = new.to(bf).contiguous()
    from gen3c_b200 import _lib

    shape = (C.c_int64 * 2)(*wt.shape)
    _lib.check(_lib.load().g3c_dit_load(net._engine(), key.encode(), wt.data_ptr(), shape, 2, 0), "g3c_dit_load")
    got = read_modulation(net, t2)
    assert not torch.equal(got[0][1], a2[0][1])
    assert torch.equal(got[0][0], a2[0][0]) and torch.equal(got[1], a2[1])
    assert modulation_errors(got, modulation64(sd2, cfg, t2), D) <= 1e-5
