"""ORACLE (test infrastructure only) — engine-vs-oracle comparison of the DiT forward at BASELINE width, shared by
tests/test_fullsize_parity_gpu.py.  Needs a CUDA device: the fp32 oracle graph
(oracle/dit_oracle.py, TF32 off, explicit fp32 attention) runs on the GPU next to the engine, on the same weights.

What is measured, per depth (number of FA-CA-MLP blocks, final layer always applied):
  engine   : rel-L2 of this repo's CUDA engine (bf16 operands, fp32 accumulation / residual) against the fp32 oracle
  bf16     : rel-L2 of the oracle graph run with every tensor stored in bf16 (the reference's own inference precision:
             config/inference/cosmos-1-diffusion-gen3c.py sets bf16) against the same fp32 oracle
"""
from __future__ import annotations

import torch

from . import cases, dit_oracle


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def build_engine_net(cfg: dit_oracle.DitCfg, sd: dict, num_blocks: int, device):
    from gen3c_b200.dit import VideoExtendGeneralDIT

    net = VideoExtendGeneralDIT(max_img_h=cfg.max_h * 2, max_img_w=cfg.max_w * 2, max_frames=cfg.max_frames,
                                in_channels=cfg.in_channels, out_channels=cfg.out_channels,
                                model_channels=cfg.model_channels, num_blocks=num_blocks, num_heads=cfg.num_heads,
                                crossattn_emb_channels=cfg.context_dim, adaln_lora_dim=cfg.adaln_lora_dim,
                                rope_t_extrapolation_ratio=cfg.rope_t_ratio, device=device)
    want = net.state_dict().keys()
    net.load_state_dict({k: sd[k].to(torch.bfloat16) for k in want}, strict=True)
    return net


def engine_forward(net, inp: dict, T: int, device, cond: bool = True) -> torch.Tensor:
    bf = torch.bfloat16
    d = lambda t: t.to(device=device, dtype=bf)  # noqa: E731
    out = net(x=d(inp["x"])[None], timesteps=torch.tensor([inp["timestep"]], device=device, dtype=bf),
              crossattn_emb=d(inp["ctx_c"] if cond else inp["ctx_u"])[None], fps=torch.tensor([24.0], device=device),
              padding_mask=d(inp["padding"])[None, None], condition_video_input_mask=d(inp["cond_mask"])[None],
              condition_video_indicator=torch.zeros(1, 1, T, 1, 1, device=device, dtype=bf),
              condition_video_pose=d(inp["pose"])[None] if cond else None)
    return out[0].float()


@torch.no_grad()
def depth_sweep(T: int, H: int = 88, W: int = 160, ctx_len: int = 512, depths=(2, 8, 28), seed: int = 31,
                device="cuda", with_bf16: bool = True, log=print) -> dict:
    """Errors of the engine (and of a bf16 run of the oracle graph) against the fp32 oracle at the 7B width for the given
    depths, on T latent frames of the 720p grid.  Returns {depth: {"engine": e, "bf16": b}}."""
    device = torch.device(device)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = dit_oracle.DitCfg(num_blocks=max(depths))
    sd = dit_oracle.random_state_dict_on(cfg, device, seed=seed)
    inp = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in cases.dit_inputs(cfg, T, H, W, ctx_len, seed=seed + 1).items()}
    res = {}
    for nb in depths:
        want = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"],
                                  inp["ctx_c"], num_blocks=nb)
        net = build_engine_net(cfg, sd, nb, device)
        got = engine_forward(net, inp, T, device)
        r = {"engine": rel_l2(got, want)}
        del net, got
        if with_bf16:
            ob = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"],
                                    inp["ctx_c"], num_blocks=nb, compute_dtype=torch.bfloat16).float()
            r["bf16"] = rel_l2(ob, want)
            del ob
        del want
        torch.cuda.empty_cache()
        res[nb] = r
        log(f"  tokens {T * (H // 2) * (W // 2):6d}  blocks {nb:2d}: engine vs fp32 oracle rel-L2 {r['engine']:.3e}"
            + (f" ; bf16 run of the oracle graph vs fp32 {r['bf16']:.3e}" if with_bf16 else ""))
    return res
