"""Test reference of the fp8 (e4m3) Linear mode (DESIGN.md §3.1): the row quantiser in torch, and the DiT forward of
oracle/dit_oracle.py with that quantisation applied to the eight Linears the mode covers (self-attention to_q, to_k,
to_v, to_out; cross-attention to_q, to_out; MLP layer1, layer2), their input rows taken in the compute dtype (fp32).
Everything else is dit_oracle's arithmetic, op for op."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import dit_oracle as O


def quantize_rows_e4m3(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """amax_r = max |x[r]|, codes = e4m3_rn_satfinite(x * (448 / amax_r)), scale_r = amax_r / 448; a zero row gets codes
    0 and scale 1.  Returns (codes as torch.float8_e4m3fn, scales float32).  Divisions are tensor / tensor so that they
    are IEEE divisions on every device (torch may turn a division by a Python scalar into a reciprocal multiply)."""
    xf = x.float()
    amax = xf.abs().amax(dim=-1)
    nz = amax > 0
    c448 = torch.full_like(amax, 448.0)
    inv = torch.where(nz, c448 / torch.where(nz, amax, c448), torch.zeros_like(amax))
    # the clamp is satfinite; RNE is torch's float8 cast
    codes = (xf * inv[..., None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    scale = torch.where(nz, amax / c448, torch.ones_like(amax))
    return codes, scale


def linear_fp8(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """a [M, K] @ w[N, K]^T with both operands row-quantised: (codes_a . codes_w^T) * scale_a[m] * scale_w[n], summed in
    fp32, the scales applied before anything else (the GEMM's order)."""
    ca, sa = quantize_rows_e4m3(a)
    cw, sw = quantize_rows_e4m3(w)
    return (ca.float() @ cw.float().T) * sa[:, None] * sw[None, :]


def forward(sd, cfg: O.DitCfg, x, cond_mask, cond_pose, padding_mask, timestep: float, ctx, fps: float = 24.0,
            t0: int = 0, compute_dtype: torch.dtype = torch.float32):
    """dit_oracle.forward (B = 1, no context parallelism) with the fp8 Linear mode's quantisation."""
    dt, dev = compute_dtype, x.device
    D, heads = cfg.model_channels, cfg.num_heads
    _, T, H, W = x.shape
    Hp, Wp = H // 2, W // 2
    L = T * Hp * Wp
    npose = cfg.in_channels - 17

    def w(k):
        return sd[k].to(device=dev, dtype=dt)

    def lin(v, key):
        return linear_fp8(v, w(key)).to(dt)

    parts = [x.to(dt), cond_mask.to(dt)]
    if npose > 0:
        parts.append(cond_pose.to(dt) if cond_pose is not None else torch.zeros(npose, T, H, W, dtype=dt, device=dev))
    if cfg.concat_padding_mask:
        pm = padding_mask.to(dt) if padding_mask is not None else torch.zeros(H, W, dtype=dt, device=dev)
        parts.append(pm[None, None].expand(1, T, H, W))
    tok = O.patchify(torch.cat(parts, 0))
    h = tok @ w("x_embedder.proj.1.weight").T
    sdv = sd if sd["extra_pos_embedder.pos_emb_t"].device == dev else {k: sd[k].to(dev) for k in (
        "extra_pos_embedder.pos_emb_t", "extra_pos_embedder.pos_emb_h", "extra_pos_embedder.pos_emb_w")}
    pos = O.abs_pos_emb(sdv, cfg, T, Hp, Wp, t0).to(dt)
    ang = O.rope_angles(cfg, T, Hp, Wp, fps, t0, device=dev)
    s, emb, lora = O.modulation_vectors(sd, cfg, timestep, dt)

    def mod(prefix, n):
        a = w(prefix + "adaLN_modulation.1.weight") @ F.silu(emb)
        m = w(prefix + "adaLN_modulation.2.weight") @ a + lora[: n * D]
        return m.chunk(n)

    def ln(v):
        return F.layer_norm(v, (D,), eps=1e-6)

    def nrm(v, key):
        return O.rms_norm(v, sd[key].to(dev)).to(dt)

    def rope(v):
        return O.apply_rope(v.float(), ang).to(dt)

    ctx = ctx.to(dt)
    for i in range(cfg.num_blocks):
        h = h + pos
        p = f"blocks.block{i}.blocks.0."
        shift, scale, gate = mod(p, 3)
        xn = ln(h) * (1 + scale) + shift
        q = lin(xn, p + "block.attn.to_q.0.weight")
        k = lin(xn, p + "block.attn.to_k.0.weight")
        v = lin(xn, p + "block.attn.to_v.0.weight")
        q = rope(nrm(q.reshape(L, heads, 128), p + "block.attn.to_q.1.weight")).reshape(L, D)
        k = rope(nrm(k.reshape(L, heads, 128), p + "block.attn.to_k.1.weight")).reshape(L, D)
        o = O.attention(q, k, v, heads)
        h = h + gate * lin(o, p + "block.attn.to_out.0.weight")
        del q, k, v, o
        p = f"blocks.block{i}.blocks.1."
        shift, scale, gate = mod(p, 3)
        xn = ln(h) * (1 + scale) + shift
        q = lin(xn, p + "block.attn.to_q.0.weight")
        kc = ctx @ w(p + "block.attn.to_k.0.weight").T
        vc = ctx @ w(p + "block.attn.to_v.0.weight").T
        q = nrm(q.reshape(L, heads, 128), p + "block.attn.to_q.1.weight").reshape(L, D)
        kc = nrm(kc.reshape(-1, heads, 128), p + "block.attn.to_k.1.weight").reshape(-1, D)
        o = O.attention(q, kc, vc, heads)
        h = h + gate * lin(o, p + "block.attn.to_out.0.weight")
        del q, o
        p = f"blocks.block{i}.blocks.2."
        shift, scale, gate = mod(p, 3)
        xn = ln(h) * (1 + scale) + shift
        hid = F.gelu(lin(xn, p + "block.layer1.weight"))
        h = h + gate * lin(hid, p + "block.layer2.weight")
        del hid, xn
    shift, scale = mod("final_layer.", 2)
    y = (ln(h) * (1 + scale) + shift) @ w("final_layer.linear.weight").T
    return O.unpatchify(y, T, Hp, Wp, cfg.out_channels)
