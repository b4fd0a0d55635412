"""g3c_dit_forward restated from the per-operator entry points of gen3c_b200.ops, for one rank or for every rank of a
context-parallel group, and the engine forward with its launches per profiling category.

The kernels use no split-K and no atomics, so the same launches on the same operands give the same bits: a replay is
compared with torch.equal.  Inputs the engine derives itself are read back (the adaLN vectors through
g3c_dit_read_modulation, the RoPE and abs-pos tables through g3c_dit_read_tables) or rebuilt exactly: the query gain,
the padded patch weight, patchify and unpatchify.
"""
import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

from gen3c_b200 import _lib, ops

bf = torch.bfloat16
LN2 = 0.6931471805599453  # the attention scale: 1/sqrt(128) * log2(e) is folded into the query gain
# that factor as the engine computes it: a product of two fp32 constants, rounded to fp32
Q_SCALE = np.float32(0.08838834764831845) * np.float32(1.4426950408889634)
CATEGORIES = ("gemm", "attn_self", "attn_cross", "eltwise", "comm", "vector")


def launches(blocks, fp8, vectors=True):
    """The launches per category of one forward of a `blocks`-block net (the K / V^T exchange of the peer-memory
    mode is copies, not launches).  vectors=False: the adaLN vectors of the timestep are cached already."""
    return dict(gemm=10 * blocks + 2, attn_self=blocks, attn_cross=blocks, eltwise=3 * blocks + 3 + (3 * blocks if fp8 else 0),
                comm=0, vector=6 * blocks + 5 if vectors else 0)


def engine_forward(net, x, mask, pose, pad, timestep, ctx):
    """g3c_dit_forward with profiling on: (output [16, T, H, W] bf16, launches per category, ms the self-attention
    loaders spent polling peer flags)."""
    lib, h = _lib.load(), net._engine()
    out = torch.empty_like(x)
    _lib.check(lib.g3c_dit_profile(h, 1), "g3c_dit_profile")
    _lib.check(lib.g3c_dit_forward(h, _lib.ptr(x), _lib.ptr(mask), _lib.ptr(pose), _lib.ptr(pad), timestep,
                                   _lib.ptr(ctx), out.data_ptr(), _lib.stream_ptr()), "g3c_dit_forward")
    ms, n = (C.c_float * 6)(), (C.c_int * 6)()
    _lib.check(lib.g3c_dit_profile_read(h, ms, n, 6), "g3c_dit_profile_read")
    wait = C.c_float()
    _lib.check(lib.g3c_dit_profile_wait_ms(h, C.byref(wait)), "g3c_dit_profile_wait_ms")
    _lib.check(lib.g3c_dit_profile(h, 0), "g3c_dit_profile")
    assert net.last_launch_count() == sum(n)
    return out, dict(zip(CATEGORIES, n)), wait.value


def read_modulation(net, timestep):
    """The engine's adaLN vectors at `timestep`: mods [num_blocks*3, 3D], modf [2D] f32."""
    D = net.model_channels
    mods = torch.empty((net.num_blocks * 3, 3 * D), device="cuda")
    modf = torch.empty(2 * D, device="cuda")
    _lib.check(_lib.load().g3c_dit_read_modulation(net._engine(), timestep, _lib.ptr(mods), _lib.ptr(modf),
                                                   _lib.stream_ptr()), "g3c_dit_read_modulation")
    return mods, modf


def read_tables(net, t0, L):
    """The RoPE cos|sin [L, 128] f32 and abs-pos [L, D] bf16 tables of a rank whose first latent frame is t0."""
    rope = torch.empty((L, 128), device="cuda")
    pos = torch.empty((L, net.model_channels), device="cuda", dtype=bf)
    _lib.check(_lib.load().g3c_dit_read_tables(net._engine(), t0, _lib.ptr(rope), _lib.ptr(pos), _lib.stream_ptr()),
               "g3c_dit_read_tables")
    return rope, pos


def gated_attention(q, k, vt, heads, first):
    """The self-attention launch of the peer-memory mode: K [cp*L, D] and V^T [cp][D][L] in chunks of L keys, visited
    from chunk `first` (the rank's own); every flag raised."""
    o = torch.empty_like(q)
    flags = torch.ones(vt.shape[0], device="cuda", dtype=torch.int32)
    D = q.shape[1]
    _lib.check(_lib.load().g3c_attn_fwd_gated(_lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.ptr(o), q.shape[0], k.shape[0],
                                              heads, D, D, D, vt.shape[2], LN2, _lib.ptr(flags), 1, first, None,
                                              _lib.stream_ptr()), "g3c_attn_fwd_gated")
    return o


def replay(sd, cfg, ranks, ctx, mods, modf, fp8, drop_remote=False, self_kv=None):
    """g3c_dit_forward restated with gen3c_b200.ops for every rank of a context-parallel group at once.

    ranks: one (x_in, mask, pose, pad, rope, pos) per rank, its T slice and its position tables.  One rank is the
    single-GPU forward (ungated attention); with more, every self-attention layer gathers the K and V^T of all ranks in
    the [cp][L][D] / [cp][D][L] layout of the peer-memory region, and rank r attends from chunk r.  Returns (the
    output [16, T, H, W] of every rank, the gathered (K, V^T) of every self-attention layer).

    In fp8 mode the eight large Linears of a block (self-attention q / k / v / out, cross-attention q / out, MLP
    layer1 / layer2) take e4m3 codes of their weight and their activation rows: xn straight from the fused LN-modulate,
    att and hid from a separate quantisation pass.  K and V^T stay bf16.

    Broken variants for negative controls: drop_remote, each rank attends to its own chunk only; self_kv(layer, k, vt),
    the self-attention of a layer reads the (K, V^T) it returns instead of its own."""
    D, heads, Co = cfg.model_channels, cfg.num_heads, cfg.out_channels
    cp = len(ranks)
    _, T, H, W = ranks[0][0].shape
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

    def ln_mod(x, m, p=None):  # x += p in place, then LN(x) * (1 + scale) + shift
        return (ops.ln_modulate_fp8 if fp8 else ops.ln_modulate)(x, m[:D], m[D:2 * D], pos=p)

    # patch embedding: column c*4 + m*2 + n of token (t, h, w) is channel c at (2h + m, 2w + n); zero-padded columns
    w_patch = sd["x_embedder.proj.1.weight"]
    kpad = (w_patch.shape[1] + 63) // 64 * 64
    w_patch = F.pad(w_patch, (0, kpad - w_patch.shape[1])).contiguous()
    xs = []
    for x_in, mask, pose, pad, _, _ in ranks:
        if pose is None:
            pose = torch.zeros((cfg.in_channels - 17, T, H, W), device="cuda", dtype=bf)
        src = torch.cat([x_in, mask, pose, pad.expand(1, T, H, W)])
        tok = src.reshape(-1, T, Hp, 2, Wp, 2).permute(1, 2, 4, 0, 3, 5).reshape(L, -1)
        tok = F.pad(tok, (0, kpad - tok.shape[1])).contiguous()
        xs.append(ops.gemm(tok, w_patch, ops.EPI_F32))

    q_scale = torch.tensor(float(Q_SCALE), dtype=torch.float32, device="cuda")
    kv = []
    for i in range(cfg.num_blocks):
        p = f"blocks.block{i}.blocks."
        for j in (0, 1):
            a = f"{p}{j}.block.attn."
            m = mods[3 * i + j]
            gq = sd[a + "to_q.1.weight"].float() * q_scale
            gk = sd[a + "to_k.1.weight"].float()
            if j == 0:  # self-attention, the abs-pos table added to x first
                xns = [ln_mod(x, m, r[5]) for x, r in zip(xs, ranks)]
                ks = [norm_rope(xn, sd[a + "to_k.0.weight"], gk, r[4]) for xn, r in zip(xns, ranks)]
                vts = [linear_vt(xn, sd[a + "to_v.0.weight"]) for xn in xns]
                k, vt = torch.cat(ks), torch.stack(vts)
                kv.append((k, vt))
                if self_kv is not None:
                    k, vt = self_kv(i, k, vt)
            else:  # cross-attention to the text context, whose K / V^T stay bf16
                xns = [ln_mod(x, m) for x in xs]
                k = ops.gemm_norm_rope(ctx, sd[a + "to_k.0.weight"], gk, None)
                vt = ops.gemm(sd[a + "to_v.0.weight"], ctx)
            for r, (x, xn) in enumerate(zip(xs, xns)):
                q = norm_rope(xn, sd[a + "to_q.0.weight"], gq, ranks[r][4] if j == 0 else None)
                if j == 1 or cp == 1:
                    att = ops.attention(q, k, vt, heads, scale=LN2, vt_chunk_len=L if j == 0 else M)
                elif drop_remote:
                    att = ops.attention(q, ks[r], vts[r], heads, scale=LN2, vt_chunk_len=L)
                else:
                    att = gated_attention(q, k, vt, heads, first=r)
                linear(rows(att), sd[a + "to_out.0.weight"], out=x, gate=m[2 * D:], **gated)
        m = mods[3 * i + 2]
        for x in xs:
            hid = linear(ln_mod(x, m), sd[p + "2.block.layer1.weight"], epilogue=ops.EPI_GELU_BF16)
            linear(rows(hid), sd[p + "2.block.layer2.weight"], out=x, gate=m[2 * D:], **gated)

    outs = []
    for x in xs:
        xn = ops.ln_modulate(x, modf[:D], modf[D:])
        y = ops.gemm(xn, sd["final_layer.linear.weight"], ops.EPI_F32, block_n=64)
        # unpatchify: column (p1*2 + p2)*C + c of token (t, h, w) -> channel c at (2h + p1, 2w + p2)
        outs.append(y.reshape(T, Hp, Wp, 2, 2, Co).permute(5, 0, 1, 3, 2, 4).reshape(Co, T, H, W).to(bf))
    return outs, kv
