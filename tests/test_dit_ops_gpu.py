"""GPU parity for the Path D operators (through the C ABI) against plain fp32 torch references.
Floating point: bf16 operands, fp32 accumulation -> relative L2 error <= 2e-3 vs an fp32 reference
evaluated on the same bf16-rounded inputs (output rounding to bf16 alone is ~1.1e-3 rms)."""
import math

import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def bf(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * s).to(torch.bfloat16)


@pytest.mark.parametrize("M,N,K,bn", [(128, 256, 64, 0), (256, 256, 4096, 0), (200, 384, 328 + 56, 128),
                                       (1000, 4096, 1024, 0), (128, 64, 256, 64), (384, 1000, 512, 0),
                                       (4096, 7040, 256, 0)])
def test_gemm_bf16(M, N, K, bn):
    from gen3c_b200 import ops

    a, b = bf(M, K, seed=1), bf(N, K, seed=2, s=0.05)
    ref = a.float() @ b.float().T
    out = ops.gemm(a, b, ops.EPI_BF16, block_n=bn)
    assert rel(out, ref) < 3e-3, rel(out, ref)
    out32 = ops.gemm(a, b, ops.EPI_F32, block_n=bn)
    assert rel(out32, ref) < 1e-5, rel(out32, ref)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 512, 4096), (1000, 4096, 1024), (4096, 7168, 256), (128, 256, 512),
                                   (7040, 4096, 4096)])
def test_gemm_cta_pair(M, N, K):
    """block_n = 512, the C ABI's request for the widest tile (256 columns per CTA), with every epilogue."""
    from gen3c_b200 import ops

    a, b = bf(M, K, seed=21), bf(N, K, seed=22, s=0.05)
    ref = a.float() @ b.float().T
    assert rel(ops.gemm(a, b, ops.EPI_BF16, block_n=512), ref) < 3e-3
    assert rel(ops.gemm(a, b, ops.EPI_F32, block_n=512), ref) < 1e-5
    x = torch.randn(M, N, device="cuda")
    gate = torch.randn(N, device="cuda")
    got = ops.gemm(a, b, ops.EPI_GATED_RESIDUAL_F32, out=x.clone(), gate=gate, block_n=512)
    assert rel(got, x + gate * ref) < 1e-5
    assert rel(ops.gemm(a, b, ops.EPI_GELU_BF16, block_n=512), torch.nn.functional.gelu(ref)) < 3e-3


def test_gemm_epilogues():
    from gen3c_b200 import ops

    M, N, K = 512, 512, 256
    a, b = bf(M, K, seed=3), bf(N, K, seed=4, s=0.1)
    ref = a.float() @ b.float().T
    out = ops.gemm(a, b, ops.EPI_GELU_BF16)
    assert rel(out, torch.nn.functional.gelu(ref)) < 3e-3
    x = torch.randn(M, N, device="cuda")
    gate = torch.randn(N, device="cuda")
    want = x + gate * ref
    got = ops.gemm(a, b, ops.EPI_GATED_RESIDUAL_F32, out=x.clone(), gate=gate)
    assert rel(got, want) < 1e-5


def test_gemm_transposed_output_by_operand_swap():
    """V^T = W_v . x^T comes from swapping the operands, no transpose pass."""
    from gen3c_b200 import ops

    x, w = bf(640, 256, seed=5), bf(256, 256, seed=6, s=0.05)
    vt = ops.gemm(w, x)
    assert rel(vt, (x.float() @ w.float().T).T) < 3e-3


@pytest.mark.parametrize("M,N,K,rope", [(1000, 256, 512, True), (512, 4096, 1024, False), (4096, 4096, 512, True),
                                          (300, 128, 256, True)])
def test_gemm_norm_rope(M, N, K, rope):
    """Projection + per-head RMSNorm + RoPE in the GEMM epilogue (128- and 256-column tiles) against the composition
    gemm (fp32 out) -> oracle RMSNorm / RoPE."""
    from gen3c_b200 import ops
    from oracle import dit_oracle

    a, b = bf(M, K, seed=41), bf(N, K, seed=42, s=0.05)
    gamma = (1 + 0.1 * torch.randn(128, device="cuda")).contiguous()
    ang = torch.rand(M, 64, device="cuda") * 6.0
    cs = torch.cat([torch.cos(ang), torch.sin(ang)], dim=1).contiguous()
    heads = N // 128
    acc = (a.float() @ b.float().T).cpu()
    ref = dit_oracle.rms_norm(acc.reshape(M, heads, 128), gamma.cpu())
    if rope:
        ref = dit_oracle.apply_rope(ref, torch.cat([ang, ang], 1).cpu())
    got = ops.gemm_norm_rope(a, b, gamma, cs if rope else None)
    assert rel(got.cpu(), ref.reshape(M, N)) < 3e-3, rel(got.cpu(), ref.reshape(M, N))


def sdpa_ref(q, k, v, heads):
    Lq, D = q.shape
    qh = q.float().reshape(Lq, heads, 128).permute(1, 0, 2)
    kh = k.float().reshape(-1, heads, 128).permute(1, 0, 2)
    vh = v.float().reshape(-1, heads, 128).permute(1, 0, 2)
    o = torch.nn.functional.scaled_dot_product_attention(qh[None], kh[None], vh[None])[0]
    return o.permute(1, 0, 2).reshape(Lq, D)


# one to 55 KV tiles (n_kv odd and even against the two-stage K/V ring),
# ragged Lq (rows of the last tile and whole padding CTAs masked at the store), an odd number of query tiles, and a
# chunked V^T layout (the context-parallel K/V order)
@pytest.mark.parametrize("Lq,Lk,heads,chunks", [(256, 128, 1, 1), (256, 512, 2, 1), (384, 1024, 2, 1),
                                                  (1280, 2560, 4, 1), (512, 1024, 2, 2), (7040, 7040, 2, 1),
                                                  (300, 1152, 1, 1), (200, 1280, 2, 1), (130, 1408, 1, 1),
                                                  (640, 2048, 2, 2), (896, 3072, 1, 3)])
def test_attention(Lq, Lk, heads, chunks):
    from gen3c_b200 import ops

    D = heads * 128
    q, k, v = bf(Lq, D, seed=7), bf(Lk, D, seed=8), bf(Lk, D, seed=9)
    ref = sdpa_ref(q, k, v, heads)
    cl = Lk // chunks
    vt = v.reshape(chunks, cl, D).permute(0, 2, 1).contiguous()  # [chunks, D, chunk_len]
    o = ops.attention(q, k, vt, heads, vt_chunk_len=cl)
    assert rel(o, ref) < 5e-3, rel(o, ref)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5)


@pytest.mark.parametrize("Lk", [1024, 2048])
def test_attention_peaked_softmax(Lk):
    """Large logits: exercises the rescale of O (scores spread over ~+-40) as the row max keeps growing over the
    KV tiles."""
    from gen3c_b200 import ops

    heads, Lq = 1, 256
    q, k, v = bf(Lq, 128, seed=10, s=3.0), bf(Lk, 128, seed=11, s=3.0), bf(Lk, 128, seed=12)
    # make later keys systematically larger so the max keeps growing across KV tiles
    k = (k.float() * torch.linspace(0.2, 2.0, Lk, device="cuda")[:, None]).to(torch.bfloat16)
    ref = sdpa_ref(q, k, v, heads)
    o = ops.attention(q, k, v.T.contiguous(), heads)
    assert rel(o, ref) < 8e-3, rel(o, ref)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5)


@pytest.mark.parametrize("jump", [4.0, 9.5])
def test_attention_score_jump(jump):
    """A block of keys far above everything before it, inside one KV tile: exp of the jump relative to the earlier
    tiles is ~2^65 (jump=4) or ~2^155 (jump=9.5, beyond fp32), so the running max, O and the row sums must be rescaled
    at that tile without overflow.  Both must match the fp32 reference."""
    from gen3c_b200 import ops

    heads, Lq, Lk = 2, 384, 2048
    q, k, v = bf(Lq, heads * 128, seed=20, s=0.5), bf(Lk, heads * 128, seed=21, s=0.5), bf(Lk, heads * 128, seed=22)
    q[:, :128] = 1.0  # head 0: constant queries; head 1 stays random
    k[300:340, :128] = jump  # scores 128 * jump / sqrt(128) = 11.3 * jump nats above the rest, in KV tile 2
    ref = sdpa_ref(q, k, v, heads)
    o = ops.attention(q, k, v.T.contiguous(), heads)
    assert torch.isfinite(o.float()).all()
    assert rel(o, ref) < 5e-3, rel(o, ref)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5)


@pytest.mark.parametrize("first_key", [260, 330])
def test_attention_score_jump_in_one_key_half(first_key):
    """Each row of a 128-key tile is spread over the four threads of a quad (columns interleaved in groups of 8).  A jump
    confined to the lower (keys 260..291 = columns 4..35 of tile 2) or the upper (330..361 = columns 74..105) half of
    the tile is seen by part of each quad's columns only: the row max must be reduced over the whole quad so that every
    column and all of O move to the same reference."""
    from gen3c_b200 import ops

    heads, Lq, Lk = 2, 384, 2048
    q, k, v = bf(Lq, heads * 128, seed=23, s=0.5), bf(Lk, heads * 128, seed=24, s=0.5), bf(Lk, heads * 128, seed=25)
    q[:, :128] = 1.0
    k[first_key:first_key + 32, :128] = 4.0
    ref = sdpa_ref(q, k, v, heads)
    o = ops.attention(q, k, v.T.contiguous(), heads)
    assert torch.isfinite(o.float()).all()
    assert rel(o, ref) < 5e-3, rel(o, ref)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5)


@pytest.mark.parametrize("gain", [1.0, 6.0])
def test_attention_log2_units(gain):
    """scale = ln 2: the caller folded softmax_scale * log2(e) into Q (what the DiT engine does through the query
    RMSNorm gain), so S arrives in log2 units and the kernel exponentiates without a scale multiply.  gain=1: moderate
    scores; gain=6: row maxima beyond 2^40."""
    from gen3c_b200 import ops

    heads, Lq, Lk = 2, 512, 2048
    q, k, v = bf(Lq, heads * 128, seed=30, s=gain), bf(Lk, heads * 128, seed=31, s=gain), bf(Lk, heads * 128, seed=32)
    qs = (q.float() * (128 ** -0.5 * math.log2(math.e))).to(torch.bfloat16)
    ref = sdpa_ref(qs.float() * math.log(2.0) * 128 ** 0.5, k, v, heads)  # softmax(qs k^T ln2) == softmax(q k^T / sqrt(d))
    o = ops.attention(qs, k, v.T.contiguous(), heads, scale=math.log(2.0))
    assert rel(o, ref) < 5e-3, rel(o, ref)
    # gain=6: scores of std ~52 (log2 units), row maxima near 180, so P spans far beyond fp32 before each rescale; the
    # score error term of attn_ref64 (eta ~ 4e-3 for sum |q k| ~ 380) is still first order, so both checks apply
    attn_ref64.check(o, qs, k, v, heads, math.log(2.0))


def test_ln_modulate():
    from gen3c_b200 import ops

    L, D = 300, 512
    x = torch.randn(L, D, device="cuda") * 2 + 0.3
    pos = bf(L, D, seed=13, s=0.5)
    shift, scale = torch.randn(D, device="cuda") * 0.1, torch.randn(D, device="cuda") * 0.1
    x2 = x.clone()
    y = ops.ln_modulate(x2, shift, scale, pos=pos)
    xr = x + pos.float()
    torch.testing.assert_close(x2, xr, atol=1e-6, rtol=0)
    ref = torch.nn.functional.layer_norm(xr, (D,), eps=1e-6) * (1 + scale) + shift
    assert rel(y, ref) < 3e-3
    y0 = ops.ln_modulate(x.clone(), shift, scale)
    assert rel(y0, torch.nn.functional.layer_norm(x, (D,), eps=1e-6) * (1 + scale) + shift) < 3e-3


def test_rmsnorm_rope():
    from gen3c_b200 import ops
    from oracle import dit_oracle

    L, heads = 384, 3
    q = bf(L, heads * 128, seed=14)
    gamma = 1 + 0.1 * torch.randn(128, device="cuda")
    ang = torch.rand(L, 64, device="cuda") * 6.0
    cs = torch.cat([torch.cos(ang), torch.sin(ang)], dim=1).contiguous()
    ref = dit_oracle.rms_norm(q.float().cpu().reshape(L, heads, 128), gamma.cpu())
    ref_rope = dit_oracle.apply_rope(ref, torch.cat([ang, ang], 1).cpu()).reshape(L, -1)
    got = ops.rmsnorm_rope_(q.clone(), heads, gamma, cs)
    assert rel(got.cpu(), ref_rope) < 3e-3
    got2 = ops.rmsnorm_rope_(q.clone(), heads, gamma, None)
    assert rel(got2.cpu(), ref.reshape(L, -1)) < 3e-3
