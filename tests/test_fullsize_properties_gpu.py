"""BASELINE-size checks through size-independent properties (no oracle can run 56 320 tokens on the host):
attention normalisation / key-permutation invariance / agreement of sampled rows with an fp32 reference,
GEMM linearity and sampled-row agreement, LayerNorm-modulate statistics.  All through the C ABI."""
import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu

L_FULL, HEADS = 56320, 32


def bf(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * s).to(torch.bfloat16)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def test_attention_full_size_rows_sum_to_one_and_match_reference_rows():
    """Lq = Lk = 56 320, 4 heads (enough to fill the GPU; every head runs the same code path):
    (1) V = 1 -> O = 1 exactly up to bf16 rounding (checks the running-max / row-sum bookkeeping over 440 KV tiles);
    (2) 64 sampled query rows against an fp32 softmax(QK^T)V reference, and 256 against both float64 checks of
    tests/attn_ref64.py (every head)."""
    from gen3c_b200 import ops

    H = 4
    D = H * 128
    q, k = bf(L_FULL, D, seed=1), bf(L_FULL, D, seed=2)
    ones_t = torch.ones(D, L_FULL, device="cuda", dtype=torch.bfloat16)
    o = ops.attention(q, k, ones_t, H)
    assert float((o.float() - 1).abs().max()) < 8e-3
    v = bf(L_FULL, D, seed=3)
    o = ops.attention(q, k, v.T.contiguous(), H)
    rows = torch.randint(0, L_FULL, (64,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    for h in range(H):
        sl = slice(h * 128, (h + 1) * 128)
        s = (q[rows, sl].float() @ k[:, sl].float().T) * 128 ** -0.5
        ref = torch.softmax(s, dim=-1) @ v[:, sl].float()
        assert rel(o[rows, sl], ref) < 5e-3
    rows64 = torch.randint(0, L_FULL, (256,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    attn_ref64.check(o, q, k, v, H, 128 ** -0.5, rows=rows64, label="full size")


def test_attention_key_permutation_invariance():
    from gen3c_b200 import ops

    H, Lq, Lk = 2, 1024, 56320
    q, k, v = bf(Lq, H * 128, seed=5), bf(Lk, H * 128, seed=6), bf(Lk, H * 128, seed=7)
    perm = torch.randperm(Lk, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    a = ops.attention(q, k, v.T.contiguous(), H)
    b = ops.attention(q, k[perm].contiguous(), v[perm].T.contiguous(), H)
    assert rel(a, b) < 4e-3  # only the accumulation order and bf16 rounding of P differ
    rows = torch.arange(0, Lq, 4, device="cuda")
    ref = attn_ref64.Reference(q, k, v, H, 128 ** -0.5, rows)
    ref.check(a[rows], "keys in order")
    ref.check(b[rows], "keys permuted")


def test_gemm_full_size_linearity_and_sampled_rows():
    """[56 320, 4096] x [4096, 4096]^T: D(a1 + a2) = D(a1) + D(a2) in the fp32 epilogue, sampled rows vs fp32."""
    from gen3c_b200 import ops

    a1, a2 = bf(L_FULL, 4096, seed=9), bf(L_FULL, 4096, seed=10)
    w = bf(4096, 4096, seed=11, s=0.02)
    asum = (a1.float() + a2.float()).to(torch.bfloat16)
    exact = asum.float() == (a1.float() + a2.float())  # rows where the bf16 sum is exact are rare; use fp32 path
    d1, d2 = ops.gemm(a1, w, ops.EPI_F32), ops.gemm(a2, w, ops.EPI_F32)
    # gated-residual epilogue accumulates: x = d1 ; x += 1 * (a2 w^T)  ==  d1 + d2
    x = d1.clone()
    ops.gemm(a2, w, ops.EPI_GATED_RESIDUAL_F32, out=x, gate=torch.ones(4096, device="cuda"))
    assert rel(x, d1 + d2) < 1e-6
    rows = torch.arange(0, L_FULL, 877, device="cuda")
    ref = a1[rows].float() @ w.float().T
    assert rel(d1[rows], ref) < 1e-5
    assert rel(ops.gemm(a1, w, ops.EPI_BF16)[rows], ref) < 3e-3
    del exact


def test_ln_modulate_full_size_statistics():
    from gen3c_b200 import ops

    D = 4096
    x = torch.randn(L_FULL, D, device="cuda") * 3 + 1
    y = ops.ln_modulate(x, torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")).float()
    assert float(y.mean(dim=1).abs().max()) < 2e-3
    assert float((y.var(dim=1, unbiased=False) - 1).abs().max()) < 5e-3
