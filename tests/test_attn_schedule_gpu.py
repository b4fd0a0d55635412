"""GPU cases of the pipelined attention schedule (S lookahead, separate K and V rings, turn token between the two consumer
warpgroups) that tests/test_dit_ops_gpu.py does not cover: KV tile counts around the ring depth, CTAs whose second
consumer warpgroup has no or only some valid rows, V^T chunk boundaries that fall mid-ring, and the determinism of a
full-width launch (a ring stage reused too early would make repeated launches differ)."""
import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def bf(*shape, seed=0, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * s).to(torch.bfloat16)


def sdpa_ref(q, k, v, heads):
    Lq, D = q.shape
    qh = q.float().reshape(Lq, heads, 128).permute(1, 0, 2)
    kh = k.float().reshape(-1, heads, 128).permute(1, 0, 2)
    vh = v.float().reshape(-1, heads, 128).permute(1, 0, 2)
    o = torch.nn.functional.scaled_dot_product_attention(qh[None], kh[None], vh[None])[0]
    return o.permute(1, 0, 2).reshape(Lq, D)


def run(Lq, Lk, heads, chunks, seed):
    """(o, fp32 reference); o also passes both float64 checks of tests/attn_ref64.py"""
    from gen3c_b200 import ops

    D = heads * 128
    q, k, v = bf(Lq, D, seed=seed), bf(Lk, D, seed=seed + 1), bf(Lk, D, seed=seed + 2)
    cl = Lk // chunks
    vt = v.reshape(chunks, cl, D).permute(0, 2, 1).contiguous()  # [chunks, D, chunk_len]
    o = ops.attention(q, k, vt, heads, vt_chunk_len=cl)
    attn_ref64.check(o, q, k, v, heads, 128 ** -0.5, label=f"Lq={Lq} Lk={Lk} chunks={chunks}")
    return o, sdpa_ref(q, k, v, heads)


@pytest.mark.parametrize("n_kv", [2, 3, 5, 6])
def test_kv_tiles_around_ring_depth(n_kv):
    o, ref = run(384, 128 * n_kv, 2, 1, seed=40)
    assert rel(o, ref) < 5e-3, rel(o, ref)


@pytest.mark.parametrize("Lq", [64, 100])
def test_single_cta_with_idle_second_warpgroup(Lq):
    """Lq = 64: the second consumer warpgroup has no valid row; Lq = 100: only 36 of its 64.  It still takes its turns."""
    for n_kv in (1, 4, 7):
        o, ref = run(Lq, 128 * n_kv, 1, 1, seed=50 + n_kv)
        assert o.shape[0] == Lq
        assert rel(o, ref) < 5e-3, (n_kv, rel(o, ref))


def test_chunk_boundaries_mid_ring():
    """3 V^T chunks of 384 keys (3 tiles each): chunk boundaries fall at ring positions that differ per chunk."""
    o, ref = run(512, 3 * 384, 2, 3, seed=60)
    assert rel(o, ref) < 5e-3, rel(o, ref)


def test_full_width_repeat_is_bit_identical():
    """Full self-attention width (56 320 keys, 440 KV tiles), 2 heads: the schedule is deterministic, so a second launch
    must reproduce the first exactly; the first is also checked against the fp32 reference and the float64 checks of
    tests/attn_ref64.py on a subset of query rows."""
    from gen3c_b200 import ops

    L, heads = 56320, 2
    D = heads * 128
    q, k, v = bf(L, D, seed=70), bf(L, D, seed=71), bf(L, D, seed=72)
    vt = v.T.contiguous()
    o1 = ops.attention(q, k, vt, heads)
    o2 = ops.attention(q, k, vt, heads)
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    rows = torch.arange(0, L, 97, device="cuda")
    ref = sdpa_ref(q[rows], k, v, heads)
    assert rel(o1[rows], ref) < 5e-3, rel(o1[rows], ref)
    attn_ref64.check(o1, q, k, v, heads, 128 ** -0.5, rows=rows, label="full width")
