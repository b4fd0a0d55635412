"""The TE-compatible attention operator on the GPU (gen3c_b200.attention_op.DotProductAttention ->
g3c_attn_fwd_sbhd -> k_attn_fwd with token-major V): sbhd inputs, any key count, batch folded into the heads,
context parallelism.  Floating point: bf16 operands, fp32 accumulation -> relative L2 error < 5e-3 against fp32 SDPA
(the bar of test_dit_ops_gpu.py::test_attention)."""
import math
import os

import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu

TOL = 5e-3


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


def sbhd(s, b, h, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(s, b, h, 128, device="cuda", generator=g) * scale).to(torch.bfloat16)


def ref(q, k, v, scale=128 ** -0.5):
    """fp32 SDPA on [s, b, h, d] -> [s, b, h*d]"""
    qq, kk, vv = (t.permute(1, 2, 0, 3).float() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, scale=scale)
    s, b, h, d = q.shape
    return o.permute(2, 0, 1, 3).reshape(s, b, h * d)


def check64(o, q, k, v, scale=128 ** -0.5, label=""):
    """both float64 checks of tests/attn_ref64.py on sbhd tensors (batch x heads = the kernel's heads)"""
    s, b, h, _ = q.shape
    attn_ref64.check(o.reshape(s, -1), q.reshape(s, -1), k.reshape(k.shape[0], -1), v.reshape(v.shape[0], -1), b * h,
                     scale, label=label)


def op(h, **kw):
    from gen3c_b200.attention_op import DotProductAttention

    return DotProductAttention(h, 128, **kw)


def test_pv_operand_layout_one_hot():
    """Pins the MN-major descriptor of the P.V operand (LBO between the two 64-dim halves, SBO between 8-key row
    groups, 16 keys per k-step): query row r scores one key (r % 128) 884 nats above all others, so P is exactly
    one-hot and O row r must be exactly V row r % 128 — every key of a tile and every head dim in its place."""
    Lq, Lk, h = 256, 384, 2
    q = torch.zeros(Lq, 1, h, 128, device="cuda")
    q[torch.arange(Lq), 0, :, torch.arange(Lq) % 128] = 100.0
    k = torch.zeros(Lk, 1, h, 128, device="cuda")
    k[torch.arange(128) + 128, 0, :, torch.arange(128)] = 100.0  # key 128 + c matches the queries r % 128 == c
    v = sbhd(Lk, 1, h, seed=1)
    o = op(h)(q.to(torch.bfloat16), k.to(torch.bfloat16), v)
    want = v[128 + torch.arange(Lq) % 128].reshape(Lq, 1, h * 128)
    assert torch.equal(o, want)


@pytest.mark.parametrize("b,h", [(1, 1), (2, 2), (1, 4)])
@pytest.mark.parametrize("Lq", [1, 77, 300])
@pytest.mark.parametrize("Lk", [1, 7, 127, 128, 129, 512, 1000, 2049, 7040])
@pytest.mark.parametrize("log2_units", [False, True])
def test_parity_with_sdpa(Lk, Lq, b, h, log2_units):
    """softmax scale 1/sqrt(128), and ln 2 with Q pre-scaled by softmax_scale * log2(e) (the kernel then
    exponentiates S directly)."""
    q, k, v = sbhd(Lq, b, h, seed=Lk + Lq), sbhd(Lk, b, h, seed=2 * Lk + 1), sbhd(Lk, b, h, seed=3 * Lk + 2)
    want = ref(q, k, v)
    scale = 128 ** -0.5
    if log2_units:
        q = (q.float() * (128 ** -0.5 * math.log2(math.e))).to(torch.bfloat16)
        want = ref(q, k, v, scale=math.log(2.0))
        scale = math.log(2.0)
        o = op(h, softmax_scale=scale)(q, k, v)
    else:
        o = op(h)(q, k, v)
    assert o.shape == (Lq, b, h * 128)
    assert rel(o, want) < TOL, rel(o, want)
    check64(o, q, k, v, scale, label=f"Lk={Lk} Lq={Lq} b={b} h={h} log2={log2_units}")


@pytest.mark.parametrize("Lq,Lk,h", [(300, 128, 2), (1000, 1024, 2), (77, 7040, 1), (56320, 56320, 32)])
def test_bit_identical_to_vt_layout(Lq, Lk, h):
    """With Lk a multiple of 128 and b = 1 the token-major instantiation issues the same products in the same wgmma
    order as the V^T one (only the B operand's shared-memory layout differs), so the outputs are bitwise equal —
    including at the self-attention shape of the benchmark (56 320 x 56 320, 32 heads)."""
    from gen3c_b200 import ops

    q, k, v = sbhd(Lq, 1, h, seed=40), sbhd(Lk, 1, h, seed=41), sbhd(Lk, 1, h, seed=42)
    o = op(h)(q, k, v)
    o_vt = ops.attention(q.view(Lq, -1), k.view(Lk, -1), v.view(Lk, -1).T.contiguous(), h)
    assert torch.equal(o.view(Lq, -1), o_vt)


@pytest.mark.parametrize("Lk", [77, 200, 1000])
def test_tail_mask_negative_control(Lk):
    """Every valid key scores about -11 nats against every query, so the zero-filled K rows of the last tile (score 0)
    would carry almost all of the softmax if they were not masked.  The output must match the reference and miss
    "attention including the zero keys" by >= 10x the tolerance.  K and V are the first Lk rows of longer buffers whose
    extra rows are huge, so reading past Lk would show too."""
    b, h, Lq = 1, 2, 200
    pad = 128 - Lk % 128
    q = torch.ones(Lq, b, h, 128, device="cuda", dtype=torch.bfloat16)
    k_buf = torch.full((Lk + 300, b, h, 128), 1e4, device="cuda", dtype=torch.bfloat16)
    v_buf = torch.full((Lk + 300, b, h, 128), 1e4, device="cuda", dtype=torch.bfloat16)
    k_buf[:Lk] = (-1.0 - 0.5 * torch.rand(Lk, b, h, 128, device="cuda")).to(torch.bfloat16)
    v_buf[:Lk] = sbhd(Lk, b, h, seed=50)
    k, v = k_buf[:Lk], v_buf[:Lk]
    want = ref(q, k, v)
    zeros = torch.zeros(pad, b, h, 128, device="cuda", dtype=torch.bfloat16)
    with_zero_keys = ref(q, torch.cat([k, zeros]), torch.cat([v, zeros]))
    assert rel(with_zero_keys, want) >= 10 * TOL
    o = op(h)(q, k, v)
    assert rel(o, want) < TOL, rel(o, want)
    check64(o, q, k, v)


@pytest.mark.parametrize("Lk,first", [(100, 40), (1000, 950)])
def test_score_jump_in_partial_last_tile(Lk, first):
    """Keys far above all earlier ones inside the partial last tile (the only tile when Lk = 100): the running max,
    O and the row sums are rescaled in the masked step."""
    b, h, Lq = 1, 2, 384
    q, k, v = sbhd(Lq, b, h, seed=60, scale=0.5), sbhd(Lk, b, h, seed=61, scale=0.5), sbhd(Lk, b, h, seed=62)
    q[:, :, 0] = 1.0
    k[first:first + 20, :, 0] = 4.0
    want = ref(q, k, v)
    o = op(h)(q, k, v)
    assert torch.isfinite(o.float()).all()
    assert rel(o, want) < TOL, rel(o, want)
    check64(o, q, k, v)


def test_batch_isolation():
    """b = 2 is one launch of 2 x h heads: huge keys in batch 1 must not leak into batch 0, which is bitwise equal to a
    b = 1 run on batch 0 alone (passed as strided views: token stride 2 x h x 128)."""
    h, Lq, Lk = 2, 300, 1000
    q, k, v = sbhd(Lq, 2, h, seed=70), sbhd(Lk, 2, h, seed=71), sbhd(Lk, 2, h, seed=72)
    k[:, 1] = 1e3
    o2 = op(h)(q, k, v)
    o1 = op(h)(q[:, :1], k[:, :1], v[:, :1])
    assert torch.equal(o2[:, 0], o1[:, 0])
    assert rel(o2, ref(q, k, v)) < TOL
    check64(o2, q, k, v)


def test_errors():
    from gen3c_b200.attention_op import DotProductAttention

    for kw in (dict(attention_dropout=0.1), dict(attn_mask_type="causal"), dict(num_gqa_groups=1),
               dict(qkv_format="bshd"), dict(kv_channels=64)):
        args = dict(num_attention_heads=2, kv_channels=128)
        args.update(kw)
        with pytest.raises(NotImplementedError):
            DotProductAttention(**args)
    a = op(2)
    q = sbhd(64, 1, 2, seed=80)
    with pytest.raises(NotImplementedError):  # bias
        a(q, q, q, core_attention_bias_type="post_scale_bias", core_attention_bias=torch.zeros(1, 2, 64, 64))
    with pytest.raises(NotImplementedError):  # head_dim
        a(q[..., :64].contiguous(), q[..., :64].contiguous(), q[..., :64].contiguous())
    with pytest.raises(NotImplementedError):  # GQA at call time
        a(q, q[:, :, :1].contiguous(), q[:, :, :1].contiguous())
    with pytest.raises(ValueError):  # not CUDA
        a(q.cpu(), q.cpu(), q.cpu())
    with pytest.raises(ValueError):  # not bf16
        a(q.float(), q, q)
    wide = torch.zeros(64, 1, 2, 256, device="cuda", dtype=torch.bfloat16)[..., :128]
    with pytest.raises(ValueError):  # (b, h, d) block not contiguous
        a(wide, q, q)
    odd = torch.zeros(64, 2 * 128 + 4, device="cuda", dtype=torch.bfloat16)[:, :256].view(64, 1, 2, 128)
    with pytest.raises(ValueError):  # token stride 260 not a multiple of 8
        a(q, odd, q)
    shifted = torch.zeros(64 * 256 + 4, device="cuda", dtype=torch.bfloat16)[4:].view(64, 1, 2, 128)
    with pytest.raises(ValueError):  # base pointer 8 bytes off a 16-byte boundary
        a(q, q, shifted)
    with pytest.raises(ValueError):  # no keys
        a(q, q[:0], q[:0])
    with pytest.raises(ValueError):  # batch differs
        a(q, sbhd(64, 2, 2, seed=81), sbhd(64, 2, 2, seed=82))


def _cp_worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        S, b, h = 2 * 1000, 2, 2
        q, k, v = (t.cuda() for t in _cp_inputs(S, b, h))
        s = S // world
        a = op(h)
        a.set_context_parallel_group(dist.group.WORLD, list(range(world)), torch.cuda.Stream())
        out = a(q[rank * s:(rank + 1) * s], k[rank * s:(rank + 1) * s], v[rank * s:(rank + 1) * s])
        ret.put((rank, out.cpu()))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _cp_inputs(S, b, h):
    g = torch.Generator().manual_seed(90)
    return [torch.randn(S, b, h, 128, generator=g).to(torch.bfloat16) for _ in range(3)]


@pytest.mark.timeout(600)
def test_context_parallel_cp2_equals_single_gpu():
    """cp = 2 over NCCL: each rank passes its half of the sequence (1000 tokens: the gathered 2000 keys end in a partial
    tile); the concatenated outputs are bitwise equal to the single-GPU op on the full sequence."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    S, b, h = 2000, 2, 2
    q, k, v = (t.cuda() for t in _cp_inputs(S, b, h))
    want = op(h)(q, k, v).cpu()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + (os.getpid() + 500) % 2000
    procs = [ctx.Process(target=_cp_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(ret.get(timeout=500) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert torch.equal(torch.cat([got[0], got[1]]), want)
