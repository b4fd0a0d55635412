"""The TE-compatible attention operator (gen3c_b200.attention_op.DotProductAttention) without a GPU: its interface
against the reference's call site, the configurations it refuses, the size checks of g3c_attn_fwd_sbhd, and the
context-parallel host logic over gloo with the kernel replaced by SDPA."""
import inspect
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.ref_stubs import _TEDotProductAttention


def _keywords(fn, skip):
    return {n for n, p in inspect.signature(fn).parameters.items()
            if n not in skip and p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)}


def test_accepts_the_reference_call_site():
    """Every keyword the reference passes to TE DotProductAttention (the stub restates that call) is accepted by the
    constructor, forward and set_context_parallel_group, and the reference's call itself goes through."""
    from gen3c_b200.attention_op import DotProductAttention

    stub_init = _keywords(_TEDotProductAttention.__init__, {"self", "heads", "dim_head"})
    assert stub_init <= _keywords(DotProductAttention.__init__, {"self"})
    stub_fwd = _keywords(_TEDotProductAttention.forward, {"self", "q", "k", "v"})
    assert stub_fwd <= _keywords(DotProductAttention.forward, {"self"})
    kw = dict(num_gqa_groups=32, attention_dropout=0, qkv_format="sbhd", attn_mask_type="no_mask", tp_size=1,
              tp_group=None, sequence_parallel=False)
    op = DotProductAttention(32, 128, **kw)
    _TEDotProductAttention(32, 128, **kw)
    assert op.softmax_scale == pytest.approx(128 ** -0.5)
    op.set_context_parallel_group(None, [0], None)
    assert op.cp_group is None
    assert DotProductAttention(32, 128, softmax_scale=0.5).softmax_scale == 0.5


@pytest.mark.parametrize("kw", [dict(attention_dropout=0.1), dict(attn_mask_type="causal"), dict(num_gqa_groups=8),
                                dict(qkv_format="bshd"), dict(kv_channels=64)])
def test_unsupported_configuration_raises(kw):
    from gen3c_b200.attention_op import DotProductAttention

    args = dict(num_attention_heads=32, kv_channels=128)
    args.update(kw)
    with pytest.raises(NotImplementedError):
        DotProductAttention(**args)


def test_bias_and_cpu_tensors_are_refused():
    from gen3c_b200.attention_op import DotProductAttention

    op = DotProductAttention(2, 128)
    q = torch.zeros(4, 1, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        op(q, q, q, core_attention_bias_type="post_scale_bias", core_attention_bias=torch.zeros(1, 2, 4, 4))
    with pytest.raises(ValueError):
        op(q, q, q)
    with pytest.raises(NotImplementedError):
        op(torch.zeros(4, 1, 2, 64), torch.zeros(4, 1, 2, 64), torch.zeros(4, 1, 2, 64))


@pytest.mark.parametrize("args,what", [
    ((0, 128, 1, 1, 128, 128, 128, 128), "Lq"),
    ((128, 0, 1, 1, 128, 128, 128, 128), "Lk"),
    ((128, 128, 0, 1, 128, 128, 128, 128), "batch"),
    ((128, 128, 300, 300, 128, 128, 128, 128), "batch"),
    ((128, 128, 2, 1, 128, 256, 256, 256), "leading"),
    ((128, 128, 1, 1, 132, 128, 128, 128), "leading"),
    ((128, 128, 1, 1, 128, 128, 128, 120), "leading"),
])
def test_c_abi_size_checks(args, what):
    """g3c_attn_fwd_sbhd rejects bad sizes with G3C_EINVAL and a message before it touches memory."""
    from gen3c_b200 import _lib

    lib = _lib.load()
    p = 1 << 20  # never dereferenced: the checks come first
    rc = lib.g3c_attn_fwd_sbhd(p, p, p, p, *args, 0.088, None)
    assert rc == -1
    assert what in lib.g3c_last_error().decode()
    assert lib.g3c_attn_fwd_sbhd(p, p, p, p + 8, 128, 128, 1, 1, 128, 128, 128, 128, 0.088, None) == -1
    assert "aligned" in lib.g3c_last_error().decode()


def _sdpa_sbhd(q, k, v, scale):
    qq, kk, vv = (t.permute(1, 2, 0, 3).float() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, scale=scale)
    s, b, h, d = q.shape
    return o.permute(2, 0, 1, 3).reshape(s, b, h * d)


def _cp_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from gen3c_b200 import attention_op, ops

        seen = {}

        def fake_kernel(q, k, v, scale):
            seen["k"], seen["v"] = k, v
            return _sdpa_sbhd(q, k, v, scale)

        ops.attention_sbhd = fake_kernel  # this process only
        q, k, v = _inputs()
        s = q.shape[0] // world
        local = slice(rank * s, (rank + 1) * s)
        op = attention_op.DotProductAttention(3, 128)
        op.set_context_parallel_group(dist.group.WORLD, list(range(world)), None)
        out = op(q[local], k[local], v[local])
        ret.put((rank, out, torch.equal(seen["k"], k) and torch.equal(seen["v"], v)))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _inputs():
    g = torch.Generator().manual_seed(11)
    return [torch.randn(40, 2, 3, 128, generator=g).to(torch.bfloat16) for _ in range(3)]


@pytest.mark.timeout(300)
def test_context_parallel_gloo_world2():
    """Each rank passes its slice of the sequence; forward gathers K and V in rank order (so the kernel sees exactly
    the unsharded K and V) and returns the rows of its own queries.  Concatenated in rank order they equal the
    single-process result."""
    q, k, v = _inputs()
    want = _sdpa_sbhd(q, k, v, 128 ** -0.5)
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + (os.getpid() + 1000) % 2000
    procs = [ctx.Process(target=_cp_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict((r, (o, ok)) for r, o, ok in (ret.get(timeout=240) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert got[0][1] and got[1][1], "the gathered K / V differ from the unsharded tensors"
    got = torch.cat([got[0][0], got[1][0]])
    assert got.shape == want.shape and float((got - want).norm() / want.norm()) < 1e-6
