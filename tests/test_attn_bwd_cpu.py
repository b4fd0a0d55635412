"""The attention backward without a GPU: the float64 restatement of tests/attn_bwd_ref64.py against torch autograd, a
torch fp32 emulation of the kernels' roundings inside its bound (and wrong emulations outside it), the context-parallel
gradient of DotProductAttention over gloo at world size 2 with the kernel replaced by SDPA, and the argument checks of
g3c_attn_fwd_sbhd_lse and g3c_attn_bwd_sbhd."""
import math
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import attn_bwd_ref64 as ref64
from tests.attn_ref64 import LN2, scale_log2


def _inputs(Lq, Lk, heads, seed, logit=None, dominant=False):
    g = torch.Generator().manual_seed(seed)
    q, k, v, do = (torch.randn(L, heads * 128, generator=g) for L in (Lq, Lk, Lk, Lq))
    if logit is not None:  # scores up to +-logit (times scale): q and k near a common direction
        u = torch.randn(128, generator=g)
        u /= u.norm()
        c = math.sqrt(logit) * 128 ** 0.25
        for h in range(heads):
            hs = slice(h * 128, (h + 1) * 128)
            q[:, hs] = torch.sign(torch.randn(Lq, 1, generator=g)) * u * c + 0.1 * q[:, hs]
            k[:, hs] = torch.rand(Lk, 1, generator=g) * u * c + 0.1 * k[:, hs]
    if dominant:  # key 0 is the query's own direction, 8 x stronger
        k[0] = q[0] * 8
    return [t.to(torch.bfloat16) for t in (q, k, v, do)]


def _autograd64(q, k, v, do, heads, scale):
    """dq, dk, dv of float64 SDPA at the kernels' effective scale sl2 ln 2, with dQ and dK carried by `scale`."""
    eff = scale_log2(scale) * LN2
    qq, kk, vv = (t.double().view(t.shape[0], heads, 128).transpose(0, 1).requires_grad_() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, scale=eff)
    o.backward(do.double().view(do.shape[0], heads, 128).transpose(0, 1))
    g = [t.grad.transpose(0, 1).reshape(t.shape[1], heads * 128) for t in (qq, kk, vv)]
    return g[0] * (scale / eff), g[1] * (scale / eff), g[2]


@pytest.mark.parametrize("Lq,Lk,heads,scale", [(37, 300, 2, 128 ** -0.5), (129, 127, 1, math.log(2)), (1, 1, 1, 0.3)])
def test_restatement_equals_float64_autograd(Lq, Lk, heads, scale):
    q, k, v, do = _inputs(Lq, Lk, heads, 1)
    r = ref64.BwdReference(q, k, v, do, heads, scale)
    for got, want in zip((r.dq, r.dk, r.dv), _autograd64(q, k, v, do, heads, scale)):
        assert float((got - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max()))


def test_row_selection_matches_full_reference():
    q, k, v, do = _inputs(200, 150, 2, 2)
    full = ref64.BwdReference(q, k, v, do, 2, 128 ** -0.5, block=64)
    part = ref64.BwdReference(q, k, v, do, 2, 128 ** -0.5, q_rows=[0, 77, 199], k_rows=[3, 149], block=64)
    for a, b, rows in ((part.dq, full.dq, [0, 77, 199]), (part.bq, full.bq, [0, 77, 199]), (part.dk, full.dk, [3, 149]),
                       (part.bv, full.bv, [3, 149]), (part.sk, full.sk, [3, 149])):
        torch.testing.assert_close(a, b[rows], rtol=1e-12, atol=1e-300)


CASES = [
    dict(Lq=200, Lk=300, heads=2, scale=128 ** -0.5),
    dict(Lq=129, Lk=1, heads=1, scale=128 ** -0.5),
    dict(Lq=64, Lk=400, heads=1, scale=math.log(2)),
    dict(Lq=100, Lk=260, heads=1, scale=128 ** -0.5, logit=250.0),
    dict(Lq=90, Lk=200, heads=1, scale=128 ** -0.5, dominant=True),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_fp32_emulation_within_bound(case):
    """The kernels' roundings, emulated in torch fp32, stay inside the element bound and the statistical bar."""
    c = dict(case)
    Lq, Lk, heads, scale = c.pop("Lq"), c.pop("Lk"), c.pop("heads"), c.pop("scale")
    q, k, v, do = _inputs(Lq, Lk, heads, 3, **c)
    r = ref64.BwdReference(q, k, v, do, heads, scale)
    dq, dk, dv = ref64.emulate(q, k, v, do, heads, scale)
    out = r.check(dq, dk, dv, label=str(case), stat="logit" not in case)
    assert max(x[0] for x in out.values()) > 1e-4  # the bound is not vacuous


def test_wrong_emulations_miss_the_bound():
    """Controls on the emulation: a shifted lse, Delta = 0, and a dropped 128-key tile each miss by >= 10x."""
    Lq, Lk, heads, scale = 256, 1000, 1, 128 ** -0.5
    q, k, v, do = _inputs(Lq, Lk, heads, 4)
    r = ref64.BwdReference(q, k, v, do, heads, scale)
    sl2 = scale_log2(scale)
    x = (q.double() @ k.double().T) * sl2
    lse = (torch.logsumexp(x * LN2, 1) / LN2).float()[None]
    o = (torch.softmax(x * LN2, 1) @ v.double()).to(torch.bfloat16)
    worst = lambda d: max(max(e, s) for e, s, _ in d.values())  # noqa: E731
    assert worst(r.ratios(*ref64.emulate(q, k, v, do, heads, scale, o=o, lse=lse))) <= 1.0
    assert worst(r.ratios(*ref64.emulate(q, k, v, do, heads, scale, o=o, lse=lse + 1))) >= 10
    assert worst(r.ratios(*ref64.emulate(q, k, v, do, heads, scale, o=torch.zeros_like(o), lse=lse))) >= 10
    k2, v2 = k.clone(), v.clone()
    k2[128:256], v2[128:256] = k[0:128], v[0:128]
    dq, _, _ = ref64.emulate(q, k2, v2, do, heads, scale, o=o, lse=lse)
    assert worst(r.ratios(dq=dq)) >= 10


def _sdpa_sbhd(q, k, v, scale):
    qq, kk, vv = (t.permute(1, 2, 0, 3).double() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, scale=scale)
    s, b, h, d = q.shape
    return o.permute(2, 0, 1, 3).reshape(s, b, h * d)


def _cp_inputs():
    g = torch.Generator().manual_seed(12)
    return [torch.randn(40, 2, 3, 128, generator=g, dtype=torch.float64) for _ in range(4)]


def _cp_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from gen3c_b200 import attention_op, ops

        ops.attention_sbhd = _sdpa_sbhd  # this process only: differentiable through torch autograd
        q, k, v, do = _cp_inputs()
        s = q.shape[0] // world
        local = slice(rank * s, (rank + 1) * s)
        ql, kl, vl = (t[local].clone().requires_grad_() for t in (q, k, v))
        op = attention_op.DotProductAttention(3, 128)
        op.set_context_parallel_group(dist.group.WORLD, list(range(world)), None)
        out = op(ql, kl, vl)
        out.backward(do[local].reshape(out.shape))
        ret.put((rank, out.detach(), ql.grad, kl.grad, vl.grad))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_context_parallel_gradient_gloo_world2():
    """Each rank holds a slice of q, k, v; the K/V gather's backward reduce-scatters the gathered gradients (real
    reduce_scatter_tensor over gloo), so each rank's dK / dV equals its slice of the unsharded gradient, and its dQ
    the rows of its own queries."""
    q, k, v, do = _cp_inputs()
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = _sdpa_sbhd(qq, kk, vv, 128 ** -0.5)
    o.backward(do.reshape(o.shape))
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + (os.getpid() + 1500) % 2000
    procs = [ctx.Process(target=_cp_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = {r: rest for r, *rest in (ret.get(timeout=240) for _ in procs)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    s = q.shape[0] // 2
    for r in range(2):
        sl = slice(r * s, (r + 1) * s)
        out, gq, gk, gv = got[r]
        torch.testing.assert_close(out, o.detach()[sl], rtol=1e-12, atol=1e-12)
        for g, want in ((gq, qq.grad[sl]), (gk, kk.grad[sl]), (gv, vv.grad[sl])):
            torch.testing.assert_close(g, want, rtol=1e-12, atol=1e-12)


BWD_OK = (128, 128, 1, 1, 128, 128, 128, 128, 128, 128, 128, 128)


@pytest.mark.parametrize("i,val,what", [
    (0, 0, "Lq"), (1, 0, "Lk"), (2, 0, "batch"), (3, 70000, "batch"),
    (4, 132, "leading"), (7, 120, "leading"), (8, 64, "leading"), (11, 100, "leading"),
])
def test_bwd_c_abi_size_checks(i, val, what):
    """g3c_attn_bwd_sbhd rejects bad sizes with G3C_EINVAL and a message before it touches memory."""
    from gen3c_b200 import _lib

    lib = _lib.load()
    p = 1 << 20  # never dereferenced: the checks come first
    args = list(BWD_OK)
    args[i] = val
    assert lib.g3c_attn_bwd_sbhd(p, p, p, p, p, p, p, p, p, p, *args, 0.088, None) == -1
    assert what in lib.g3c_last_error().decode()


def test_bwd_c_abi_pointer_checks():
    from gen3c_b200 import _lib

    lib = _lib.load()
    p = 1 << 20
    ptrs = [p] * 10
    for j in range(10):
        bad = list(ptrs)
        bad[j] = None
        assert lib.g3c_attn_bwd_sbhd(*bad, *BWD_OK, 0.088, None) == -1
        assert "null" in lib.g3c_last_error().decode()
    for j in (0, 1, 2, 3, 4, 7, 8, 9):
        bad = list(ptrs)
        bad[j] = p + 8
        assert lib.g3c_attn_bwd_sbhd(*bad, *BWD_OK, 0.088, None) == -1
        assert "16-byte aligned" in lib.g3c_last_error().decode()
    for j in (5, 6):
        bad = list(ptrs)
        bad[j] = p + 2
        assert lib.g3c_attn_bwd_sbhd(*bad, *BWD_OK, 0.088, None) == -1
        assert "4-byte aligned" in lib.g3c_last_error().decode()


def test_lse_forward_c_abi_checks():
    from gen3c_b200 import _lib

    lib = _lib.load()
    p = 1 << 20
    assert lib.g3c_attn_fwd_sbhd_lse(p, p, p, p, None, 128, 128, 1, 1, 128, 128, 128, 128, 0.088, None) == -1
    assert "lse" in lib.g3c_last_error().decode()
    assert lib.g3c_attn_fwd_sbhd_lse(p, p, p, p, p + 2, 128, 128, 1, 1, 128, 128, 128, 128, 0.088, None) == -1
    assert "4-byte aligned" in lib.g3c_last_error().decode()
    assert lib.g3c_attn_fwd_sbhd_lse(p, p, p, p, p, 0, 128, 1, 1, 128, 128, 128, 128, 0.088, None) == -1
    assert "Lq" in lib.g3c_last_error().decode()


def test_autograd_function_is_used_only_when_grad_is_needed(monkeypatch):
    """Without a GPU: attention_sbhd takes the autograd path exactly when grad mode is on and an input requires grad
    (the kernels are replaced, so the dispatch and the backward's shapes are what is checked)."""
    from gen3c_b200 import ops

    calls = []

    def fake_lse(q, k, v, scale=None):
        calls.append("lse")
        o = _sdpa_sbhd(q, k, v, scale).to(torch.bfloat16)
        return o, torch.zeros(q.shape[1] * q.shape[2], q.shape[0])

    def fake_bwd(q, k, v, o, lse, dout, scale=None):
        calls.append("bwd")
        assert dout.dtype == torch.bfloat16 and dout.is_contiguous()
        return (torch.ones(q.shape, dtype=torch.bfloat16), torch.ones(k.shape, dtype=torch.bfloat16),
                torch.ones(v.shape, dtype=torch.bfloat16))

    monkeypatch.setattr(ops, "attention_sbhd_lse", fake_lse)
    monkeypatch.setattr(ops, "attention_sbhd_backward", fake_bwd)
    monkeypatch.setattr(ops, "_sbhd_operands", lambda q, k, v: (0, 0, 0))
    q, k, v = (torch.randn(5, 1, 2, 128).to(torch.bfloat16) for _ in range(3))
    k.requires_grad_()
    o = ops.attention_sbhd(q, k, v)
    assert calls == ["lse"] and o.requires_grad
    o.float().sum().backward()
    assert calls == ["lse", "bwd"] and k.grad.shape == k.shape and torch.all(k.grad == 1)
