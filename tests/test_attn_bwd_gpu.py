"""The attention backward on the GPU (g3c_attn_fwd_sbhd_lse + g3c_attn_bwd_sbhd, behind ops.attention_sbhd's autograd
function and attention_op.DotProductAttention): every gradient element against the float64 bound of
tests/attn_bwd_ref64.py, the rel-L2 error next to torch's bf16 SDPA backward, the LSE forward against the plain one,
bitwise reproducibility, the engine's shapes, negative controls built from wrong inputs, and the context-parallel
gradient on two GPUs."""
import json
import math
import os
import subprocess
import sys
import time

import pytest
import torch

from tests import attn_bwd_ref64 as ref64

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)
SCALES = [128 ** -0.5, LN2]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def sbhd(s, b, h, seed, scale=1.0):
    return (torch.randn(s, b, h, 128, device="cuda", generator=gen(seed)) * scale).to(torch.bfloat16)


def qscale(scale):
    """Query magnitude for a scale: under the log2 convention (scale = ln 2) q carries 1/sqrt(128) * log2(e)."""
    return 128 ** -0.5 * 1.4426950408889634 if scale == LN2 else 1.0


def flat(t):
    return t.reshape(t.shape[0], -1)


def backward(q, k, v, do, scale):
    from gen3c_b200 import ops

    o, lse = ops.attention_sbhd_lse(q, k, v, scale)
    return (o, lse) + ops.attention_sbhd_backward(q, k, v, o, lse, do, scale)


def check(q, k, v, do, scale, label, stat=True, **kw):
    """Runs the forward and backward, checks dq, dk, dv against the float64 bound; returns (reference, dq, dk, dv)."""
    _, _, dq, dk, dv = backward(q, k, v, do, scale)
    b, h = q.shape[1], q.shape[2]
    r = ref64.BwdReference(flat(q), flat(k), flat(v), flat(do), b * h, scale, **kw)
    qr, kr = kw.get("q_rows"), kw.get("k_rows")
    pick = lambda g, rows: flat(g) if rows is None else flat(g)[rows]  # noqa: E731
    r.check(pick(dq, qr), pick(dk, kr), pick(dv, kr), label=label, stat=stat)
    return r, dq, dk, dv


LENS = [1, 127, 128, 129, 1000, 4133]


@pytest.mark.parametrize("Lq", LENS)
@pytest.mark.parametrize("Lk", LENS)
def test_every_element_within_bound(Lq, Lk):
    """Every element of dQ, dK and dV within the float64 bound for ragged and whole tiles on both sides (query rows
    past Lq contribute nothing to dK / dV, keys past Lk nothing to dQ)."""
    scale = SCALES[(Lq + Lk) % 2]
    q = sbhd(Lq, 1, 2, 1, qscale(scale))
    k, v = sbhd(Lk, 1, 2, 2), sbhd(Lk, 1, 2, 3)
    do = sbhd(Lq, 1, 2, 4)
    check(q, k, v, do, scale, f"Lq {Lq} Lk {Lk} scale {scale:.4f}")


@pytest.mark.parametrize("scale", SCALES)
def test_batch_and_heads(scale):
    """b = 3 x h = 5: the batch folds into the kernels' heads; each (batch, head) only sees its own 128 columns."""
    q = sbhd(300, 3, 5, 11, qscale(scale))
    k, v, do = sbhd(520, 3, 5, 12), sbhd(520, 3, 5, 13), sbhd(300, 3, 5, 14)
    check(q, k, v, do, scale, f"b3 h5 scale {scale:.4f}")


def test_strided_views_of_fused_qkv():
    """q, k and v as strided views of one fused [s, 3, b, h, 128] tensor (token stride 3 b h 128), self-attention:
    the gradients equal those of contiguous copies bit for bit and are within the bound."""
    s, b, h = 700, 2, 2
    qkv = torch.randn(s, 3, b, h, 128, device="cuda", generator=gen(21)).to(torch.bfloat16)
    q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
    assert q.stride(0) == 3 * b * h * 128
    do = sbhd(s, b, h, 22)
    _, dq, dk, dv = check(q, k, v, do, 128 ** -0.5, "fused qkv views")
    _, _, dq2, dk2, dv2 = backward(q.contiguous(), k.contiguous(), v.contiguous(), do, 128 ** -0.5)
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dv, dv2)


def test_large_logits_dominant_key_and_single_key():
    """+-250-logit rows (q and k near one direction), one dominant key per query, and Lk = 1 (dQ = dK = 0 exactly
    up to rounding)."""
    Lq, Lk = 300, 500
    g = torch.Generator(device="cuda").manual_seed(31)
    u = torch.randn(128, device="cuda", generator=g)
    u /= u.norm()
    c = math.sqrt(250.0) * 128 ** 0.25
    sign = torch.sign(torch.randn(Lq, 1, 1, 1, device="cuda", generator=g))
    q = (sign * u * c + 0.1 * torch.randn(Lq, 1, 1, 128, device="cuda", generator=g)).to(torch.bfloat16)
    k = (torch.rand(Lk, 1, 1, 1, device="cuda", generator=g) * u * c
         + 0.1 * torch.randn(Lk, 1, 1, 128, device="cuda", generator=g)).to(torch.bfloat16)
    v, do = sbhd(Lk, 1, 1, 32), sbhd(Lq, 1, 1, 33)
    check(q, k, v, do, 128 ** -0.5, "+-250 logits", stat=False)
    # one dominant key: key j is 8 x query j's own direction for the first 200 queries
    q = sbhd(Lq, 1, 1, 34)
    k = sbhd(Lk, 1, 1, 35)
    k[:200] = q[:200] * 8
    check(q, k, v, do, 128 ** -0.5, "dominant key")
    k1, v1 = sbhd(1, 1, 2, 36), sbhd(1, 1, 2, 37)
    r, dq, dk, _ = check(sbhd(Lq, 1, 2, 38), k1, v1, sbhd(Lq, 1, 2, 39), 128 ** -0.5, "Lk = 1")
    assert float(dq.float().abs().max()) < 1e-2 * float(r.dq.abs().max() + 1)


def _rel(g, ref):
    return float((g.double() - ref).norm() / ref.norm())


@pytest.mark.parametrize("scale", SCALES)
def test_rel_l2_against_torch_bf16_backward(scale):
    """Each gradient's rel-L2 error against float64 is at most 2x that of torch's bf16 SDPA backward on the same
    tensors."""
    Lq, Lk, b, h = 1000, 1500, 2, 2
    q = sbhd(Lq, b, h, 41, qscale(scale))
    k, v, do = sbhd(Lk, b, h, 42), sbhd(Lk, b, h, 43), sbhd(Lq, b, h, 44)
    _, _, dq, dk, dv = backward(q, k, v, do, scale)
    r = ref64.BwdReference(flat(q), flat(k), flat(v), flat(do), b * h, scale)
    eff = ref64.scale_log2(scale) * LN2
    qq, kk, vv = (t.permute(1, 2, 0, 3).detach().requires_grad_() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, scale=eff)
    o.backward(do.permute(1, 2, 0, 3))
    tq, tk, tv = (flat(t.grad.permute(2, 0, 1, 3)) for t in (qq, kk, vv))
    f = scale / eff
    for name, mine, theirs, want in (("dq", dq, tq.double() * f, r.dq), ("dk", dk, tk.double() * f, r.dk),
                                     ("dv", dv, tv, r.dv)):
        a, t = _rel(flat(mine), want), _rel(theirs, want)
        print(f"rel-L2 {name} scale {scale:.4f}: native {a:.3e}, torch bf16 SDPA {t:.3e}, ratio {a / t:.2f}")
        assert a <= 2 * t, (name, a, t)


@pytest.mark.parametrize("Lq,Lk", [(1, 1), (129, 4133), (1000, 127)])
@pytest.mark.parametrize("scale", SCALES)
def test_lse_forward(Lq, Lk, scale):
    """The LSE forward's O equals g3c_attn_fwd_sbhd's bit for bit; its lse is within the bound of float64."""
    from gen3c_b200 import ops

    q = sbhd(Lq, 2, 2, 51, qscale(scale))
    k, v = sbhd(Lk, 2, 2, 52), sbhd(Lk, 2, 2, 53)
    o, lse = ops.attention_sbhd_lse(q, k, v, scale)
    assert torch.equal(o, ops.attention_sbhd(q, k, v, scale))
    want, bound = ref64.lse_reference(flat(q), flat(k), 4, scale)
    ratio = float(((lse.double() - want).abs() / bound).max())
    print(f"lse Lq {Lq} Lk {Lk} scale {scale:.4f}: error / bound {ratio:.3g}")
    assert ratio <= 1.0


def test_backward_is_bitwise_reproducible():
    """Two backward runs are bitwise equal, and so are two autograd runs under torch.use_deterministic_algorithms
    (every gradient element has one writer: nothing for it to refuse or reorder)."""
    from gen3c_b200 import ops

    q, k, v, do = sbhd(2000, 1, 4, 61), sbhd(3000, 1, 4, 62), sbhd(3000, 1, 4, 63), sbhd(2000, 1, 4, 64)
    first = backward(q, k, v, do, 128 ** -0.5)
    second = backward(q, k, v, do, 128 ** -0.5)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
            runs.append(torch.autograd.grad(ops.attention_sbhd(qg, kg, vg), (qg, kg, vg), do.view(2000, 1, 512)))
    finally:
        torch.use_deterministic_algorithms(was)
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    assert all(torch.equal(a, b) for a, b in zip(runs[0], first[2:]))


def test_dot_product_attention_autograd_graph():
    """torch.autograd.grad through Linear -> DotProductAttention -> Linear: the gradients reaching q, k and v are
    within the float64 bound of the (q, k, v, dO) the operator saw, and the gradients of the input and the weights
    match float64 autograd of the whole graph."""
    from gen3c_b200.attention_op import DotProductAttention

    s, b, h = 333, 2, 2
    g = gen(71)
    x = torch.randn(s, b, 256, device="cuda", generator=g).to(torch.bfloat16).requires_grad_()
    w_qkv = (torch.randn(3 * h * 128, 256, device="cuda", generator=g) / 16).to(torch.bfloat16).requires_grad_()
    w_o = (torch.randn(64, h * 128, device="cuda", generator=g) / 16).to(torch.bfloat16).requires_grad_()
    op = DotProductAttention(h, 128)

    def graph(x, w_qkv, w_o, attn):
        qkv = (x @ w_qkv.T).view(s, b, 3, h, 128).transpose(1, 2).contiguous()  # [s, 3, b, h, 128]
        q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
        o = attn(q, k, v)
        return (o @ w_o.T).square().sum(), q, k, v, o

    loss, q, k, v, o = graph(x, w_qkv, w_o, op)
    gx, gw, gwo, dq, dk, dv, do = torch.autograd.grad(loss, [x, w_qkv, w_o, q, k, v, o])
    r = ref64.BwdReference(flat(q.detach()), flat(k.detach()), flat(v.detach()), flat(do), b * h, 128 ** -0.5)
    r.check(flat(dq), flat(dk), flat(dv), label="through DotProductAttention")

    def sdpa64(q, k, v):
        qq, kk, vv = (t.permute(1, 2, 0, 3) for t in (q, k, v))
        return torch.nn.functional.scaled_dot_product_attention(qq, kk, vv).permute(2, 0, 1, 3).reshape(s, b, -1)

    x64, w64, wo64 = (t.detach().double().requires_grad_() for t in (x, w_qkv, w_o))
    loss64 = graph(x64, w64, wo64, sdpa64)[0]
    for name, got, want in zip(("x", "w_qkv", "w_o"), (gx, gw, gwo), torch.autograd.grad(loss64, [x64, w64, wo64])):
        e = _rel(got, want)
        print(f"graph gradient {name}: rel-L2 {e:.3e}")
        assert e < 2e-2, (name, e)


_PROFILE_CHILD = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from gen3c_b200.attention_op import DotProductAttention

mode = sys.argv[1]
op = DotProductAttention(2, 128)
g = torch.Generator(device="cuda").manual_seed(81)
q, k, v = (torch.randn(n, 1, 2, 128, device="cuda", generator=g).to(torch.bfloat16) for n in (200, 300, 300))
if mode != "plain":
    q.requires_grad_()
op(q, k, v)  # module load outside the profiled window
with torch.no_grad() if mode == "no_grad" else torch.enable_grad():
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        op(q, k, v)
        torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type.name == "CUDA" and "attn" in e.name]))
"""


def _attn_kernels(mode):
    """Names of the attention kernels one DotProductAttention call launches, profiled in a child process (a profiler
    session leaves CUPTI state behind in the process that ran it)."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, mode], cwd=root, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=root), timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_no_grad_runs_todays_kernel():
    """Without requires_grad (or under no_grad) the operator launches exactly the forward kernel it launched before
    (no lse); with it, the LSE build of the same kernel."""
    for mode, want in (("plain", "k_attn_fwd<false, true, false>"), ("no_grad", "k_attn_fwd<false, true, false>"),
                       ("requires_grad", "k_attn_fwd<false, true, true>")):
        names = _attn_kernels(mode)
        print(mode, names)
        assert len(names) == 1 and want in names[0], (mode, names)


# ------------------------------------------------------------------------------------------------------------------
# the engine's shapes
# ------------------------------------------------------------------------------------------------------------------
L_FULL, CTX_LEN, HEADS = 56320, 512, 32
KQ_SCALE = 128 ** -0.5 * 1.4426950408889634  # folded into q by the engine (scale = ln 2)


def engine_inputs(Lq, Lk, seed):
    """[L, 1, 32, 128] q (rows' magnitudes spread 0.5x - 4x around the folded scale, shuffled), k, v, dO."""
    g = gen(seed)
    mags = KQ_SCALE * math.sqrt(2.0) * torch.logspace(-math.log10(2.828), math.log10(2.828), Lq, device="cuda")
    mags = mags[torch.randperm(Lq, device="cuda", generator=g)]
    q = (torch.randn(Lq, 1, HEADS, 128, device="cuda", generator=g) * mags[:, None, None, None]).to(torch.bfloat16)
    k, v = (torch.randn(Lk, 1, HEADS, 128, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2))
    do = torch.randn(Lq, 1, HEADS, 128, device="cuda", generator=g).to(torch.bfloat16)
    return q, k, v, do


def sampled_rows(L):
    """Two rows of every 128-row tile, one per consumer warpgroup (rows 0-63 / 64-127 of the tile), rotating through
    the warps and fragment rows with the tile index; the last (ragged) tile's rows below L."""
    n = (L + 127) // 128
    t = torch.arange(n, device="cuda")
    r_a = 16 * (t % 4) + (t // 4) % 16
    r_b = 64 + 16 * ((t + 1) % 4) + (t // 4 + 5) % 16
    rows = torch.stack([128 * t + r_a, 128 * t + r_b], 1).reshape(-1)
    return rows[rows < L]


@pytest.mark.parametrize("Lk", [L_FULL, CTX_LEN])
def test_engine_shape_every_tile(Lk):
    """56 320 queries x 56 320 (self) or 512 (cross) keys, 32 heads, scale ln 2: two dQ rows of every query tile and
    two dK / dV rows of every key tile, every head, within the float64 bound."""
    t0 = time.time()
    q, k, v, do = engine_inputs(L_FULL, Lk, 91 + Lk)
    torch.cuda.synchronize()
    t1 = time.time()
    _, _, dq, dk, dv = backward(q, k, v, do, LN2)
    torch.cuda.synchronize()
    t2 = time.time()
    qr, kr = sampled_rows(L_FULL), sampled_rows(Lk)
    r = ref64.BwdReference(flat(q), flat(k), flat(v), flat(do), HEADS, LN2, q_rows=qr, k_rows=kr, block=2048)
    r.check(flat(dq)[qr], flat(dk)[kr], flat(dv)[kr], label=f"engine shape {L_FULL} x {Lk}")
    print(f"engine shape {L_FULL} x {Lk}: forward + backward {t2 - t1:.2f} s (first call), reference and checks "
          f"{time.time() - t2:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------------------
# negative controls: wrong inputs, correct kernels
# ------------------------------------------------------------------------------------------------------------------
def test_negative_controls_miss_by_10x():
    """lse + 1, Delta = 0 (O = 0), dO with one 64-query tile zeroed, and K with one 128-key tile taken from its
    neighbour: each backward misses the bound of the correct inputs by >= 10x."""
    from gen3c_b200 import ops

    Lq, Lk, b, h, scale = 1000, 1200, 1, 2, 128 ** -0.5
    q, k, v, do = sbhd(Lq, b, h, 101), sbhd(Lk, b, h, 102), sbhd(Lk, b, h, 103), sbhd(Lq, b, h, 104)
    o, lse = ops.attention_sbhd_lse(q, k, v, scale)
    r = ref64.BwdReference(flat(q), flat(k), flat(v), flat(do), b * h, scale)

    def worst(q_, k_, o_, lse_, do_):
        g = ops.attention_sbhd_backward(q_, k_, v, o_, lse_, do_, scale)
        return max(max(e, s) for e, s, _ in r.ratios(*(flat(t) for t in g)).values())

    good = worst(q, k, o, lse, do)
    assert good <= 1.0
    do_bad = do.clone()
    do_bad[320:384] = 0
    k_bad = k.clone()
    k_bad[512:640] = k[640:768]
    for name, args in (("lse + 1", (q, k, o, lse + 1, do)), ("Delta = 0", (q, k, torch.zeros_like(o), lse, do)),
                       ("dO tile zeroed", (q, k, o, lse, do_bad)), ("K tile from neighbour", (q, k_bad, o, lse, do))):
        m = worst(*args)
        print(f"negative control {name}: {m:.3g} x the bound (correct inputs: {good:.3g})")
        assert m >= 10, (name, m)


# ------------------------------------------------------------------------------------------------------------------
# context parallelism on two GPUs
# ------------------------------------------------------------------------------------------------------------------
def _cp_worker(rank, world, port, ret):
    import torch.distributed as dist

    from gen3c_b200.attention_op import DotProductAttention

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        q, k, v, do = (t.cuda() for t in _cp_inputs())
        s = q.shape[0] // world
        sl = slice(rank * s, (rank + 1) * s)
        ql, kl, vl = (t[sl].clone().requires_grad_() for t in (q, k, v))
        a = DotProductAttention(2, 128)
        a.set_context_parallel_group(dist.group.WORLD, list(range(world)), torch.cuda.Stream())
        out = a(ql, kl, vl)
        out.backward(do[sl].reshape(out.shape))
        ret.put((rank, ql.grad.cpu(), kl.grad.cpu(), vl.grad.cpu()))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _cp_inputs():
    g = torch.Generator().manual_seed(111)
    return [torch.randn(2000, 2, 2, 128, generator=g).to(torch.bfloat16) for _ in range(4)]


@pytest.mark.timeout(600)
def test_context_parallel_gradient_two_gpus():
    """cp = 2 over NCCL: each rank's dQ, dK and dV are within the float64 bound of its slice of the unsharded
    gradient (dK / dV: the sum of both ranks' contributions, reduce-scattered)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    q, k, v, do = (t.cuda() for t in _cp_inputs())
    r = ref64.BwdReference(flat(q), flat(k), flat(v), flat(do), 4, 128 ** -0.5)
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + (os.getpid() + 900) % 2000
    procs = [ctx.Process(target=_cp_worker, args=(rk, 2, port, ret)) for rk in range(2)]
    for p in procs:
        p.start()
    got = {rk: rest for rk, *rest in (ret.get(timeout=500) for _ in procs)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    dq, dk, dv = (torch.cat([got[0][i], got[1][i]]).cuda() for i in range(3))
    # the dK / dV of each rank are a sum of two bf16 partial gradients: one more bf16 rounding than the bound's
    out = r.ratios(flat(dq), flat(dk), flat(dv))
    print("cp = 2 gradients:", out)
    assert out["dq"][0] <= 1.0 and out["dk"][0] <= 2.0 and out["dv"][0] <= 2.0
