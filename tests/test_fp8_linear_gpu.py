"""The fp8 (e4m3) Linear mode on the GPU: the row quantisers against the torch reference byte for byte, the fp8 GEMM
against an fp64 product of the dequantised operands (every epilogue and tile width, tails, the swapped V^T shape, the
block's real shapes), the engine and the denoise step with the mode on against the fp8 reference (tests/fp8_oracle.py),
and the mode switch itself."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cases, dit_oracle, parity
from tests import fp8_oracle

pytestmark = pytest.mark.gpu

bf = torch.bfloat16


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def ref_quant(x):
    """The contract's quantiser (oracle), on the GPU tensor's exact fp32 values; codes as bytes."""
    c, s = fp8_oracle.quantize_rows_e4m3(x.float().cpu())
    return c.view(torch.uint8), s


def edge_rows(C: int) -> torch.Tensor:
    """zero row, a single outlier, values at +-448, e4m3 subnormals after scaling, all negative, mixed magnitudes."""
    g = torch.Generator().manual_seed(5)
    rows = [torch.zeros(C), torch.full((C,), 0.01), torch.zeros(C), torch.randn(C, generator=g) * 1e-3,
            -torch.rand(C, generator=g), torch.randn(C, generator=g) * 300.0]
    rows[1][C // 3] = -1000.0
    grid = torch.arange(127, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
    vals = torch.cat([grid, -grid]).repeat(C // 254 + 1)[:C]
    rows[2] = vals.to(bf).float()
    rows[2][0] = 448.0
    rows[3][1] = 1.0  # the rest lands in the subnormal range of e4m3
    return torch.stack(rows)


@pytest.mark.parametrize("R,C,pad", [(6, 64, 0), (37, 4096, 64), (9, 16384, 8), (128, 1024, 0)])
def test_quantize_rows_matches_reference_bytewise(R, C, pad):
    g = torch.Generator().manual_seed(R)
    x = torch.randn(R, C, generator=g) * torch.logspace(-4, 4, R)[:, None]
    x[: min(R, 6)] = edge_rows(C)[: min(R, 6)]
    wide = torch.zeros(R, C + pad, dtype=bf, device="cuda")
    wide[:, :C] = x.to(bf).cuda()
    xin = wide[:, :C]  # ld = C + pad
    from gen3c_b200 import ops

    codes, scales = ops.quantize_rows_fp8(xin)
    want_c, want_s = ref_quant(xin)
    assert torch.equal(codes.cpu().view(torch.uint8), want_c)
    assert torch.equal(scales.cpu().view(torch.int32), want_s.view(torch.int32))
    assert float(scales[0]) == 1.0 and int(codes[0].view(torch.uint8).max()) == 0


def test_ln_modulate_fp8_quantiser_and_statistics():
    """(1) scale = -1 makes the modulated row exactly `shift`, so the fused quantiser is checked byte for byte on the edge
    rows; (2) on random inputs the codes are the quantisation of the fp32 LayerNorm result (up to rounding-boundary
    flips from the statistics' summation order) and x += pos is the same as in the bf16 kernel."""
    from gen3c_b200 import ops

    L, D = 64, 4096
    for row in edge_rows(D):
        x = torch.randn(L, D, device="cuda")
        shift = (row.to(bf).float() + 0.0).cuda().contiguous()  # + 0.0: -0 becomes +0, as fmaf(z, 0, -0) = +0 does
        codes, scales = ops.ln_modulate_fp8(x, shift, torch.full((D,), -1.0, device="cuda"))
        want_c, want_s = ref_quant(shift[None].expand(L, D))
        assert torch.equal(codes.cpu().view(torch.uint8), want_c)
        assert torch.equal(scales.cpu().view(torch.int32), want_s.view(torch.int32))
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(L, D, device="cuda", generator=g) * 3 + 1
    pos = torch.randn(L, D, device="cuda", generator=g).to(bf)
    shift, scale = 0.1 * torch.randn(D, device="cuda", generator=g), 0.1 * torch.randn(D, device="cuda", generator=g)
    x2 = x.clone()
    codes, scales = ops.ln_modulate_fp8(x, shift, scale, pos=pos)
    ops.ln_modulate(x2, shift, scale, pos=pos)
    assert torch.equal(x, x2)
    y = F.layer_norm(x.double(), (D,), eps=1e-6) * (1 + scale.double()) + shift.double()
    want_c, want_s = ref_quant(y.float())
    assert torch.allclose(scales.cpu(), want_s, rtol=1e-5)
    same = (codes.cpu().view(torch.uint8) == want_c).double().mean()
    assert same > 0.995, same
    assert rel(codes.float() * scales[:, None], y) < 0.04


def _operands(M, N, K, seed, spread=2.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.logspace(-spread, spread, M, device="cuda")[:, None]
    b = torch.randn(N, K, device="cuda", generator=g) * torch.logspace(spread, -spread, N, device="cuda")[:, None]
    from gen3c_b200 import ops

    a8, sa = ops.quantize_rows_fp8(a.to(bf))
    b8, sb = ops.quantize_rows_fp8(b.to(bf))
    return a8, sa, b8, sb


def _exact(a8, sa, b8, sb):
    return (a8.double() * sa.double()[:, None]) @ (b8.double() * sb.double()[:, None]).T


def _epi_ref(acc, epi, base, gate):
    from gen3c_b200 import ops

    if epi == ops.EPI_GELU_BF16:
        return F.gelu(acc)
    if epi == ops.EPI_GATED_RESIDUAL_F32:
        return base.double() + gate.double()[None] * acc
    return acc


# bf16 outputs: their rounding.  fp32 outputs: the e4m3 wgmma's own sum of each k32 step is not a full fp32 sum (H100:
# rel-L2 7e-5 at K = 48, 1.2e-4 at every K from 336 to 16 384, bit-identical bf16 results to torch._scaled_mm); the kernel
# adds each k-block's partial sum into fp32 registers so that this does not grow with K.  Summing all of K inside the
# instruction instead measures 1.3e-3 at K = 4096 and 3.5e-3 at K = 16 384: the block-shape cases below fail that.
TOL = {0: 3e-3, 1: 3e-3, 2: 3e-4, 3: 3e-4}


def _run_gemm(a8, sa, b8, sb, epi, bn):
    from gen3c_b200 import ops

    M, N = a8.shape[0], b8.shape[0]
    base = gate = out = None
    if epi == ops.EPI_GATED_RESIDUAL_F32:
        base = torch.randn(M, N, device="cuda")
        gate = torch.rand(N, device="cuda") + 0.5
        out = base.clone()
    got = ops.gemm_fp8(a8, sa, b8, sb, epilogue=epi, out=out, gate=gate, block_n=bn)
    return got, base, gate


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
def test_gemm_fp8_epilogues_and_tiles(epi, bn):
    """M = 200 and K = 336 are tails (not multiples of 128); N = 512 takes every tile width.  Negative controls: the
    result without scale_a, without scale_b, or with the two roles swapped misses the tolerance by >= 10x."""
    M, N, K = 200, 512, 336
    a8, sa, b8, sb = _operands(M, N, K, seed=epi * 10 + bn)
    got, base, gate = _run_gemm(a8, sa, b8, sb, epi, bn)
    acc = _exact(a8, sa, b8, sb)
    want = _epi_ref(acc, epi, base, gate)
    tol = TOL[epi]
    e = rel(got, want)
    assert e < tol, e
    ones_m, ones_n = torch.ones_like(sa), torch.ones_like(sb)
    wrong = [_exact(a8, ones_m, b8, sb), _exact(a8, sa, b8, ones_n)]
    sq = _operands(256, 256, K, seed=99)  # a square case for the swap
    got_sq, base_sq, gate_sq = _run_gemm(*sq, epi, bn)
    a8s, sas, b8s, sbs = sq
    assert rel(got_sq, _epi_ref(_exact(*sq), epi, base_sq, gate_sq)) < tol
    for w in wrong:
        assert rel(got, _epi_ref(w, epi, base, gate)) > 10 * tol
    swapped = _exact(a8s, sbs, b8s, sas)
    assert rel(got_sq, _epi_ref(swapped, epi, base_sq, gate_sq)) > 10 * tol


@pytest.mark.parametrize("M,N,K", [(130, 200, 64), (257, 72, 48), (64, 136, 1040), (1, 16, 16)])
def test_gemm_fp8_tails(M, N, K):
    for epi in (0, 3):
        a8, sa, b8, sb = _operands(M, N, K, seed=M + N + K)
        got, _, _ = _run_gemm(a8, sa, b8, sb, epi, 0)
        assert rel(got, _exact(a8, sa, b8, sb)) < TOL[epi]


def test_gemm_fp8_swapped_vt_shape():
    """V^T = W_v . xn^T: A is the weight (its row scales are the weight's), B the tokens."""
    from gen3c_b200 import ops

    D, L = 512, 384
    w8, sw, x8, sx = _operands(D, L, D, seed=4)
    got = ops.gemm_fp8(w8, sw, x8, sx)
    assert got.shape == (D, L) and rel(got, _exact(w8, sw, x8, sx)) < 3e-3


@pytest.mark.parametrize("with_rope", [True, False])
def test_gemm_norm_rope_fp8(with_rope):
    """The RMSNorm sees the dequantised accumulators: per-column weight scales change each head's norm."""
    from gen3c_b200 import ops

    M, N, K = 300, 512, 256
    a8, sa, b8, sb = _operands(M, N, K, seed=12, spread=1.0)
    gamma = 1 + 0.1 * torch.randn(128, device="cuda")
    cs = None
    if with_rope:
        ang = torch.rand(M, 64, device="cuda") * 6.0
        cs = torch.cat([ang.cos(), ang.sin()], 1).contiguous()
    got = ops.gemm_norm_rope_fp8(a8, sa, b8, sb, gamma, cs)
    acc = _exact(a8, sa, b8, sb).reshape(M, N // 128, 128)
    y = acc * torch.rsqrt(acc.pow(2).mean(-1, keepdim=True) + 1e-6) * gamma.double()
    if with_rope:
        c, s = cs[:, None, :64].double(), cs[:, None, 64:].double()
        y = torch.cat([y[..., :64] * c - y[..., 64:] * s, y[..., 64:] * c + y[..., :64] * s], -1)
    assert rel(got, y.reshape(M, N)) < 3e-3
    # without the column scales in the norm the result is visibly different
    acc_bad = _exact(a8, sa, b8, torch.ones_like(sb)).reshape(M, N // 128, 128)
    y_bad = acc_bad * torch.rsqrt(acc_bad.pow(2).mean(-1, keepdim=True) + 1e-6) * gamma.double()
    if not with_rope:
        assert rel(got, y_bad.reshape(M, N)) > 3e-2


@pytest.mark.parametrize("M,N,K", [(7040, 4096, 4096), (7040, 16384, 4096), (7040, 4096, 16384), (4096, 7040, 4096)])
def test_gemm_fp8_block_shapes(M, N, K):
    """The block's GEMMs at 7 040 tokens (D = 4 096, F = 16 384): q/k/v/out, layer1, layer2 and the swapped V^T."""
    a8, sa, b8, sb = _operands(M, N, K, seed=7, spread=1.0)
    for epi in (0, 3):
        got, _, _ = _run_gemm(a8, sa, b8, sb, epi, 0)
        assert rel(got, _exact(a8, sa, b8, sb)) < TOL[epi]


# ---------------------------------------------------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------------------------------------------------
WIDER = dit_oracle.DitCfg(model_channels=512, num_blocks=3, num_heads=4, ffn_dim=2048, context_dim=128, adaln_lora_dim=64,
                          max_frames=8, max_h=16, max_w=16)


def _engine_vs_oracle(cfg, shp, seed, device="cpu", sd=None, floor=False):
    dev = torch.device(device)
    sd = sd if sd is not None else dit_oracle.random_state_dict(cfg, seed=seed)
    inp = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in cases.dit_inputs(cfg, **shp, seed=seed + 1).items()}
    args = (inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp["ctx_c"])
    o32 = dit_oracle.forward(sd, cfg, *args)
    o8 = fp8_oracle.forward(sd, cfg, *args)
    net = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
    net.enable_fp8_linear()
    assert net.is_fp8_linear_enabled
    got = parity.engine_forward(net, inp, shp["T"], torch.device("cuda")).to(dev)
    e8, e32, eo = rel(got, o8), rel(got, o32), rel(o8, o32)
    bar = 5e-3
    if floor:
        # a quantised graph amplifies any difference in its inputs: a value moved by d relative crosses an e4m3 rounding
        # boundary (steps of 2^-3 relative) with probability ~ d / 2^-3 and then moves by a whole step, so the fp8
        # outputs of two graphs that differ at bf16 level differ by ~ sqrt(d * 2^-3), not by ~ d.  At full width the
        # bar is therefore the one test_fullsize_parity_gpu.py uses: the same fp8 graph run with bf16 storage against
        # the fp32 one (the reference's own inference precision), as for the bf16 engine against fp32.
        ob = fp8_oracle.forward(sd, cfg, *args, compute_dtype=torch.bfloat16).float()
        bar = max(bar, rel(ob, o8))
        print(f"fp8 graph with bf16 storage vs fp32 storage {bar:.3e}")
    print(f"engine fp8 vs oracle fp8 {e8:.3e}; engine fp8 vs fp32 {e32:.3e}; oracle fp8 vs fp32 {eo:.3e}")
    assert e8 <= bar and e32 <= eo + 5e-3
    return net, inp, got


@pytest.mark.parametrize("which", ["tiny", "wider"])
def test_engine_fp8_forward_matches_oracle_fp8(which):
    if which == "tiny":
        _engine_vs_oracle(cases.TINY, cases.TINY_SHAPE, seed=0)
    else:
        _engine_vs_oracle(WIDER, dict(T=3, H=16, W=32, ctx_len=256), seed=7)


@torch.no_grad()
def test_engine_fp8_fullwidth_block_7040_tokens():
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = cases.FULLWIDTH_1BLOCK
    sd = dit_oracle.random_state_dict_on(cfg, torch.device("cuda"), seed=21)
    _engine_vs_oracle(cfg, cases.FULLWIDTH_SHAPE, seed=21, device="cuda", sd=sd, floor=True)


def _forward(net, inp, T):
    return parity.engine_forward(net, inp, T, torch.device("cuda"))


def test_mode_switch_behaviour():
    """Two fp8 forwards are bit-identical; enable -> disable equals a net that never enabled the mode; an in-place
    weight update while the mode is on is re-quantised (the output equals a fresh net built with the new weights)."""
    cfg, shp = cases.TINY, cases.TINY_SHAPE
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    inp = cases.dit_inputs(cfg, **shp)
    T = shp["T"]
    plain = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
    ref = _forward(plain, inp, T)
    net = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
    _forward(net, inp, T)
    _forward(net, inp, T)  # the timestep's modulation vectors are cached after the first forward
    n_bf16 = net.last_launch_count()
    net.enable_fp8_linear()
    a, b = _forward(net, inp, T), _forward(net, inp, T)
    assert torch.equal(a, b) and not torch.equal(a, ref)
    assert net.last_launch_count() == n_bf16 + 3 * cfg.num_blocks  # per block: att (FA, CA) and hid quantisation
    assert net.workspace_bytes() > plain.workspace_bytes()
    net.disable_fp8_linear()
    assert torch.equal(_forward(net, inp, T), ref)
    _forward(net, inp, T)  # the workspace (and the cached modulation vectors) were reallocated by the switch
    assert net.last_launch_count() == n_bf16
    assert net.workspace_bytes() == plain.workspace_bytes()
    # in-place update with the mode on
    net.enable_fp8_linear()
    _forward(net, inp, T)
    sd2 = dit_oracle.random_state_dict(cfg, seed=9)
    with torch.no_grad():
        for k, p in net.state_dict(keep_vars=True).items():
            if "layer1" in k or "to_out" in k:
                p.copy_(sd2[k].to(bf))
    got = _forward(net, inp, T)
    fresh = parity.build_engine_net(cfg, {k: (sd2[k] if ("layer1" in k or "to_out" in k) else v) for k, v in sd.items()},
                                    cfg.num_blocks, "cuda")
    fresh.enable_fp8_linear()
    assert torch.equal(got, _forward(fresh, inp, T))


def test_denoise_step_fp8_matches_oracle_fp8():
    from gen3c_b200 import sampler

    cfg, shp = cases.TINY, cases.TINY_SHAPE
    T, H, W = shp["T"], shp["H"], shp["W"]
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    sig = dit_oracle.karras_sigmas(35)
    sigma, sigma_next, guidance = float(sig[20]), float(sig[21]), 1.5
    inp = cases.dit_inputs(cfg, **shp, x_scale=math.sqrt(sigma ** 2 + 0.25))
    noise = torch.from_numpy(dit_oracle.arch_invariant_rand((16, T, H, W), 1))
    ind = torch.zeros(T)
    ind[0] = 1.0

    def onet(x_in, t, cond):
        return fp8_oracle.forward(sd, cfg, x_in, inp["cond_mask"], inp["pose"] if cond else None, inp["padding"], t,
                                  inp["ctx_c"] if cond else inp["ctx_u"])

    want = dit_oracle.denoise_step(onet, inp["x"], inp["gt"], noise, ind, sigma, sigma_next, guidance)
    net = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
    net.enable_fp8_linear()
    got = sampler.denoise_step(net, inp["x"].cuda().to(bf), inp["gt"].cuda().to(bf), noise.cuda(), ind.cuda(),
                               inp["cond_mask"].cuda().to(bf), inp["pose"].cuda().to(bf), inp["padding"].cuda().to(bf),
                               inp["ctx_c"].cuda().to(bf), inp["ctx_u"].cuda().to(bf), sigma, sigma_next,
                               guidance).float().cpu()
    e = rel(got, want)
    print(f"fp8 denoise step x_(t-1) rel-L2 vs oracle fp8: {e:.3e}")
    assert e < 1e-3


def _cp_worker(rank, world, port, layout, ret):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from gen3c_b200 import sampler
        from gen3c_b200.parallel import cat_outputs_cp, split_inputs_cp

        cfg, T, H, W, M = cases.TINY, 4, 16, 16, 128
        sd = dit_oracle.random_state_dict(cfg, seed=3)
        inp = cases.dit_inputs(cfg, T, H, W, M, seed=5)
        net = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
        net.enable_fp8_linear()
        if layout == "cfg":
            net.enable_cfg_parallel(dist.group.WORLD)
            ind = torch.zeros(T, device="cuda")
            out = sampler.denoise_step(net, inp["x"].cuda().to(bf), inp["gt"].cuda().to(bf),
                                       torch.zeros(16, T, H, W, device="cuda"), ind, inp["cond_mask"].cuda().to(bf),
                                       inp["pose"].cuda().to(bf), inp["padding"].cuda().to(bf), inp["ctx_c"].cuda().to(bf),
                                       inp["ctx_u"].cuda().to(bf), 0.67, 0.5, 1.5)
        else:
            net.enable_context_parallel(dist.group.WORLD, mode=layout)
            x_local = split_inputs_cp(inp["x"][None].cuda().to(bf), 2, dist.group.WORLD)
            o = net(x=x_local, timesteps=torch.tensor([inp["timestep"]], device="cuda", dtype=bf),
                    crossattn_emb=inp["ctx_c"][None].cuda().to(bf), fps=torch.tensor([24.0], device="cuda"),
                    padding_mask=inp["padding"][None, None].cuda().to(bf),
                    condition_video_input_mask=inp["cond_mask"][None].cuda().to(bf),
                    condition_video_indicator=torch.zeros(1, 1, T, 1, 1, device="cuda", dtype=bf),
                    condition_video_pose=inp["pose"][None].cuda().to(bf))
            out = cat_outputs_cp(o, 2, dist.group.WORLD)[0]
        if rank == 0:
            ret.put(out.float().cpu())
        torch.cuda.synchronize()
        dist.barrier()
        net._teardown_barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("layout", ["p2p", "nccl", "cfg"])
def test_fp8_composes_with_parallelism(layout):
    """cp = 2 (both K/V exchanges) and CFG-parallel runs with the mode on equal the single-GPU fp8 result within the
    sharded-parity tolerance (5e-3)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    from gen3c_b200 import sampler

    cfg, T, H, W, M = cases.TINY, 4, 16, 16, 128
    sd = dit_oracle.random_state_dict(cfg, seed=3)
    inp = cases.dit_inputs(cfg, T, H, W, M, seed=5)
    net = parity.build_engine_net(cfg, sd, cfg.num_blocks, "cuda")
    net.enable_fp8_linear()
    if layout == "cfg":
        want = sampler.denoise_step(net, inp["x"].cuda().to(bf), inp["gt"].cuda().to(bf),
                                    torch.zeros(16, T, H, W, device="cuda"), torch.zeros(T, device="cuda"),
                                    inp["cond_mask"].cuda().to(bf), inp["pose"].cuda().to(bf),
                                    inp["padding"].cuda().to(bf), inp["ctx_c"].cuda().to(bf), inp["ctx_u"].cuda().to(bf),
                                    0.67, 0.5, 1.5).float().cpu()
    else:
        want = _forward(net, inp, T).cpu()
    del net
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29700 + (os.getpid() % 1000) + {"p2p": 0, "nccl": 3, "cfg": 6}[layout]
    procs = [ctx.Process(target=_cp_worker, args=(r, 2, port, layout, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = ret.get(timeout=400)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert rel(got, want) < 5e-3, rel(got, want)


def test_single_image_entry_point_with_fp8_linear(tmp_path):
    from tests.test_entry_point_gpu import _args, _pipeline

    m, args = _args(tmp_path)
    args.fp8_linear = True
    pipe = _pipeline(args)
    (path, video), = m.demo(args, pipeline=pipe)
    assert pipe.model.net.is_fp8_linear_enabled
    assert video.dtype == "uint8" and video.shape[0] == 121
