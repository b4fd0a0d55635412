"""The denoise step's sampler glue, element by element, with the network taken out of the comparison.

g3c_denoise_step is k_sampler_pre, the conditional and the unconditional DiT forward, then k_sampler_post.  The oracle
tests compare its x_next with the fp32 oracle at rel-L2 1e-3, where the network's own error hides a glue error such as
a dropped s_aug * noise term (about 1e-3 relative on the augmented frames, under one bf16 ulp).  Here each step is read
back through g3c_dit_read_step (x~, x_in and the two branch outputs post read) and

1. x~: frames whose effective indicator is 0 equal xt bitwise; the others meet the criterion of tests/sampler_ref64.py
   against pre64;
2. x_in meets it against x~ / sqrt(sigma^2 + sd^2) of the read-back x~;
3. both branch outputs are torch.equal to g3c_dit_forward of the read-back x_in at t = bf16(fp32(0.25 ln sigma)), with
   the arguments of their branch (the uncond forward with the pose, or one bf16 ulp off in t, must differ);
4. the network output and x_next meet the criterion against post64 of the read-back x~, oc and ou;
5. the step's launch count is 2 plus those of its two forwards.

The nets are the signal-carrying nets of test_engine_signal_gpu.py, so a wrong branch input changes the forward's bits.
"""
import ctypes as C
import functools
import math

import pytest
import torch

from oracle import cases, dit_oracle
from tests import sampler_ref64 as r64
from tests.test_denoise_glue_cpu import (CONTROL_CASES, STEP_CASES, StepCase, bf16_grid_rounds_like_torch, case_sigmas,
                                         step_inputs)
from tests.test_engine_signal_gpu import build_net, signal_state_dict

pytestmark = pytest.mark.gpu

bf = torch.bfloat16
ESTATE = -4
# one block of D = 256 whose position tables hold the benchmark's 16 x 44 x 80 patch grid
BENCH_CFG = dit_oracle.DitCfg(model_channels=256, num_blocks=1, num_heads=2, ffn_dim=1024, context_dim=64,
                              adaln_lora_dim=32, max_frames=16, max_h=48, max_w=88)
OBSERVED: dict = {}  # largest ratio per output over the file's steps, for re-deriving the K of sampler_ref64


@functools.lru_cache(maxsize=None)
def net_for(kind):
    cfg = BENCH_CFG if kind == "bench" else cases.TINY
    return cfg, build_net(cfg, signal_state_dict(cfg, 0), fp8=kind == "tiny_fp8")


def lib():
    from gen3c_b200 import _lib

    return _lib.load()


def ptr(t):
    return None if t is None else t.data_ptr()


def read_step(net, like):
    bufs = [torch.full_like(like, float("nan")) for _ in range(4)]
    rc = lib().g3c_dit_read_step(net._engine(), *(b.data_ptr() for b in bufs), torch.cuda.current_stream().cuda_stream)
    return rc, bufs


def forward(net, x, mask, pose, pad, t, ctx):
    """g3c_dit_forward on the step's handle: (output, launches)."""
    out = torch.empty_like(x)
    rc = lib().g3c_dit_forward(net._engine(), ptr(x), ptr(mask), ptr(pose), ptr(pad), t, ptr(ctx), out.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib().g3c_last_error()
    net._glue_last_t = (net._shape_key, t)
    return out, net.last_launch_count()


def t_ref(sigma):
    """The timestep the step feeds the net, computed on the host as the oracle does."""
    return float(torch.tensor(0.25 * math.log(sigma), dtype=torch.float32).to(bf))


def next_bf16(t):
    return float(torch.tensor([t], dtype=bf).view(torch.int16).add(1).view(bf))


def note(name, v):
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), v.ratio)


def checked_step(net, cfg, c, d, sigma, sigma_next, xt=None):
    """One sampler.denoise_step with checks 1-5; returns the step dict of sampler_ref64.verdicts."""
    from gen3c_b200 import sampler

    xt = d["xt"] if xt is None else xt
    mask_u = torch.zeros_like(d["cond_mask"]) if c.uncond == "zeros" else None
    net_o = torch.full_like(xt, float("nan"))
    t = t_ref(sigma)
    last = getattr(net, "_glue_last_t", None)
    x_next = sampler.denoise_step(net, xt, d["gt"], d["noise"], d["ind"], d["cond_mask"], d["pose"], d["padding"],
                                  d["ctx_c"], d["ctx_u"], sigma, sigma_next, c.guidance, c.sigma_data, c.sigma_aug,
                                  cond_mask_uncond=mask_u, net_output=net_o)
    n_step = net.last_launch_count()
    # the step's first forward reuses the adaLN vectors only if the handle's last forward ran at t on this shape
    first_cached = last == (net._shape_key, t)
    rc, (xtilde, xin, oc, ou) = read_step(net, xt)
    assert rc == 0, lib().g3c_last_error()
    s = dict(xt=xt, gt=d["gt"], noise=d["noise"], ind=d["ind"], sigma=sigma, sigma_next=sigma_next,
             sigma_aug=c.sigma_aug, sigma_data=c.sigma_data, guidance=c.guidance, xtilde=xtilde, xin=xin, oc=oc,
             ou=ou, net=net_o, xnext=x_next)
    # 1, 2, 4: the glue, element by element
    off = r64.indicator64(d["ind"], xt.shape, sigma, c.sigma_aug) == 0
    assert torch.equal(xtilde[off], xt[off])
    for k, v in r64.verdicts(s).items():
        note(k, v)
        assert v.ok, (k, v)
    # 3: what each branch was fed.  The replays reuse the adaLN vectors of t (the step's second forward ran at t); the
    # control at t + 1 ulp recomputes them.
    got_c, n_cached = forward(net, xin, d["cond_mask"], d["pose"], d["padding"], t, d["ctx_c"])
    got_u, n_u = forward(net, xin, d["cond_mask"] if mask_u is None else mask_u, None, d["padding"], t, d["ctx_u"])
    assert torch.equal(got_c, oc) and torch.equal(got_u, ou)
    posed, _ = forward(net, xin, d["cond_mask"] if mask_u is None else mask_u, d["pose"], d["padding"], t, d["ctx_u"])
    assert not torch.equal(posed, ou)
    shifted, n_full = forward(net, xin, d["cond_mask"], d["pose"], d["padding"], next_bf16(t), d["ctx_c"])
    assert not torch.equal(shifted, oc)
    # 5: sampler_pre + both forwards + sampler_post
    assert n_u == n_cached and n_full == n_cached + 6 * cfg.num_blocks + 5
    assert n_step == 2 + (n_cached if first_cached else n_full) + n_cached, (n_step, n_full, n_cached)
    return s


def gpu_inputs(c, sigma, cfg, seed=3):
    return step_inputs(c, sigma, seed=seed, pose_channels=cfg.in_channels - 17, ctx_dim=cfg.context_dim,
                       device="cuda")


@pytest.mark.parametrize("name", list(STEP_CASES))
@torch.no_grad()
def test_step_glue_matches_float64(name):
    """Indicator patterns none / frame 0 / frames 0-1 / all / [0, 1, 0, 1] on T = 1, 3, 4 and non-square grids;
    guidance 0, 1, 1.5, 7; sigma_data 0.5, 1; sigma_aug 0.001, 0.5; sigma at fp32(sigma_aug) and one fp32 ulp above;
    sigma = 80 and the final step to 0; the padding mask absent and present; cond_mask_uncond NULL and zeros."""
    c = STEP_CASES[name]
    cfg, net = net_for("tiny")
    sigma, sigma_next = case_sigmas(c)
    checked_step(net, cfg, c, gpu_inputs(c, sigma, cfg), sigma, sigma_next)
    print(name, {k: round(v, 3) for k, v in OBSERVED.items()})


@torch.no_grad()
def test_all_35_steps_chained():
    """The default 35-step schedule as one loop, each step fed the engine's own x_next: sigma = 80 first, the two steps
    below sigma_aug = 0.001 and the final sigma' = 0 included."""
    cfg, net = net_for("tiny")
    base = StepCase(3, 16, 32, [0], 1.5, 0.5, 0.001, 0, True, None)
    sigma0, _ = case_sigmas(base)
    d = gpu_inputs(base, sigma0, cfg, seed=11)
    xt = d["xt"]
    for i in range(35):
        c = base._replace(sigma=i)
        sigma, sigma_next = case_sigmas(c)
        xt = checked_step(net, cfg, c, d, sigma, sigma_next, xt=xt)["xnext"]
    assert torch.isfinite(xt.float()).all()
    print("chained", {k: round(v, 3) for k, v in OBSERVED.items()})


@torch.no_grad()
def test_benchmark_shape():
    """Latent [16, 16, 88, 160] (56 320 tokens), frames 0 and 1 conditioned, sigma above and below sigma_aug: each
    thread of the grid-stride sampler kernels runs about 27 iterations."""
    cfg, net = net_for("bench")
    for i in (20, 33):
        c = StepCase(16, 88, 160, [0, 1], 1.5, 0.5, 0.001, i, True, None)
        sigma, sigma_next = case_sigmas(c)
        checked_step(net, cfg, c, gpu_inputs(c, sigma, cfg), sigma, sigma_next)
    print("bench shape", {k: round(v, 3) for k, v in OBSERVED.items()})


@torch.no_grad()
def test_fp8_linear_mode():
    """The same glue around the fp8 forward: the replays run on the fp8 handle, and a bf16 net's forward differs."""
    cfg, net = net_for("tiny_fp8")
    c = STEP_CASES["t3_frames01_g1"]
    sigma, sigma_next = case_sigmas(c)
    d = gpu_inputs(c, sigma, cfg)
    s = checked_step(net, cfg, c, d, sigma, sigma_next)
    _, bf16_net = net_for("tiny")
    bf16_net._sync_weights()
    bf16_net._set_shape(c.T, c.H, c.W, d["ctx_c"].shape[0], 24.0)
    plain, _ = forward(bf16_net, s["xin"], d["cond_mask"], d["pose"], d["padding"], t_ref(sigma), d["ctx_c"])
    assert not torch.equal(plain, s["oc"])


@pytest.mark.parametrize("name", list(CONTROL_CASES))
@torch.no_grad()
def test_negative_controls(name):
    """Wrong restatements of the glue on the engine's own step must break the criterion (sampler_ref64.control_verdicts):
    noise term dropped, c_in from sigma', indicator on at sigma <= sigma_aug, frame read from a [T, 16, H, W] layout,
    replacement before net_output is stored, x_next from x_in."""
    c = STEP_CASES[name]
    cfg, net = net_for("tiny")
    sigma, sigma_next = case_sigmas(c)
    s = checked_step(net, cfg, c, gpu_inputs(c, sigma, cfg), sigma, sigma_next)
    for k, v in r64.control_verdicts(s, CONTROL_CASES[name]).items():
        print(name, k, v)
        assert v.broken(), (k, v)


def test_bf16_grid_on_gpu():
    """The criterion's bf16 rounding on the device the checks run on."""
    bf16_grid_rounds_like_torch("cuda")


@torch.no_grad()
def test_read_step_needs_a_step():
    """g3c_dit_read_step is G3C_ESTATE before the first step, after g3c_dit_set_shape (same shape included) and after
    g3c_dit_set_linear_fp8, and writes nothing then."""
    cfg = cases.TINY
    net = build_net(cfg, signal_state_dict(cfg, 0))
    c = STEP_CASES["t3_frame0_g0_nopad"]
    sigma, sigma_next = case_sigmas(c)
    d = gpu_inputs(c, sigma, cfg)
    net._sync_weights()
    net._set_shape(c.T, c.H, c.W, 128, 24.0)
    rc, bufs = read_step(net, d["xt"])
    assert rc == ESTATE and all(torch.isnan(b.float()).all() for b in bufs)
    checked_step(net, cfg, c, d, sigma, sigma_next)
    assert read_step(net, d["xt"])[0] == 0
    assert lib().g3c_dit_set_shape(net._engine(), c.T, c.H, c.W, 128, C.c_float(24.0)) == 0
    assert read_step(net, d["xt"])[0] == ESTATE
    checked_step(net, cfg, c, d, sigma, sigma_next)
    net.enable_fp8_linear()
    assert read_step(net, d["xt"])[0] == ESTATE
    s = checked_step(net, cfg, c, d, sigma, sigma_next)
    assert read_step(net, d["xt"])[0] == 0 and torch.isfinite(s["oc"].float()).all()
