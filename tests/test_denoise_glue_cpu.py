"""tests/sampler_ref64.py pinned to the oracle, without a GPU.

dit_oracle.denoise_step runs with a fake network that returns fixed bf16 tensors, so its x~, x_in, CFG-combined network
output and x_next depend on the glue alone.  Each must meet the per-element criterion of sampler_ref64 against the
float64 restatement of the same tensors, and every negative control of the restatement must miss it.  The step cases
(STEP_CASES, step_inputs) are shared with tests/test_denoise_glue_gpu.py.
"""
from collections import namedtuple

import numpy as np
import pytest
import torch

from gen3c_b200.sampler import EDMEulerScheduler
from oracle import dit_oracle
from tests import sampler_ref64 as r64

bf = torch.bfloat16
SIGMAS = EDMEulerScheduler().set_timesteps(35).sigmas  # fp32, 35 steps then 0

# frames: the conditioned latent frames (indicator 1); sigma: a schedule index i (sigma_i -> sigma_i+1), or "at_aug" /
# "above_aug" (sigma = fp32(sigma_aug) or the next fp32 value above it, sigma' = sigma / 2); uncond: the uncond branch's
# input mask, None (the cond mask) or "zeros"
StepCase = namedtuple("StepCase", "T H W frames guidance sigma_data sigma_aug sigma padding uncond")
STEP_CASES = {
    "t1_none": StepCase(1, 16, 64, [], 1.5, 0.5, 0.001, 20, True, None),
    "t1_all_g7": StepCase(1, 16, 64, [0], 7.0, 1.0, 0.5, 10, True, "zeros"),
    "t3_frame0_g0_nopad": StepCase(3, 16, 32, [0], 0.0, 0.5, 0.001, 20, False, None),
    "t3_frames01_g1": StepCase(3, 16, 32, [0, 1], 1.0, 1.0, 0.5, 15, True, "zeros"),
    "t3_all_sigma_max": StepCase(3, 16, 32, [0, 1, 2], 1.5, 0.5, 0.001, 0, True, None),
    "t4_alternate_g7": StepCase(4, 16, 16, [1, 3], 7.0, 0.5, 0.5, 12, False, "zeros"),
    "t4_at_aug": StepCase(4, 16, 16, [0, 1, 3], 1.5, 0.5, 0.5, "at_aug", True, None),
    "t4_above_aug": StepCase(4, 16, 16, [0, 1, 3], 1.5, 1.0, 0.5, "above_aug", True, "zeros"),
    "t3_at_default_aug": StepCase(3, 16, 32, [0, 1], 1.5, 0.5, 0.001, "at_aug", True, None),
    "t3_above_default_aug": StepCase(3, 16, 32, [0, 1], 1.5, 0.5, 0.001, "above_aug", False, None),
    "t3_final_step": StepCase(3, 16, 32, [0], 1.5, 0.5, 0.001, 34, True, None),
}


def case_sigmas(c):
    """(sigma, sigma') as the fp32 numbers the kernels receive."""
    if c.sigma == "at_aug":
        s = np.float32(c.sigma_aug)
    elif c.sigma == "above_aug":
        s = np.nextafter(np.float32(c.sigma_aug), np.float32(np.inf))
    else:
        return float(SIGMAS[c.sigma]), float(SIGMAS[c.sigma + 1])
    return float(s), float(s / np.float32(2))


def step_inputs(c, sigma, seed=0, pose_channels=64, ctx_len=128, ctx_dim=64, device="cpu"):
    """The step's inputs at their storage types: xt, gt bf16 [16, T, H, W]; noise f32; ind f32 [T]; cond_mask bf16
    [1, T, H, W] (the indicator per frame); pose bf16; padding bf16 [H, W] (binary) or None; ctx_c / ctx_u bf16."""
    g = torch.Generator().manual_seed(seed)
    T, H, W = c.T, c.H, c.W
    r = lambda *shape, s=1.0: (s * torch.randn(*shape, generator=g)).to(bf)  # noqa: E731
    ind = torch.zeros(T)
    ind[c.frames] = 1.0
    d = dict(xt=r(16, T, H, W, s=float(np.sqrt(sigma ** 2 + c.sigma_data ** 2))), gt=r(16, T, H, W, s=0.5),
             noise=torch.from_numpy(dit_oracle.arch_invariant_rand((16, T, H, W), seed + 1)), ind=ind,
             cond_mask=ind.reshape(1, T, 1, 1).expand(1, T, H, W).to(bf), pose=r(pose_channels, T, H, W, s=0.5),
             padding=(torch.rand(H, W, generator=g) < 0.3).to(bf) if c.padding else None,
             ctx_c=r(ctx_len, ctx_dim), ctx_u=r(ctx_len, ctx_dim))
    return {k: (v.to(device).contiguous() if torch.is_tensor(v) else v) for k, v in d.items()}


def oracle_step(monkeypatch, c, d, oc, ou):
    """dit_oracle.denoise_step with a network returning oc / ou; its bf16-rounded intermediates are recorded."""
    sigma, sigma_next = case_sigmas(c)
    seen = []
    rounding = dit_oracle.bf16

    def record(t):
        seen.append(rounding(t))
        return seen[-1]

    monkeypatch.setattr(dit_oracle, "bf16", record)
    net = lambda x_in, t, cond: (oc if cond else ou).float()  # noqa: E731
    # every sigma as its fp32 value, so that the oracle's float64 `sigma_aug >= sigma` is the kernels' fp32 comparison
    nxt, net_o = dit_oracle.denoise_step(net, d["xt"].float(), d["gt"].float(), d["noise"], d["ind"], sigma,
                                         sigma_next, r64.f32(c.guidance), r64.f32(c.sigma_data), r64.f32(c.sigma_aug),
                                         return_net_output=True)
    monkeypatch.setattr(dit_oracle, "bf16", rounding)
    xtilde, xin = seen[0], seen[1]  # x~, then x_in (then t, the two branch outputs and x_next)
    # the oracle returns the network output in fp32; the kernel stores it in bf16, one rounding of the same fp32 value
    return dict(xt=d["xt"], gt=d["gt"], noise=d["noise"], ind=d["ind"], sigma=sigma, sigma_next=sigma_next,
                sigma_aug=c.sigma_aug, sigma_data=c.sigma_data, guidance=c.guidance, xtilde=xtilde, xin=xin, oc=oc,
                ou=ou, net=rounding(net_o), xnext=nxt)


def fake_outputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (16, c.T, c.H, c.W)
    return (torch.randn(shape, generator=g).to(bf), (0.7 * torch.randn(shape, generator=g)).to(bf))


@pytest.mark.parametrize("name", list(STEP_CASES))
def test_restatement_matches_oracle(monkeypatch, name):
    c = STEP_CASES[name]
    sigma, _ = case_sigmas(c)
    d = step_inputs(c, sigma, seed=3)
    s = oracle_step(monkeypatch, c, d, *fake_outputs(c, 4))
    v = r64.verdicts(s)
    print(name, {k: f"{x.ratio:.2f}" for k, x in v.items()})
    for k, x in v.items():
        assert x.ok, (k, x)
    # frames whose effective indicator is 0 pass xt through unchanged
    off = r64.indicator64(d["ind"], d["xt"].shape, sigma, c.sigma_aug) == 0
    assert torch.equal(s["xtilde"][off], d["xt"].float()[off])


# (case, controls that apply to it): the noise, frame and replacement controls need augmented frames next to plain ones
CONTROL_CASES = {
    "t4_alternate_g7": ("no_noise", "cin_sigma_next", "frame_major", "replace_before_store", "next_from_xin"),
    # sigma' = sigma / 2 = 5e-4 changes sqrt(sigma^2 + sd^2) by 1.5e-6 only: no cin_sigma_next here
    "t3_above_default_aug": ("no_noise", "frame_major", "replace_before_store", "next_from_xin"),
    "t4_at_aug": ("ind_always_on",),
    "t3_final_step": ("ind_always_on", "next_from_xin"),
}


@pytest.mark.parametrize("name", list(CONTROL_CASES))
def test_negative_controls_miss_oracle(monkeypatch, name):
    c = STEP_CASES[name]
    sigma, _ = case_sigmas(c)
    d = step_inputs(c, sigma, seed=3)
    s = oracle_step(monkeypatch, c, d, *fake_outputs(c, 4))
    for k, v in r64.control_verdicts(s, CONTROL_CASES[name]).items():
        print(name, k, v)
        assert v.broken(), (k, v)


def bf16_grid_rounds_like_torch(device):
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(100000, generator=g) * 10.0 ** torch.randint(-6, 6, (100000,), generator=g),
                   torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 0.0, 255.5, -0.99951171875]),
                   2.0 ** torch.arange(-120, 120)]).to(device)
    rn = r64._bf16_grid(x.double())[0]
    assert torch.equal(rn, x.to(bf).double())
    # an output equal to a bf16 reference passes with E = 0, and one bf16 ulp off fails
    v = r64.Verdict(x.to(bf), x.to(bf).double(), torch.zeros_like(x, dtype=torch.float64), 1.0)
    assert v.ok
    off = r64.Verdict(x.to(bf)[:-240], x.to(bf).double()[:-240] * (1 + 2 ** -7) + 2 ** -100,
                      torch.zeros(x.numel() - 240, dtype=torch.float64, device=device), 1.0)
    assert off.bad == off.n


def test_bf16_grid_rounds_like_torch():
    """RN_bf16 of _bf16_grid against torch's fp32 -> bf16 cast on fp32-exact values (a single rounding), midpoints,
    powers of two and both signs included; the criterion at E = 0."""
    bf16_grid_rounds_like_torch("cpu")
