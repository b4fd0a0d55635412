"""Float64 restatement of the denoise step's sampler glue, with a per-element error budget.

The glue is k_sampler_pre / k_sampler_post (dit_elementwise.cu), restated from dit_oracle.denoise_step and SURVEY.md
§B.3.  Inputs are taken at their exact values (bf16 latents, fp32 noise) and every sigma as the fp32 number the kernels
receive.  The effective indicator is 0 when sigma_aug >= sigma in fp32, as the kernels (and torch's comparison of a
Python float with the reference's fp32 sigma tensor) decide it.

Each function returns the float64 value of a bf16 output and E, the budget for the kernels' fp32 evaluation of it:
E = K * 2^-24 * (a sum of the magnitudes the fp32 roundings scale with).  The criterion (`Verdict`) requires
RN_bf16(ref) exactly, except where ref lies within E of a bf16 rounding midpoint, where either neighbour is accepted;
and |out - ref| <= ulp/2 + E everywhere.

The K below are about 4x the largest ratio observed on one H100 80GB HBM3 (132 SMs, 700 W power limit) over
tests/test_denoise_glue_gpu.py, or the derived worst case where no ratio could be observed.  A ratio is seen only where
the kernel's bf16 output is not RN_bf16(ref): the distance from ref to the values that round to the output, over E / K,
is then a lower bound on that element's fp32 error in units of E / K.  dit_oracle.denoise_step reaches 2.05 and 0.37
on the cases of tests/test_denoise_glue_cpu.py.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
# x~ = RN(ind * (gt + noise * s_aug) * c_in_aug * sqrt(sigma^2 + sd^2)), E / K = 2^-24 (|gt| + |s_aug noise|) * scale:
# observed 2.05 (derived worst case about 7: two roundings in the sum, about 2.5 in each fp32 constant, two products)
K_XTILDE = 8.0
# x_in = RN(x~ * c_in), E / K = 2^-24 |x_in|: no element crossed a midpoint, so K is the derived worst case (about 2.5 in
# the fp32 c_in, one product)
K_XIN = 4.0
# net_output = RN(oc + g (oc - ou)), E / K = 2^-24 ((1 + g) |oc| + g |ou|): no crossing; oc - ou of two bf16 values is
# exact, and so is the rest for a g of few significant bits (0, 1, 1.5, 7).  K is the derived worst case (two roundings).
K_NET = 2.0
# x_next, E / K = 2^-24 (|x~| + r (|x~| + |x0| + c_out ((1 + g) |oc| + g |ou|) + |gt|)), r = (sigma - sigma') / sigma:
# observed 0.35 (derived worst case about 12; the budget's terms rarely add up in one element)
K_NEXT = 1.5


def f32(x) -> float:
    return float(np.float32(x))


def aug_on(sigma, sigma_aug) -> bool:
    """The conditioning frames are augmented unless sigma_aug >= sigma, compared in fp32."""
    return not (np.float32(sigma_aug) >= np.float32(sigma))


def indicator64(ind_t, shape, sigma, sigma_aug, variant=None) -> torch.Tensor:
    """The effective per-element indicator of a [16, T, H, W] latent (element i is frame (i / (H*W)) % T).
    frame_major reads the frame as if the layout were [T, 16, H, W]; ind_always_on ignores the sigma_aug switch."""
    C, T, H, W = shape
    ind = ind_t.double().to(ind_t.device).reshape(-1)
    assert ind.numel() == T and bool(((ind == 0) | (ind == 1)).all()), "the indicator is 0 or 1 per frame"
    if not aug_on(sigma, sigma_aug) and variant != "ind_always_on":
        ind = torch.zeros_like(ind)
    if variant == "frame_major":
        i = torch.arange(C * T * H * W, device=ind.device)
        return ind[i // (C * H * W)].reshape(shape)
    return ind.reshape(1, T, 1, 1).expand(shape)


def pre64(xt, gt, noise, ind_t, sigma, sigma_aug, sigma_data, variant=None):
    """x~ = ind * aug + (1 - ind) * xt,  aug = (gt + s_aug * noise) / sqrt(s_aug^2 + sd^2) * sqrt(sigma^2 + sd^2).
    Returns (x~ in float64, E).  E is 0 where the indicator is 0: x~ is then xt itself."""
    s, sa, sd = f32(sigma), f32(sigma_aug), f32(sigma_data)
    ind = indicator64(ind_t, xt.shape, s, sa, variant)
    scale = math.sqrt(s * s + sd * sd) / math.sqrt(sa * sa + sd * sd)
    n = noise.double() * sa
    g = gt.double()
    ref = ind * ((g + n) * scale) + (1 - ind) * xt.double()
    return ref, K_XTILDE * U * ind * (g.abs() + n.abs()) * scale


def xin64(xtilde, sigma, sigma_data):
    """x_in = x~ / sqrt(sigma^2 + sd^2).  Returns (x_in in float64, E)."""
    s, sd = f32(sigma), f32(sigma_data)
    ref = xtilde.double() / math.sqrt(s * s + sd * sd)
    return ref, K_XIN * U * ref.abs()


def post64(xtilde, oc, ou, gt, ind_t, guidance, sigma, sigma_next, sigma_aug, sigma_data, variant=None):
    """The CFG combination o = oc + g (oc - ou) (the network output users see), the replacement on conditioned frames
    o <- ind (gt - c_skip x~) / c_out + (1 - ind) o, and the Euler step x_next = x~ + (x~ - x0) / sigma * (sigma' - sigma)
    with x0 = c_skip x~ + c_out o.  Returns ((net_output, E), (x_next, E)) in float64.
    replace_before_store returns the replaced o as the network output."""
    s, sn, sd, g = f32(sigma), f32(sigma_next), f32(sigma_data), f32(guidance)
    ind = indicator64(ind_t, xtilde.shape, s, sigma_aug, variant)
    xs, c, u, gt = xtilde.double(), oc.double(), ou.double(), gt.double()
    c_skip = sd * sd / (s * s + sd * sd)
    c_out = s * sd / math.sqrt(s * s + sd * sd)
    o = c + g * (c - u)
    mag_o = (1 + abs(g)) * c.abs() + abs(g) * u.abs()
    o_rep = ind * ((gt - c_skip * xs) / c_out) + (1 - ind) * o
    x0 = c_skip * xs + c_out * o_rep
    nxt = xs + (xs - x0) / s * (sn - s)
    r = (s - sn) / s
    e_next = K_NEXT * U * (xs.abs() + r * (xs.abs() + x0.abs() + c_out * mag_o + gt.abs()))
    net = o_rep if variant == "replace_before_store" else o
    return (net, K_NET * U * mag_o), (nxt, e_next)


def _bf16_grid(ref):
    """(RN_bf16(ref) with ties to even, the bf16 spacing at |ref|) of a float64 tensor.  The spacing is built from the
    exponent bits (log2 / pow on the GPU are not exact at every power of two)."""
    biased = ref.abs().clamp_min(2.0 ** -126).view(torch.int64) >> 52
    ulp = ((biased - 7) << 52).view(torch.float64)
    q = torch.floor(ref / ulp)
    lo, hi = q * ulp, (q + 1) * ulp
    mid = lo + ulp / 2
    even = torch.remainder(q, 2) == 0
    return torch.where(ref < mid, lo, torch.where(ref > mid, hi, torch.where(even, lo, hi))), ulp


class Verdict:
    """The criterion applied to one output: out must be RN_bf16 of some value within E of ref, which is RN_bf16(ref),
    or its other neighbour where ref lies within E of the midpoint (more values only where E exceeds an ulp), and
    |out - ref| <= ulp/2 + E.  `bad` counts the elements that break it; `ratio` is the largest distance from ref to the
    values that round to out, in units of E / K, over elements where out is not RN_bf16(ref) (the kernel's fp32 error
    there was at least that); `excess` the largest (|out - ref| - ulp/2) / E over elements with E > 0."""

    def __init__(self, out, ref, E, K):
        o = out.double()
        rn = _bf16_grid(ref)[0]
        ulp = _bf16_grid(ref.abs() + E)[1]
        ok = (_bf16_grid(ref - E)[0] <= o) & (o <= _bf16_grid(ref + E)[0]) & ((o - ref).abs() <= ulp / 2 + E)
        self.n = ref.numel()
        self.bad = int((~ok).sum())
        # distance from ref to the interval that rounds to out (sign-normalised by out; its inner gap is half as wide
        # when |out| is a power of two)
        sgn = torch.where(o < 0, -1.0, 1.0).to(o)
        a, r = o.abs(), ref * sgn
        ulp_o = _bf16_grid(a)[1]
        ulp_in = torch.where(torch.frexp(a).mantissa == 0.5, ulp_o / 2, ulp_o)
        dist = torch.where(r > a, r - a - ulp_o / 2, a - r - ulp_in / 2)
        crossed = (o != rn) & (E > 0) & (o != 0)
        self.ratio = float((dist / E * K)[crossed].max()) if bool(crossed.any()) else 0.0
        pos = E > 0
        self.excess = float((((o - ref).abs() - ulp / 2) / E)[pos].max()) if bool(pos.any()) else 0.0
        self.first = None  # (flat index, out, ref, E) of the first bad element
        if self.bad:
            i = int(torch.nonzero(~ok.reshape(-1))[0])
            self.first = (i, float(o.reshape(-1)[i]), float(ref.reshape(-1)[i]), float(E.reshape(-1)[i]))

    @property
    def ok(self) -> bool:
        return self.bad == 0

    def broken(self) -> bool:
        """A negative control: the criterion fails on many elements, or by more than 10x E."""
        return self.bad >= max(64, self.n // 1000) or self.excess > 10.0

    def __repr__(self):
        return f"Verdict(bad={self.bad}/{self.n}, ratio={self.ratio:.3g}, excess={self.excess:.3g}, first={self.first})"


def verdicts(s):
    """The criterion on every output of one step.  s: dict with the step's inputs xt, gt, noise, ind, sigma,
    sigma_next, sigma_aug, sigma_data, guidance and its outputs xtilde, xin, oc, ou, net, xnext (the x~ and the branch
    outputs the step itself read, so each output is checked against exact inputs of its own stage)."""
    a = (s["sigma"], s["sigma_aug"], s["sigma_data"])
    xt, E = pre64(s["xt"], s["gt"], s["noise"], s["ind"], *a)
    xi, Ei = xin64(s["xtilde"], s["sigma"], s["sigma_data"])
    (net, En), (nxt, Ex) = post64(s["xtilde"], s["oc"], s["ou"], s["gt"], s["ind"], s["guidance"], s["sigma"],
                                  s["sigma_next"], s["sigma_aug"], s["sigma_data"])
    return {"xtilde": Verdict(s["xtilde"], xt, E, K_XTILDE), "xin": Verdict(s["xin"], xi, Ei, K_XIN),
            "net": Verdict(s["net"], net, En, K_NET), "xnext": Verdict(s["xnext"], nxt, Ex, K_NEXT)}


def control_verdicts(s, names):
    """Wrong restatements of the glue, applied to one step (same dict as `verdicts`); each must be `broken()`.
    no_noise             the s_aug * noise term dropped (x~)
    cin_sigma_next       x_in = x~ / sqrt(sigma'^2 + sd^2) (x_in)
    ind_always_on        conditioned frames replaced even when sigma_aug >= sigma (x~)
    frame_major          the frame of element i read as if the layout were [T, 16, H, W] (x~)
    replace_before_store the replaced o returned as the network output (net_output)
    next_from_xin        the Euler step taken from x_in instead of x~ (x_next)"""
    a = (s["sigma"], s["sigma_aug"], s["sigma_data"])
    post = lambda xs, variant=None: post64(xs, s["oc"], s["ou"], s["gt"], s["ind"], s["guidance"],  # noqa: E731
                                           s["sigma"], s["sigma_next"], s["sigma_aug"], s["sigma_data"], variant)
    out = {}
    for name in names:
        if name == "no_noise":
            out[name] = Verdict(s["xtilde"], *pre64(s["xt"], s["gt"], torch.zeros_like(s["noise"]), s["ind"], *a),
                                K_XTILDE)
        elif name == "cin_sigma_next":
            out[name] = Verdict(s["xin"], *xin64(s["xtilde"], s["sigma_next"], s["sigma_data"]), K_XIN)
        elif name in ("ind_always_on", "frame_major"):
            out[name] = Verdict(s["xtilde"], *pre64(s["xt"], s["gt"], s["noise"], s["ind"], *a, variant=name),
                                K_XTILDE)
        elif name == "replace_before_store":
            out[name] = Verdict(s["net"], *post(s["xtilde"], name)[0], K_NET)
        elif name == "next_from_xin":
            out[name] = Verdict(s["xnext"], *post(s["xin"])[1], K_NEXT)
        else:
            raise ValueError(name)
    return out
