"""Float64 restatement of the attention kernel (gen3c_b200/csrc/attn_wgmma.cu, k_attn_fwd) with a per-element error
bound and a per-(row, head) statistical bar.

Test infrastructure only.  Per head (128 dims) and query row the kernel computes

    o = bf16( sum_j bf16(p_j) v_j / sum_j p_j ),    p_j = ex2.approx.ftz(fma(s_j, sl2, -m)),

with s_j = q . k_j from wgmma (fp32 accumulation), sl2 = fp32(scale * log2(e)) (exactly 1 when scale = ln 2), m the
lazy reference of softmax_tile (at most 8 below the row max in log2 units, never above it), l = sum_j p_j added in fp32
from the fp32 p_j, and O = sum_j bf16(p_j) v_j accumulated in fp32 by the P.V wgmma, both rescaled by alpha =
ex2(m_old - m_new) when m moves.  The reference takes the bf16 inputs at their exact values and evaluates
w_j = 2^(x_j - max x) / sum, x_j = (q . k_j) sl2, and o64 = sum_j w_j v_j in float64; A[r, d] = sum_j w_j |v_jd|.

The per-element bound on |o - o64| is the sum of
  * P rounded to bf16 in the numerator only (pack_bf16x2 is round-to-nearest, relative error <= 2^-8):  2^-8 A;
  * score and exponential errors, common to numerator and denominator:  sum_j w_j eta_j |v_jd - o64_d|, bounded by
    (W eta) |V| + (sum_j w_j eta_j) |o64| and doubled for second-order terms, with eta_j (relative error of p_j, capped
    at 1) = ln 2 (sl2 S_REL sum_i |q_i k_ji| + 2^-24 (|x_j - max x| + 8)) + 2^-22: the wgmma score error of a 128-term
    bf16 dot product, the rounding of the fma argument (|x_j - m| <= |x_j - max x| + 8), and ex2.approx.  The
    rounding of m itself is common to every p of the row and cancels;
  * fp32 accumulation of O and l, and the alpha rescales:  ((ACC_PER_TILE n_kv + ACC_C) 2^-24 + n_kv 2^-22)(A + |o64|);
  * flushed exponentials (ex2.approx.ftz, and an alpha flushed to 0):  Lk 2^-118 max|v|;
  * the output rounding:  one bf16 spacing at |o64|;
and the sum is multiplied by MARGIN = 2.  The terms are worst cases, but the first and the last add up: a row whose
weight sits on one key of fractional exponent (P = 2^f rounded to bf16, by up to 2^-8) can reach 0.75 of the unscaled
sum, and a torch-fp32 emulation of the kernel reaches 0.59 over the cases of tests/test_attn_ref64_cpu.py; the margin
keeps the kernel's own approximations (ex2.approx, the wgmma accumulator) clear of the bar.

A diffuse row (thousands of keys of similar weight) has A ~ 0.8 max|v| against |o64| ~ max|v| / sqrt(Lk), so the
2^-8 A term exceeds the kernel's actual error by two orders of magnitude: the bound cannot see a dropped tile there.
The statistical check closes that gap.  The bf16 roundings of P and of the output are independent with variances
(2^-16 / 3) p^2 (at most; uniform error over a spacing of 2^-7 p) and spacing^2 / 12, so the 128-element error norm of
one (row, head) has expectation below sigma, sigma^2 = sum_d [(2^-16 / 3) sum_j w_j^2 v_jd^2 + spacing(o64_d)^2 / 12]
(the other error terms are orders smaller for such rows); it must be at most SIGMA_BAR sigma.  128 terms concentrate
the norm within a few percent of its mean, so 6 sigma leaves room for the approximations and none for a real error:
dropping one of 55 KV tiles moves a diffuse row by about 50 sigma.

Scores beyond a few thousand (log2 units) make eta meaningless (2^-24 |x| approaches 1): such inputs are checked
by their relative L2 error only.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
LN2 = math.log(2.0)
BF16_P = 2.0 ** -8          # relative rounding error of bf16 P (round to nearest, 8 significant bits)
EX2_REL = 2.0 ** -22        # ex2.approx.ftz.f32, PTX ISA maximum relative error
S_REL = 2.0 ** -16          # score error per unit of sl2 sum |q k|: 128 roundings of up to 2^-23 (wgmma truncates)
ACC_PER_TILE = 16           # fp32 roundings per KV tile on the O and l chains: 8 k-steps of the P.V wgmma, each up
ACC_C = 8                   # to one ulp (2^-23); the normalisation and the quad reduction of l add a few more
FLUSH = 2.0 ** -118         # per key: flushed p (< 2^-126), or an earlier tile's p <= 2^8 behind a flushed alpha
MARGIN = 2.0
SIGMA_BAR = 6.0
TILE = 128


def scale_log2(scale: float) -> float:
    """sl2 as attn_wgmma.cu computes it: fp32(scale * 1.4426950408889634f), or exactly 1 within 1e-6 of it."""
    s = np.float32(scale) * np.float32(1.4426950408889634)
    return 1.0 if abs(float(s) - 1.0) < 1e-6 else float(np.float32(s))


def bf16_spacing(x: torch.Tensor) -> torch.Tensor:
    """Spacing of the bf16 grid at |x| (float64), down to bf16's smallest normal spacing 2^-133."""
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), (e - 8).clamp_min(-133))


class Reference:
    """float64 o64, the per-element bound and sigma of the query rows `rows` (all rows when None).
    q [Lq, heads*128], k and v [Lk, heads*128] token-major (V, not V^T), any dtype and device (evaluated there)."""

    def __init__(self, q, k, v, heads, scale, rows=None, block=1024):
        self.sl2 = scale_log2(scale)
        Lk = k.shape[0]
        n_kv = (Lk + TILE - 1) // TILE
        qs = q if rows is None else q[rows]
        R = qs.shape[0]
        dev = q.device
        self.o = torch.empty(R, heads * 128, dtype=torch.float64, device=dev)
        self.bound = torch.empty_like(self.o)
        self.sigma = torch.empty(R, heads, dtype=torch.float64, device=dev)
        acc = (ACC_PER_TILE * n_kv + ACC_C) * U + n_kv * EX2_REL
        for h in range(heads):
            hs = slice(h * 128, (h + 1) * 128)
            kh, vh = k[:, hs].double(), v[:, hs].double()
            kabs, vabs = kh.abs(), vh.abs()
            flush = Lk * FLUSH * float(vabs.max())
            for r0 in range(0, R, block):
                qh = qs[r0:r0 + block, hs].double()
                x = (qh @ kh.T) * self.sl2
                xm = x - x.amax(1, keepdim=True)
                p = torch.exp2(xm)
                w = p / p.sum(1, keepdim=True)
                o = w @ vh
                A = w @ vabs
                eta = LN2 * (self.sl2 * S_REL * (qh.abs() @ kabs.T) + U * (xm.abs() + 8.0)) + EX2_REL
                we = w * eta.clamp(max=1.0)
                pert = we @ vabs + we.sum(1, keepdim=True) * o.abs()
                sp = bf16_spacing(o)
                self.o[r0:r0 + block, hs] = o
                self.bound[r0:r0 + block, hs] = MARGIN * (BF16_P * A + 2 * pert + acc * (A + o.abs()) + flush + sp)
                var = (2.0 ** -16 / 3) * ((w * w) @ (vh * vh)) + sp * sp / 12
                self.sigma[r0:r0 + block, h] = var.sum(1).sqrt()
        self.heads = heads

    def ratios(self, out):
        """(largest |out - o64| / bound over the elements, largest ||out - o64||_2 / (SIGMA_BAR sigma) over the (row,
        head) pairs, index (row, head) of the latter).  out [R, heads*128], the kernel's rows in the order of `rows`."""
        d = out.double().to(self.o.device) - self.o
        e = float((d.abs() / self.bound).max()) if d.numel() else 0.0
        n = d.reshape(d.shape[0], self.heads, 128).norm(dim=2)
        s = torch.where(n == 0, torch.zeros_like(n), n / (SIGMA_BAR * self.sigma))
        i = int(s.argmax())
        return e, float(s.reshape(-1)[i]), divmod(i, self.heads)

    def check(self, out, label=""):
        """Both checks of `out` (the rows of this reference); returns (element ratio, statistical ratio)."""
        assert torch.isfinite(out.float()).all(), f"{label}: non-finite output"
        e, s, (r, h) = self.ratios(out)
        print(f"attn_ref64 {label}: element/bound {e:.3g}, norm/(6 sigma) {s:.3g}")
        assert e <= 1.0, f"{label}: |o - o64| reaches {e:.3g} x the per-element bound"
        assert s <= 1.0, f"{label}: the error norm of row {r}, head {h} is {s:.3g} x {SIGMA_BAR} sigma"
        return e, s


def check(out, q, k, v, heads, scale, rows=None, label=""):
    """Both checks of the kernel output `out` [Lq, heads*128] (of its rows `rows` when given) against the float64
    reference of q, k and token-major v; returns (element ratio, statistical ratio), both must be <= 1."""
    return Reference(q, k, v, heads, scale, rows).check(out if rows is None else out[rows], label)
