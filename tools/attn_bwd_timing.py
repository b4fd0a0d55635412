"""Timing of the differentiable drop-in attention at the benchmark's self-attention shape (Lq = Lk = 56 320, 32 heads,
head dim 128, scale = ln 2), sbhd tensors:

  fwd       g3c_attn_fwd_sbhd (ops.attention_sbhd without grad)
  fwd_lse   g3c_attn_fwd_sbhd_lse (the forward inside an autograd graph)
  bwd       g3c_attn_bwd_sbhd (Delta, dK/dV and dQ launches)
  torch_bwd torch's bf16 scaled_dot_product_attention backward on the same tensors (graph retained, backward only)

    python tools/attn_bwd_timing.py [--rounds 3] [--launches 5] [--lk LK]

The four are timed in alternation, `launches` launches each per round between CUDA events, for `rounds` rounds; the
JSON line gives every round's ms per launch, the median, and TFLOP/s: the forward on 4 Lq Lk 128 heads, the backward on
the algorithmic 10 Lq Lk 128 heads (dV, dP, dQ, dK and the recomputed S: 5 products) with the 14 Lq Lk 128 heads the
native backward executes (S and dP computed in both of its kernels: 7 products) beside it.  The card name and power
limit are read with nvidia-smi (--query-gpu only; nothing is set) in the same run."""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L, HEADS = 56320, 32


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--lk", type=int, default=L)
    args = ap.parse_args()
    Lk = args.lk

    import torch

    from gen3c_b200 import ops

    assert torch.cuda.is_available(), "attn_bwd_timing needs a CUDA device"
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(7)
    scale = math.log(2.0)
    q = (torch.randn(L, 1, HEADS, 128, device=dev, generator=g) * (128 ** -0.5 * 1.4426950408889634)).to(torch.bfloat16)
    k, v = (torch.randn(Lk, 1, HEADS, 128, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    do = torch.randn(L, 1, HEADS * 128, device=dev, generator=g).to(torch.bfloat16)
    o, lse = ops.attention_sbhd_lse(q, k, v, scale)
    qt, kt, vt = (t.permute(1, 2, 0, 3).detach().requires_grad_() for t in (q, k, v))
    eff = scale  # q carries log2(e) / sqrt(128); torch takes the natural-log scale: the same scores
    ot = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, scale=eff)
    dot = do.view(L, 1, HEADS, 128).permute(1, 2, 0, 3)

    work = {
        "fwd": lambda: ops.attention_sbhd(q, k, v, scale),
        "fwd_lse": lambda: ops.attention_sbhd_lse(q, k, v, scale),
        "bwd": lambda: ops.attention_sbhd_backward(q, k, v, o, lse, do, scale),
        "torch_bwd": lambda: torch.autograd.grad(ot, (qt, kt, vt), dot, retain_graph=True),
    }
    for fn in work.values():  # warm-up: module load, algorithm choice
        fn()
    torch.cuda.synchronize()
    ms = {name: [] for name in work}
    for _ in range(args.rounds):
        for name, fn in work.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.launches):
                fn()
            b.record()
            b.synchronize()
            ms[name].append(a.elapsed_time(b) / args.launches)
    med = {name: statistics.median(t) for name, t in ms.items()}
    f_fwd, f_bwd, f_exec = 4.0 * L * Lk * 128 * HEADS, 10.0 * L * Lk * 128 * HEADS, 14.0 * L * Lk * 128 * HEADS
    out = {
        "shape": f"{L} x {Lk} x {HEADS} heads x 128, scale ln 2",
        "gpu": gpu_info(),
        "ms_per_launch": {name: [round(x, 3) for x in t] for name, t in ms.items()},
        "median_ms": {name: round(x, 3) for name, x in med.items()},
        "tflops_fwd": {n: round(f_fwd / med[n] / 1e9, 1) for n in ("fwd", "fwd_lse")},
        "tflops_bwd_algorithmic_10": {n: round(f_bwd / med[n] / 1e9, 1) for n in ("bwd", "torch_bwd")},
        "tflops_bwd_executed_14": round(f_exec / med["bwd"] / 1e9, 1),
        "flop_bwd_algorithmic": f_bwd,
        "bwd_over_torch_bwd": round(med["bwd"] / med["torch_bwd"], 3),
        "fwd_lse_over_fwd": round(med["fwd_lse"] / med["fwd"], 4),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
