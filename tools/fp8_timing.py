"""Measure the fp8 (e4m3) Linear mode against the bf16 forward on the benchmark's workload, in one process:

  * the full denoise step (7B DiT, latent [16,16,88,160], 512-token context, random weights), mode off and on,
    alternating, with the per-category device time of g3c_dit_profile;
  * g3c_gemm_fp8 against g3c_gemm_bf16 and torch._scaled_mm (row-wise scales) at the block's four GEMM shapes for
    M = 56 320 tokens;
  * the rel-L2 of the fp8 x_(t-1) against the bf16 one;
  * the card name, power limit and SM clock, read in the same run.

    python tools/fp8_timing.py [--rounds 3] [--steps 2] [--out DIR]

Prints one JSON object and writes it to DIR/fp8_timing.json when --out is given.  Needs an H100; nothing falls back."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def time_ms(torch, fn, iters):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def gemm_bench(torch, M, iters):
    from gen3c_b200 import ops

    D, Fd = 4096, 16384
    shapes = {"q/k/v/out [M,D]x[D,D]": (M, D, D), "V^T [D,M] (swapped)": (D, M, D), "layer1 [M,F]": (M, Fd, D),
              "layer2 [M,D] K=F": (M, D, Fd)}
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    for name, (m, n, k) in shapes.items():
        a = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
        b = (0.02 * torch.randn(n, k, device="cuda", generator=g)).to(torch.bfloat16)
        a8, sa = ops.quantize_rows_fp8(a)
        b8, sb = ops.quantize_rows_fp8(b)
        out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
        flop = 2.0 * m * n * k
        r = {"M": m, "N": n, "K": k}
        r["bf16_ms"] = time_ms(torch, lambda: ops.gemm(a, b, out=out), iters)
        r["fp8_ms"] = time_ms(torch, lambda: ops.gemm_fp8(a8, sa, b8, sb, out=out), iters)
        sa2, sb2 = sa[:, None].contiguous(), sb[None, :].contiguous()
        r["torch_scaled_mm_ms"] = time_ms(
            torch, lambda: torch._scaled_mm(a8, b8.t(), scale_a=sa2, scale_b=sb2, out_dtype=torch.bfloat16), iters)
        for key in ("bf16", "fp8", "torch_scaled_mm"):
            r[key + "_tflops"] = flop / (r[key + "_ms"] * 1e-3) / 1e12
        ref = torch._scaled_mm(a8, b8.t(), scale_a=sa2, scale_b=sb2, out_dtype=torch.bfloat16).float()
        got = ops.gemm_fp8(a8, sa, b8, sb).float()
        r["fp8_vs_scaled_mm_rel_l2"] = float((got - ref).norm() / ref.norm())
        res[name] = r
        del a, b, a8, b8, out, ref, got
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gemm-iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    from gen3c_b200 import _lib, sampler

    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    result = {"card_before": card()}
    result["gemm_M56320"] = gemm_bench(torch, 16 * 44 * 80, args.gemm_iters)

    net = bench.build_net(torch, dev)
    LAT, CTX, bf = bench.LAT, bench.CTX, torch.bfloat16
    g = torch.Generator().manual_seed(1)
    sch = sampler.EDMEulerScheduler().set_timesteps(35)
    d = {"xt": (torch.randn(LAT, generator=g) * sch.init_noise_sigma).to(bf), "gt": (0.5 * torch.randn(LAT, generator=g)).to(bf),
         "noise": sampler.arch_invariant_rand(LAT, 1), "pose": (0.5 * torch.randn(64, *LAT[1:], generator=g)).to(bf),
         "mask": torch.zeros(1, *LAT[1:]).to(bf), "ctx_c": torch.randn(CTX, generator=g).to(bf),
         "ctx_u": torch.randn(CTX, generator=g).to(bf), "pad": torch.zeros(LAT[2], LAT[3]).to(bf)}
    d["mask"][:, 0] = 1
    ind = torch.zeros(LAT[1])
    ind[0] = 1.0
    d = {k: v.to(dev) for k, v in d.items()}
    ind = ind.to(dev)
    sig = [float(s) for s in sch.sigmas]
    lib = _lib.load()

    def step(i):
        return sampler.denoise_step(net, d["xt"], d["gt"], d["noise"], ind, d["mask"], d["pose"], d["pad"], d["ctx_c"],
                                    d["ctx_u"], sig[i % 34], sig[i % 34 + 1], 1.0)

    names = ["gemm", "attn_self", "attn_cross", "eltwise", "comm", "vector"]
    runs = {"bf16": [], "fp8": []}
    x_next = {}
    for r in range(args.rounds):
        for mode in ("bf16", "fp8"):
            (net.enable_fp8_linear if mode == "fp8" else net.disable_fp8_linear)()
            for i in range(args.warmup):
                step(i)
            if r == 0:
                x_next[mode] = step(0).float().clone()
            torch.cuda.synchronize()
            _lib.check(lib.g3c_dit_profile(net._engine(), 1), "g3c_dit_profile")
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(args.steps):
                step(i)
            e.record()
            torch.cuda.synchronize()
            cat_ms, cat_n = (C.c_float * 6)(), (C.c_int * 6)()
            _lib.check(lib.g3c_dit_profile_read(net._engine(), cat_ms, cat_n, 6), "g3c_dit_profile_read")
            _lib.check(lib.g3c_dit_profile(net._engine(), 0), "g3c_dit_profile")
            ms = s.elapsed_time(e) / args.steps
            runs[mode].append({"ms_per_step": ms, "steps_per_s": 1e3 / ms,
                               "category_ms_per_step": {n: cat_ms[j] / args.steps for j, n in enumerate(names)},
                               "launches_per_step": cat_n[0] // args.steps + sum(cat_n[j] for j in range(1, 6)) // args.steps})
            print(mode, f"round {r}: {ms:.1f} ms/step, GEMM {cat_ms[0] / args.steps:.1f} ms, "
                  f"eltwise {cat_ms[3] / args.steps:.1f} ms", flush=True)
    result["step"] = runs
    result["x_next_fp8_vs_bf16_rel_l2"] = float((x_next["fp8"] - x_next["bf16"]).norm() / x_next["bf16"].norm())
    result["fp8_weight_and_workspace_bytes"] = net.workspace_bytes()
    result["card_after"] = card()
    txt = json.dumps(result, indent=1)
    print(txt)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_timing.json"), "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
